/* nope_nerf_b200 — C ABI of the H100-native (sm_90a) NoPe-NeRF render / pose-optimisation hot path.
 *
 * The reference (ActiveVisionLab/nope-nerf @ 47c861f6) is pure Python/PyTorch and has no
 * FFI layer (SURVEY.md 8(b)); the drop-in boundary is its Python class surface.  The host
 * mirror of that surface (nope_nerf_b200/model/) binds THIS library with ctypes; the
 * reference-side stub a maintainer would add is shown in INTEGRATION.md.
 *
 * Conventions: every pointer is a DEVICE pointer unless named host_*; fp32 contiguous;
 * buffers are borrowed for the duration of the call; all work is enqueued on `stream`
 * (a cudaStream_t passed as void*), nothing synchronises; return 0 = ok, negative = error
 * (nnb_last_error() gives the message, thread-local).  No exceptions cross the ABI, no
 * hidden allocations: scratch memory is a caller-provided workspace sized by
 * nnb_workspace_bytes().
 */
#ifndef NOPE_NERF_B200_H
#define NOPE_NERF_B200_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define NNB_NUM_PARAMS 595844 /* OfficialStaticNerf, hidden_dim 256 (model/official_nerf.py:20-37) */

/* rendering flags (configs/default.yaml:32-44 -> model/rendering.py:41-46) */
#define NNB_DIST_ALPHA 1u   /* rendering.dist_alpha     (rendering.py:122-128, official_nerf.py:82) */
#define NNB_NDC 2u          /* rendering.sample_option == 'ndc' (rendering.py:168-180)           */
#define NNB_NORMALISE 4u    /* rendering.normalise_ray  (rendering.py:68-71)                      */
#define NNB_USE_DIR 8u      /* rendering.use_ray_dir    (rendering.py:103-104)                    */
#define NNB_WHITE_BG 16u    /* rendering.white_background (rendering.py:145-147)                  */
#define NNB_EVAL 32u        /* eval_ argument           (rendering.py:150-154)                    */
#define NNB_SOFTPLUS 64u    /* model.occ_activation == 'softplus' (official_nerf.py:77-80)        */
#define NNB_SHIFT_FIRST 128u /* training.shift_first    (training.py:241-245)                     */
#define NNB_STASH 256u      /* keep activations in the workspace for nnb_render_bwd               */
#define NNB_RAW_DENSITY 2048u /* nnb_field_fwd/bwd only: out_rgba[3] = the density LOGIT (fc_density output, official_nerf.py:66-67
                                * infer_occ) instead of alpha / sigma; used for OfficialStaticNerf.gradient() (normals)            */
#define NNB_HVP 16384u      /* with NNB_STASH on NNB_ENGINE_SIMT: the workspace also holds the tangent stash of nnb_field_hvp; sizes only */
#define NNB_OCC_ONLY 32768u /* nnb_field_fwd on NNB_ENGINE_TC only: out_rgba = (0, 0, 0, a); the colour branch (fc_feature, rgb_layers.0,
                             * fc_rgb) is not evaluated.  a is bit-identical to the full query's (OfficialStaticNerf.forward(only_occupancy=True)) */
/* A flag bit not defined above is rejected (rc -7) by nnb_render_fwd / bwd, nnb_field_fwd / bwd / hvp and nnb_debug_wgrad, and
 * nnb_workspace_bytes(_dim) returns 0 for it.  Bits 512, 1024, 4096 and 8192 were defined before version 105 and are rejected too. */

/* engines */
#define NNB_ENGINE_SIMT 0 /* exact fp32 FMA path                                        */
#define NNB_ENGINE_TC 1   /* wgmma tensor cores, split 16-bit (hi/lo) operands, fp32 acc */

/* One ray batch of one camera.  Mirrors the arguments of nope_nerf.forward
 * (model/network.py:19-20) + Renderer.nope_nerf (model/rendering.py:36-37) after the host
 * mirror has resolved world_mat -> c2w (training.py:238 / common.py:139-141). */
typedef struct nnb_render_args {
  const float* weights;   /* [nnb_num_params(hidden_dim)] flat, OfficialStaticNerf.parameters() order */
  const float* c2w;       /* [16] row-major camera-to-world (LearnPose.forward, poses.py:23-31)     */
  const float* cam;       /* [16] camera_mat diag(kx,ky,-1,1) (dataset.py:101-104); [0],[5] are read */
  const int64_t* ray_idx; /* [N] row-major pixel ids (training.py:257) or NULL                      */
  const float* pixels;    /* [N,2] in [-1,1] (common.py:13-39) or NULL -> derived from ray_idx,H,W  */
  const float* depth;     /* [N] prior depth per ray, or NULL -> gathered from depth_map           */
  const float* depth_map; /* [h_d,w_d] raw DPT map (network.py:22-24 nearest gather)                */
  const float* scale;     /* [1] depth distortion scale or NULL (=1)  (distortions.py:19-27)        */
  const float* shift;     /* [1] depth distortion shift or NULL (=0)                                */
  const float* noise;     /* [N,S] stratified jitter U[0,1) (rendering.py:189) or NULL              */
  /* S = rendering.num_points, samples per ray: 2..1024 on NNB_ENGINE_SIMT, 16..1024 on NNB_ENGINE_TC; other values are rejected
   * (rc < 0).  The Python package runs S < 16 on the SIMT engine and every other S on the tensor-core engine by default. */
  int32_t N, S, H, W, h_d, w_d;
  float near_, far_;      /* rendering.depth_range                                                  */
  uint32_t flags;
  int32_t engine;
  /* outputs (rendering.py:159-166; depth_* are dense, `mask` selects the reference's rows) */
  float* rgb;        /* [N,3] */
  float* depth_pred; /* [N]   */
  float* depth_gt;   /* [N]   */
  uint8_t* mask;     /* [N]   */
  float* z_vals;     /* [N,S] or NULL */
  float* alpha;      /* [N,S] or NULL */
  void* workspace;
  size_t workspace_bytes;
  /* explicit-point field queries (nnb_field_fwd/bwd/hvp/vjp only; nnb_render_fwd / nnb_render_bwd never read them):
   * OfficialStaticNerf.forward(p, ray_d) */
  const float* pts;  /* [N,3] */
  const float* dirs; /* [N,3] or NULL (-> ones, like use_ray_dir = False) */
  /* model.hidden_dim (official_nerf.py:11): 64, 128 or 256; 0 means 256.  `weights` / g_weights then hold nnb_num_params(hidden_dim)
   * floats and the workspace is sized by nnb_workspace_bytes_dim(..., hidden_dim).  Other widths are rejected (rc < 0). */
  int32_t hidden_dim;
} nnb_render_args;

typedef struct nnb_render_bwd_args {
  nnb_render_args fwd;       /* same inputs / workspace as the forward call (NNB_STASH set)  */
  const float* g_rgb;        /* [N,3] */
  const float* g_depth_pred; /* [N] dense (0 where masked out) or NULL */
  const float* g_depth_gt;   /* [N] dense or NULL                      */
  /* outputs, all ACCUMULATED (+=): caller zeroes them.  Reproducible: every reduction runs in a fixed order, so the same inputs give
   * the same bits on every run.  g_weights gets plain adds (and g_depth is overwritten): no other work may write them during the call.  g_c2w, g_cam
   * and g_scale_shift get one atomic add per element: other work may add into them concurrently (the sums stay correct), but the bits
   * are reproducible only when that work is ordered before or after the call. */
  float* g_weights; /* [nnb_num_params(fwd.hidden_dim)] or NULL (pose-only: Trainer_pose, eval_pose_one_epoch.py:25-41) */
  float* g_c2w;     /* [16] (rows 0..2 written) */
  float* g_cam;     /* [16] ([0],[5] written) or NULL */
  float* g_depth;   /* [N] d/d prior depth (overwritten) or NULL */
  float* g_scale_shift; /* [2] d/d scale, d/d shift when depth_map is used, or NULL */
} nnb_render_bwd_args;

const char* nnb_last_error(void);
int nnb_version(void);   /* >= 101: nnb_chamfer with adjoints takes nnb_chamfer_workspace_bytes(P, Q) of keys; >= 102: nnb_field_hvp;
                          * >= 103: nnb_field_fwd honours NNB_ENGINE_TC, NNB_OCC_ONLY; >= 104: nnb_ray_march;
                          * >= 105: nnb_render_bwd_args ends at g_scale_shift.  Its former trailing fields phase, wg_state and wg_seed are
                          *   gone, so every nnb_render_bwd call runs the whole backward: a caller that still issues a phase-1 call and
                          *   then a phase-2 call runs the backward twice.  NNB_TCBWD (512), NNB_WG16 (1024), NNB_FWD_DROP_WLO (4096)
                          *   and NNB_FWD_DROP_ALO (8192) are removed and rejected as undefined bits. */
/* Profiling hook used by bench.py: `events` is a HOST array of cudaEvent_t handles that stays alive until
 * nnb_profile_events(NULL,0).  Every nnb_render_fwd records 4 marks (start, weights imaged, field done,
 * composited) and every nnb_render_bwd 5 marks (start, compositing adjoint, data-gradient chain,
 * weight gradients, ray adjoint) on the call's stream, consuming the array in order. */
int nnb_profile_events(void** events, int32_t count);
int nnb_profile_cursor(void);
/* test aid: byte offsets of the workspace sections {records, h0..h7, feat, hr, enc, denc, total} */
int nnb_debug_layout(int32_t N, int32_t S, uint32_t flags, int32_t engine, size_t* out14);
/* test aid: the weight-gradient stage that nnb_render_bwd runs for a->engine, alone, on whatever the workspace's activation / output-
 * gradient stash holds (layout of nnb_debug_layout); g_weights [nnb_num_params(a->hidden_dim)] is ACCUMULATED (+=).  Reads a->N, S,
 * flags (NNB_STASH required), engine, hidden_dim, workspace and workspace_bytes only. */
int nnb_debug_wgrad(const nnb_render_args* a, float* g_weights, void* stream);
/* bytes of workspace needed by nnb_render_fwd (+bwd when NNB_STASH) at hidden_dim 256; 0 for an undefined flag bit */
size_t nnb_workspace_bytes(int32_t N, int32_t S, uint32_t flags, int32_t engine);
/* the same for the field of width hidden_dim (0 = 256); 0 for an unsupported width or an undefined flag bit */
size_t nnb_workspace_bytes_dim(int32_t N, int32_t S, uint32_t flags, int32_t engine, int32_t hidden_dim);
/* floats of the flat MLP parameter vector of width hidden_dim (0 = 256; NNB_NUM_PARAMS at 256); 0 for an unsupported width */
size_t nnb_num_params(int32_t hidden_dim);
int nnb_render_fwd(const nnb_render_args* a, void* stream);
/* OfficialStaticNerf.forward(p, ray_d, return_addocc=True) on explicit points (model/official_nerf.py:69-96).  Uses a->pts/dirs,
 * N points (S is ignored), weights, flags (NNB_DIST_ALPHA / NNB_SOFTPLUS / NNB_RAW_DENSITY / NNB_STASH) and the workspace;
 * out_rgba [N,4] = (r,g,b, alpha-or-sigma-or-logit).  nnb_field_bwd: g_rgba [N,4] -> g_pts [N,4], g_dirs [N,4] (xyz used),
 * g_weights (+=, may be NULL).
 * Engine of nnb_field_fwd: a->engine == NNB_ENGINE_TC runs the tensor-core kernel (inference only); every other value runs the
 * exact-fp32 engine, as in versions < 103, which ignored the field.  nnb_field_bwd and nnb_field_hvp always run exact fp32; the data
 * gradients alone run on tensor cores through nnb_field_vjp.
 *   NNB_ENGINE_TC: flags NNB_DIST_ALPHA / NNB_SOFTPLUS / NNB_RAW_DENSITY / NNB_OCC_ONLY.  NNB_STASH is rejected (rc -6): gradients
 *   need the exact-fp32 engine.  The workspace holds nnb_workspace_bytes_dim(N, 1, flags, NNB_ENGINE_TC, hidden_dim) bytes, 256-byte
 *   aligned; out_rgba is 16-byte aligned; c2w / cam / ray_idx are not read.  Rows of out_rgba past N are not written.
 *   Precision: every layer is the split-fp16 product of the render path (three MMAs a_lo*b_hi + a_hi*b_lo + a_hi*b_hi, 22-bit
 *   operands, fp32 accumulation): outputs agree with float64 to about 1e-6 of the tensor's maximum.  fp16 halves have a limited
 *   exponent range: the low half is a normal number only for |x| above about 2^-3, is subnormal (absolute quantum 2^-24) below
 *   that, and an operand below about 6e-8 vanishes, so a field whose activations are very small is evaluated less accurately than
 *   on the exact engine.
 *   Every other engine value: NNB_OCC_ONLY is rejected (rc -6); the workspace rule is that of NNB_ENGINE_SIMT. */
int nnb_field_fwd(const nnb_render_args* a, float* out_rgba, void* stream);
int nnb_field_bwd(const nnb_render_args* a, const float* g_rgba, float* g_pts, float* g_dirs, float* g_weights, void* stream);
/* Second-order backward of the surface normal n(p) = d s / d p, s the density logit (OfficialStaticNerf.gradient with
 * create_graph=True, official_nerf.py:46-58): for a cotangent u [N,4] (xyz used) on n, with s' = u . n,
 *   g_pts [N,4] = d s' / d p (xyz; overwritten; may be NULL),  g_weights += sum over the points of d s' / d weights (may be NULL).
 * Recomputes everything from a->pts and a->weights (forward, data-gradient chain, tangent chain, weight gradients); reads a->pts, N,
 * weights, hidden_dim, workspace.  a->flags must contain NNB_STASH | NNB_HVP and the workspace be sized by
 * nnb_workspace_bytes_dim(N, 1, flags, NNB_ENGINE_SIMT, hidden_dim); dirs and the activation flags do not enter (the logit is raw).
 * u and g_pts are 16-byte aligned.  Exact-fp32 engine; every sum runs in a fixed order, so the same inputs give the same bits. */
int nnb_field_hvp(const nnb_render_args* a, const float* u, float* g_pts, float* g_weights, void* stream);
/* Data gradients of OfficialStaticNerf.forward on explicit points, tensor-core engine: forward and data-gradient chain in one call (the
 * surface normals of the geometry view: NNB_RAW_DENSITY | NNB_OCC_ONLY with g_rgba = (0, 0, 0, 1) gives g_pts = d logit / d p).
 * Reads a->pts [N,3], a->dirs [N,3] or NULL (ones), N, weights, hidden_dim, flags (NNB_DIST_ALPHA | NNB_SOFTPLUS | NNB_RAW_DENSITY |
 * NNB_OCC_ONLY), engine and the workspace;  g_rgba [N,4] is the cotangent on (r, g, b, a).
 *   out_rgba [N,4] (optional, NULL = not wanted): bit-identical to nnb_field_fwd on NNB_ENGINE_TC with the same flags.
 *   g_pts [N,4] (xyz; w is 0) = d<g_rgba, out>/d p;  g_dirs [N,4] (optional) = d<g_rgba, out>/d dirs (the ones when dirs is NULL).
 *   Overwritten, rows < N only.  There are no weight gradients: they, and nnb_field_bwd / nnb_field_hvp, stay on the exact engine.
 * NNB_OCC_ONLY: the colour branch is neither evaluated nor differentiated; g_rgba[:, :3] is not read and g_dirs must be NULL.
 * Errors, with nothing launched: an engine other than NNB_ENGINE_TC (rc -4); an undefined flag bit (-7); NNB_STASH or NNB_HVP (-6);
 * g_dirs with NNB_OCC_ONLY (-6); an unsupported width (-8); N < 0, a NULL pts / weights / g_rgba / g_pts, or one of g_rgba, out_rgba,
 * g_pts, g_dirs not 16-byte aligned (-3); a workspace smaller than nnb_field_vjp_workspace_bytes(N, flags, hidden_dim) or not 256-byte
 * aligned (-5).  N == 0 returns 0 and does nothing.
 * Precision: the forward is nnb_field_fwd's split-fp16 product (three MMAs per layer, fp32 accumulation), the chain runs through the
 * transposed weights as bf16 hi | lo products like the render backward (tc_dgrad), gated by the ReLU bits the forward writes; the
 * encoding adjoints are fp32.  Measured against float64 evaluated with the same ReLU gates: g_pts within 2.5e-5 of its maximum, g_dirs
 * within 1.1e-5, out_rgba within 3e-7 (the exact engine's gradients: within 1e-6).  Where a point's ReLU pre-activation lies within the
 * forward's rounding of 0 (measured: within 8e-7 of the layer's largest), this engine may gate that unit differently from float64 or from
 * the exact engine, and the gradient, which is discontinuous there, then differs by that unit's contribution.  The fp16 caveat of nnb_field_fwd
 * holds for the forward: a field whose activations are very small (below about 2^-3 the low half is subnormal, below about 6e-8 an
 * operand vanishes) is evaluated, and so gated, less accurately than on the exact engine.
 * A point's outputs depend on that point alone (not on N, its tile or its row), like the forward's.
 * Workspace, each section 256-byte aligned (Npad = N rounded up to 128, D = hidden_dim): per-point records (32 Npad bytes) | ReLU gate
 * bits of h0..h7 (Npad D bytes) and, unless NNB_OCC_ONLY, of the rgb hidden layer (Npad D / 16 bytes) | the forward weight image (its
 * occupancy-only prefix with NNB_OCC_ONLY) | the transposed weight image (its trunk part with NNB_OCC_ONLY).  The size query returns 0 for
 * N <= 0, an undefined flag bit or an unsupported width. */
size_t nnb_field_vjp_workspace_bytes(int32_t N, uint32_t flags, int32_t hidden_dim);
int nnb_field_vjp(const nnb_render_args* a, const float* g_rgba, float* out_rgba, float* g_pts, float* g_dirs, void* stream);
/* The whole first-order backward of OfficialStaticNerf.forward on explicit points, tensor-core engine: what nnb_field_fwd (NNB_STASH) +
 * nnb_field_bwd compute on the exact engine, in one call that recomputes everything from a->pts, a->dirs and a->weights (nothing is
 * carried over from an earlier forward, as in nnb_field_hvp).  It runs the points forward with the fp32 training stash, the data-gradient
 * chain of nnb_field_vjp with the dY stash, and the weight-gradient stage of the render backward (nnb_render_bwd on NNB_ENGINE_TC) on
 * that stash.  No version bump: the symbol marks the capability.
 * Reads a->pts [N,3], a->dirs [N,3] or NULL (ones), N, weights, hidden_dim, flags (NNB_DIST_ALPHA | NNB_SOFTPLUS | NNB_RAW_DENSITY |
 * NNB_OCC_ONLY), engine and the workspace;  g_rgba [N,4] is the cotangent on (r, g, b, a).
 *   out_rgba [N,4] (optional): bit-identical to nnb_field_fwd on NNB_ENGINE_TC with the same flags.
 *   g_pts [N,4], g_dirs [N,4] (optional): bit-identical to nnb_field_vjp with the same cotangent (xyz; w is 0; overwritten, rows < N).
 *   g_weights [nnb_num_params(hidden_dim)] (optional, 4-byte aligned) is ACCUMULATED (+=) with d<g_rgba, out>/d weights, like
 *   nnb_field_bwd; plain adds, so no other work may write it during the call.  NULL makes the call nnb_field_vjp (the stash is still
 *   written).
 * NNB_OCC_ONLY (infer_occ under autograd): the colour branch is neither evaluated nor differentiated; g_rgba[:, :3] is not read, g_dirs
 * must be NULL, and the slots of fc_feature, rgb_layers.0 and fc_rgb in g_weights are not touched.
 * Errors, with nothing launched (those of nnb_field_vjp): an engine other than NNB_ENGINE_TC (rc -4); an undefined flag bit (-7);
 * NNB_STASH or NNB_HVP, or g_dirs with NNB_OCC_ONLY (-6); an unsupported width (-8); N < 0, a NULL pts / weights / g_rgba / g_pts, one of
 * g_rgba, out_rgba, g_pts, g_dirs not 16-byte aligned or g_weights not 4-byte aligned (-3); a workspace smaller than
 * nnb_field_grad_workspace_bytes(N, flags, hidden_dim) or not 256-byte aligned (-5).  N == 0 returns 0 and does nothing.
 * Precision: the forward and the chain are those of nnb_field_fwd / nnb_field_vjp; the weight gradients are the render backward's (bf16
 * hi | lo products of the fp32 stash, fp32 accumulation; the heads in fp32).  Measured against float64 evaluated with the ReLU gates this
 * call's forward wrote (NVIDIA H100 80GB HBM3, every flag and width): every dW / db within 9.4e-5 of its tensor's maximum, g_pts within
 * 2.3e-5 and g_dirs within 1.4e-5 from 128 points on (a call of a few points has a g_pts maximum set by those points: 2.2e-4 at N = 1).  The
 * gate caveat of nnb_field_vjp holds: where a pre-activation lies within the forward's rounding of 0 this engine may gate a unit differently
 * from float64 or from the exact engine, and the gradients differ there by that unit's contribution.  The fp16 caveat of nnb_field_fwd
 * holds for the forward: a field whose activations are very small (below about 2^-3 the low half of an fp16 operand is subnormal, below
 * about 6e-8 an operand vanishes) is evaluated, and so gated and differentiated, less accurately than on the exact engine.
 * Determinism: every sum runs in a fixed order, so the same inputs give the same bits on every run; a point's out_rgba, g_pts and g_dirs
 * depend on that point alone.  The rows of the last tile past N have a zero cotangent and add exactly 0 to every dW / db, whatever the
 * workspace held before the call.
 * Workspace, each section 256-byte aligned (Npad = N rounded up to 128, D = hidden_dim): make_layout's layout for nnb_render_bwd at
 * N x 1 samples with NNB_STASH on NNB_ENGINE_TC (records, the fp32 activation and dY stash of Npad rows, the weight-gradient partials,
 * the ReLU gate bits) | the forward weight image (its occupancy-only prefix with NNB_OCC_ONLY) | the transposed weight image (its trunk
 * part with NNB_OCC_ONLY).  20 272 bytes per point at D = 256 (10 408 at 128, 5 476 at 64) plus a constant: 2 700 501 248 bytes (2.7 GB)
 * for 131 072 points at D = 256.  nnb_field_grad_workspace_bytes is the source of truth; it returns 0 for N <= 0, an undefined flag bit
 * or an unsupported width. */
size_t nnb_field_grad_workspace_bytes(int32_t N, uint32_t flags, int32_t hidden_dim);
int nnb_field_grad(const nnb_render_args* a, const float* g_rgba, float* out_rgba, float* g_pts, float* g_dirs, float* g_weights, void* stream);
/* The second-order field backward of nnb_field_hvp on the tensor-core engine: for the raw density logit s and a cotangent u on the
 * normals n = d s / d p, the gradients of s' = sum_m u[m] . n[m] to the points and the weights, recomputed from a->pts and a->weights in
 * one call.  It runs the occupancy-only forward of nnb_field_vjp (records, ReLU gate bits), its data-gradient chain for a cotangent 1 on
 * the logit with the dY stash and the point term, the tangent chain e' = J_enc(p) u, h'_l = [h_l > 0] (W_l x'_{l-1}) (no bias, gated with
 * the forward's bits), and the weight-gradient stage of nnb_field_grad on (dY, tangent) without bias jobs.  nnb_field_hvp is unchanged
 * and stays on the exact-fp32 engine.  No version bump: the symbol marks the capability.
 * Reads a->pts [N,3], N, weights, hidden_dim, flags, engine and the workspace (a->dirs is not read: the logit does not depend on the view
 * direction); the call always differentiates the raw logit of the occupancy-only query (NNB_RAW_DENSITY | NNB_OCC_ONLY are implied, and
 * NNB_DIST_ALPHA / NNB_SOFTPLUS do not change it).  u [N,4]: the cotangent on n (xyz; w is not read).
 *   g_pts [N,4] (optional): d s' / d p, only the encoding's diagonal second-derivative term (the ReLU masks are piecewise constant); xyz,
 *   w is 0; overwritten, rows < N.
 *   g_weights [nnb_num_params(hidden_dim)] (optional, 4-byte aligned) is ACCUMULATED (+=) with d s' / d weights, like nnb_field_hvp: only
 *   the slots of the trunk weights (layers 0..7) and of fc_density.weight are written; every bias slot and every colour slot is left
 *   untouched (s' has no bias term and no colour term).  Plain adds, so no other work may write it during the call.
 * Errors, with nothing launched, in nnb_field_grad's order: a NULL a (-3); an engine other than NNB_ENGINE_TC (-4); an undefined flag
 * bit (-7); NNB_STASH or NNB_HVP (-6); an unsupported width (-8); N < 0 (-3); then N == 0 returns 0 and does nothing; a NULL pts / weights
 * / u, or both g_pts and g_weights NULL, u or g_pts not 16-byte aligned, or g_weights not 4-byte aligned (-3); a workspace smaller than
 * nnb_field_hvp_tc_workspace_bytes(N, flags, hidden_dim) or not 256-byte aligned (-5).
 * Precision: the forward and its gates are those of nnb_field_vjp (occupancy-only); the chain is nnb_field_vjp's (bf16 hi | lo operands);
 * the tangent chain runs on bf16 hi | lo operands of the fp32 tangents and weights with fp32 accumulation (the fp16 hi | lo split of the
 * forward is inaccurate below about 2^-3, and tangents span the range of gradients: e' reaches 2^9 |u|); the weight gradients are
 * nnb_field_grad's.  Measured against float64 evaluated with the ReLU gates this call's forward wrote (NVIDIA H100 80GB HBM3, every
 * width): every dW within 7.9e-5 of its tensor's maximum, g_pts within 1.7e-5 at every size (DESIGN.md §4).  The gate caveat of
 * nnb_field_vjp holds: where a pre-activation lies within the forward's rounding of 0 this engine may gate a unit differently from float64
 * or from the exact engine.
 * Determinism: every sum runs in a fixed order, so the same inputs give the same bits on every run; a point's g_pts depends on that point
 * alone.  The rows of the last tile past N have u = 0 and a zero cotangent, so they add exactly 0 to every dW whatever the workspace held.
 * Workspace, each section 256-byte aligned (Npad = N rounded up to 128, D = hidden_dim): nnb_field_grad's occupancy-only layout (records,
 * the fp32 stash, whose h0..h7 / enc rows hold the tangent h'0..h'7 / e' here, the dY stash, the weight-gradient partials, the gate bits,
 * the occupancy-only forward image and the trunk part of the transposed image) | the bf16 image of the occupancy-only forward stages.
 * nnb_field_hvp_tc_workspace_bytes is the source of truth; it returns 0 for N <= 0, an undefined flag bit or an unsupported width. */
size_t nnb_field_hvp_tc_workspace_bytes(int32_t N, uint32_t flags, int32_t hidden_dim);
int nnb_field_hvp_tc(const nnb_render_args* a, const float* u, float* g_pts, float* g_weights, void* stream);
int nnb_render_bwd(const nnb_render_bwd_args* a, void* stream);

/* Fused ray marching of the geometry view: what Renderer.ray_marching + Renderer.secant (model/rendering.py:274-418) do for N rays, in
 * one stream-ordered call that never holds a point or an occupancy in global memory.  Ray n is sampled at the n_steps depths
 *   t_i = near_ (1 - frac[i]) + far_[n] frac[i],   p_i = ray0[n] + ray_dir[n] t_i,   val_i = occupancy(p_i) - tau,
 * the occupancy being OfficialStaticNerf.forward(only_occupancy=True) (alpha, or sigma with NNB_DIST_ALPHA; NNB_SOFTPLUS as in the
 * render).  first = the smallest i with val_i val_{i+1} < 0 (the rounded fp32 product, so a product that underflows to 0 is no sign
 * change).  The ray hits when first exists, val_first < 0 and val_0 < 0; its bracket (d_low, d_high, f_low, f_high) = (t_first,
 * t_{first+1}, val_first, val_{first+1}) is then refined by n_secant secant steps d = -f_low (d_high - d_low) / (f_high - f_low) + d_low,
 * f_mid = occupancy(ray0 + d ray_dir) - tau, f_mid < 0 ? (d_low, f_low) = (d, f_mid) : (d_high, f_high) = (d, f_mid).
 *   depth [N]: the secant iterate of the final bracket on a hit; 0 where val_0 >= 0 (the first sample is occupied), whatever follows;
 *     +inf otherwise.
 *   first [N] (optional, NULL = not wanted): the index above; -1 where there is none or val_0 >= 0 (such a ray is not searched further).
 *   bracket [N,4] (optional, 16-byte aligned): the bracket before the secant steps on a hit, zeros elsewhere.
 * Engine: tensor cores only.  engine != NNB_ENGINE_TC is rejected (rc < 0); the exact-fp32 engine's fused march is nnb_ray_march_engine
 * (below).  Precision is that of nnb_field_fwd on NNB_ENGINE_TC.
 * Bit-equality contract: on this engine a point's occupancy does not depend on the tile or row that evaluates it, and every product, sum
 * and quotient above is rounded on its own in the order of the torch code.  depth, first and bracket are therefore bit-identical to
 * Renderer.ray_marching / secant run on nnb_field_fwd(NNB_ENGINE_TC | NNB_OCC_ONLY) with frac = torch.linspace(0, 1, n_steps) (passed in,
 * so the library does not reproduce linspace's rounding).
 * Work: the rays advance in rounds of 128 steps; a ray whose first sign change (or occupied first sample) has been seen takes no part in
 * later rounds, so a ray costs ceil((first + 2) / 128) tiles of 128 queries instead of n_steps queries.
 * The workspace holds nnb_ray_march_workspace_bytes(N, n_steps, hidden_dim) bytes, 256-byte aligned.  After the call its first
 * int32s are counters: [0] = rays that hit, [k] (1 <= k < ceil(n_steps / 128)) = rays that took part in round k.
 * N == 0 returns 0 and does nothing.  Nothing synchronises or allocates; every launch after the first sizes itself from a counter in
 * the workspace. */
typedef struct nnb_ray_march_args {
  const float* weights;  /* [nnb_num_params(hidden_dim)] */
  const float* ray0;     /* [N,3] */
  const float* ray_dir;  /* [N,3] */
  const float* far_;     /* [N] per-ray far depth */
  const float* frac;     /* [n_steps] */
  int32_t N, n_steps /* >= 2 */, n_secant /* >= 0 */, hidden_dim /* 64, 128, 256; 0 = 256 */;
  float near_, tau;
  uint32_t flags;        /* NNB_DIST_ALPHA | NNB_SOFTPLUS */
  int32_t engine;        /* NNB_ENGINE_TC (nnb_ray_march_engine: or NNB_ENGINE_SIMT) */
  float* depth; int32_t* first; float* bracket;
  void* workspace; size_t workspace_bytes;
} nnb_ray_march_args;
size_t nnb_ray_march_workspace_bytes(int32_t N, int32_t n_steps, int32_t hidden_dim);   /* 0 on bad sizes or an unsupported width */
int nnb_ray_march(const nnb_ray_march_args* a, void* stream);
/* nnb_ray_march on a->engine: NNB_ENGINE_TC (exactly nnb_ray_march) or NNB_ENGINE_SIMT, the exact-fp32 engine; any other engine is
 * rejected (rc -4), and the other checks and codes are nnb_ray_march's.  nnb_ray_march keeps its contract (tensor cores only).  No version
 * bump: the symbols mark the capability.
 * On NNB_ENGINE_SIMT the contract above holds with the occupancy of nnb_field_fwd on NNB_ENGINE_SIMT (the exact engine's fp32 FMA field,
 * the colour branch skipped).  A point's exact occupancy does not depend on its tile or row either, so depth, first and bracket are
 * bit-identical to Renderer.ray_marching / secant on the default (exact) engine with frac = torch.linspace(0, 1, n_steps).  The same rounds
 * of 128 steps, the same counters.  Its workspace is the layout above without a weight image, checked against
 * nnb_ray_march_workspace_bytes_engine(N, n_steps, hidden_dim, NNB_ENGINE_SIMT).
 * nnb_ray_march_workspace_bytes_engine: the workspace on `engine` (nnb_ray_march_workspace_bytes is this on NNB_ENGINE_TC); 0 on bad
 * sizes, an unsupported width or an engine without the march. */
int nnb_ray_march_engine(const nnb_ray_march_args* a, void* stream);
size_t nnb_ray_march_workspace_bytes_engine(int32_t N, int32_t n_steps, int32_t hidden_dim, int32_t engine);

/* The geometry view of any set of N pixels in one stream-ordered call: what Renderer.phong_renderer (model/rendering.py:148-180) does,
 * with every ray computed per pixel, on the tensor-core engine.  No version bump: the symbol marks the capability.
 *   Rays: cw = T[:3,3] (T row-major [16], T = S^-1 W^-1 K^-1 as Renderer._rays_world forms it), pw_r = ((T[r,0] x + T[r,1] y) + T[r,2])
 *     + T[r,3] for the pixel (x, y), d = pw - cw, |d| = sqrt((d0 d0 + d1 d1) + d2 d2), dir = d / |d|.
 *   Far (Renderer._sphere_far): dot = (dir0 cw0 + dir1 cw1) + dir2 cw2, c = sqrt((cw0 cw0 + cw1 cw1) + cw2 cw2),
 *     under = dot dot - (c c - radius radius), far = sqrt(under) - dot where under > 0, else 0; then clamped at 0.
 *   March: nnb_ray_march on (ray0 = cw, dir, far) from near_ over frac, n_secant secant steps (its contract, above).
 *   An object ray has a finite depth that is not 0.  Its surface point p = ray0 + dir depth (a product, then a sum, per component);
 *     grad = -d logit / d p (OfficialStaticNerf.gradient: nnb_field_vjp with NNB_RAW_DENSITY | NNB_OCC_ONLY and the cotangent
 *     (0, 0, 0, 1), negated); n = grad / sqrt((g0 g0 + g1 g1) + g2 g2); light = cw / |cw| (the same sum order);
 *     rgb = min(0.3 + 0.7 max((n0 l0 + n1 l1) + n2 l2, 0), 1) in every channel; rgb_surf = the rgb of nnb_field_fwd (NNB_ENGINE_TC) at
 *     (p, -dir).  The clamps are comparisons: a zero gradient gives NaN, which passes through them as through torch's clamp_min / clamp_max.
 *   Any other pixel: rgb = (1, 1, 1), rgb_surf = (0, 0, 0) (and grad = 0).
 * Every product, sum, quotient and square root above is rounded on its own (no FMA contraction), in the order written.
 * Pixel independence: a pixel's outputs depend on its coordinates, T, the weights and the scalar arguments alone, not on N, its position in
 * the list or the other pixels (every tensor-core query is independent of its row).  Splitting a frame into calls of any size gives the same
 * bits.  Renderer.phong_renderer's rays come from a batched matmul whose rounding depends on the pixel count, so a frame from this call
 * differs from that path's in the last bits of its rays.
 * Stage bit-equality, from the call's own ray0 / ray_dir / far_: depth is nnb_ray_march's; grad is the negated g_pts of nnb_field_vjp at p;
 * rgb_surf is nnb_field_fwd's (NNB_ENGINE_TC) at (p, -ray_dir).
 * Errors, with nothing launched: engine != NNB_ENGINE_TC (rc -4); an undefined flag bit (-7); a defined flag other than NNB_DIST_ALPHA /
 * NNB_SOFTPLUS (-6); an unsupported width (-8); N < 0, n_steps < 2 or n_secant < 0 (-2); a NULL weights / T / pixels / frac / rgb /
 * rgb_surf, a float pointer not 4-byte aligned or grad not 16-byte aligned (-3); a workspace smaller than
 * nnb_geometry_frame_workspace_bytes(N, n_steps, hidden_dim) or not 256-byte aligned (-5).  N == 0 returns 0 and launches nothing.
 * Nothing synchronises or allocates: every launch after the first sizes itself from a counter in the workspace.
 * Workspace, each section 256-byte aligned: hit count | ray0, dir (12 N bytes each), far, depth (4 N each) | compacted rows: surface
 * points, view directions (12 N each), pixel indices (4 N), normal cotangents, normals, colours (16 N each) | nnb_ray_march's workspace
 * for N rays | nnb_field_vjp's for N points with NNB_RAW_DENSITY | NNB_OCC_ONLY | the forward weight image of the points mode (all that
 * nnb_field_fwd's tensor-core query uses of its workspace).  N rows everywhere: the worst case, every ray hits.  At N = 1080 x 1920,
 * n_steps = 512, D = 256: 945 541 632 bytes (0.95 GB). */
typedef struct nnb_geometry_args {
  const float* weights;   /* [nnb_num_params(hidden_dim)] */
  const float* T;         /* [16] row-major S^-1 W^-1 K^-1 */
  const float* pixels;    /* [N,2] image-plane pixel coordinates (arange_pixels) */
  const float* frac;      /* [n_steps] = torch.linspace(0, 1, n_steps), as for nnb_ray_march */
  int32_t N, n_steps /* >= 2 */, n_secant /* >= 0 */, hidden_dim /* 64, 128, 256; 0 = 256 */;
  float near_, tau, radius;
  uint32_t flags;         /* NNB_DIST_ALPHA | NNB_SOFTPLUS (the occupancy of the march) */
  int32_t engine;         /* NNB_ENGINE_TC (nnb_geometry_frame_engine: or NNB_ENGINE_SIMT) */
  float* rgb;             /* [N,3] shaded view */
  float* rgb_surf;        /* [N,3] surface colour */
  /* optional (NULL = not wanted): */
  float* ray0; float* ray_dir; float* far_; float* depth; float* grad;   /* [N,3] [N,3] [N] [N] [N,4] (xyz; w = 0) */
  void* workspace; size_t workspace_bytes;
} nnb_geometry_args;
size_t nnb_geometry_frame_workspace_bytes(int32_t N, int32_t n_steps, int32_t hidden_dim);   /* 0 on bad sizes or an unsupported width */
int nnb_geometry_frame(const nnb_geometry_args* a, void* stream);
/* nnb_geometry_frame on a->engine: NNB_ENGINE_TC (exactly nnb_geometry_frame) or NNB_ENGINE_SIMT, the exact-fp32 engine; any other
 * engine is rejected (rc -4), and the other checks and codes are nnb_geometry_frame's.  nnb_geometry_frame keeps its contract (tensor
 * cores only).  No version bump: the symbols mark the capability.  nnb_geometry_frame_workspace_bytes_engine: the workspace on `engine`
 * (nnb_geometry_frame_workspace_bytes is this on NNB_ENGINE_TC); 0 on bad sizes, an unsupported width or an engine without the frame.
 * On NNB_ENGINE_SIMT the same contract and flags hold with every field query on the exact engine: the march is nnb_ray_march_engine on
 * NNB_ENGINE_SIMT; grad is the negated g_pts of nnb_field_fwd + nnb_field_bwd on NNB_ENGINE_SIMT
 * with NNB_RAW_DENSITY, no view directions and the cotangent (0, 0, 0, 1) (OfficialStaticNerf.gradient on the default engine); rgb_surf
 * is the rgb of nnb_field_fwd on NNB_ENGINE_SIMT at (p, -dir).  The stage bit-equality and pixel independence above hold with those
 * calls.  The normals and colours of the compacted rows run in passes of at most 32 768 rows, so the fp32 stash of the chain does not grow
 * with N.  Workspace, each section 256-byte aligned: hit count | ray0, dir, far, depth | surface points, view directions, pixel indices,
 * normal cotangents (16 N), normals (16 Npad, Npad = N rounded up to 64), colours (16 N) | the exact march's workspace | one pass's
 * records and fp32 stash.  At N = 1080 x 1920, n_steps = 512, D = 256: 672 993 792 bytes (0.67 GB). */
int nnb_geometry_frame_engine(const nnb_geometry_args* a, void* stream);
size_t nnb_geometry_frame_workspace_bytes_engine(int32_t N, int32_t n_steps, int32_t hidden_dim, int32_t engine);

/* The volumetric view of a whole frame (or any N rays) in one stream-ordered call on the tensor-core engine, with compositing fused into
 * the field's forward: what nnb_render_fwd does without NNB_STASH, in a workspace that does not grow with S, and optionally with early ray
 * termination.  No version bump: the symbol marks the capability.
 *   Inputs and outputs are those of nnb_render_fwd (f->fwd): rgb, depth_pred, depth_gt and mask per ray, the flags NNB_DIST_ALPHA, NNB_NDC,
 *   NNB_NORMALISE, NNB_USE_DIR, NNB_WHITE_BG, NNB_EVAL, NNB_SOFTPLUS and NNB_SHIFT_FIRST, ray_idx / pixels and depth / depth_map as there.
 *   Chunk rule: the rays advance in rounds of 32 samples; round k evaluates samples 32 k .. 32 k + 31 of every ray still live and
 *   composites them as composite_fwd's chunk k does.  A ray stops after the first chunk that leaves its transmittance (the product of
 *   1 - alpha_j + 1e-6 over its samples so far) below t_min, or after its last chunk.  t_min = 0 never stops a ray.
 *   n_eval [N] (optional): samples evaluated per ray (S when the ray was not stopped); t_final [N] (optional): its transmittance after
 *   the last evaluated sample.
 * Bit-equality: at t_min = 0 every output is bit-identical to nnb_render_fwd on NNB_ENGINE_TC with the same arguments (the tensor-core
 *   field result of a sample does not depend on its tile or row, and the terms of a ray are summed in composite_fwd's order).  For any
 *   t_min, a ray with n_eval == S has exactly the bits of the t_min = 0 call.  A ray's outputs depend on that ray alone, so they are the
 *   same bits on every run and for any split of the rays into calls.
 * Error bound for t_min > 0: with eps = 1e-6, T_{j+1} = T_j (1 - alpha_j + eps), so the weight a stopped ray drops, sum_{j >= n_eval}
 *   alpha_j T_j, is at most t_final (1 + eps S (1 + eps)^S) < 1.002 t_final for S <= 1024.  rgb and the accumulated weight move by at
 *   most that (plus rounding); with NNB_WHITE_BG rgb by at most twice that; depth_pred by at most that times far_ (1 with NNB_NDC),
 *   divided by the ray's norm under NNB_EVAL | NNB_NORMALISE.
 * Errors, with nothing launched (the codes of nnb_render_fwd / nnb_ray_march for the same faults): f == NULL (rc -1); an engine other than
 *   NNB_ENGINE_TC (-4); an undefined flag bit (-7); NNB_STASH, NNB_HVP, NNB_OCC_ONLY or NNB_RAW_DENSITY (-6); an unsupported width (-8);
 *   N <= 0 or S outside 2..1024 (-2); S in 2..15 (-4, the tensor-core engine's limit); a non-NULL noise, z_vals, alpha, pts or dirs (-6);
 *   t_min negative or NaN (-2); a NULL weights / c2w / cam / output, no ray_idx or pixels, no depth or depth_map, or n_eval / t_final
 *   not 4-byte aligned (-3); a workspace smaller than nnb_render_frame_workspace_bytes(N, S, hidden_dim) or not 256-byte aligned (-5).
 * Workspace, each section 256-byte aligned: round counters (256 bytes) | carry, chunks per ray (4 N bytes each) | per-ray lane partials of
 *   the weighted colour, depth and weight (640 N bytes) | two ray lists (4 N bytes each) | the forward weight image (2 359 296 bytes at
 *   D = 256).  It does not depend on S: at N = 1080 x 1920, D = 256, 1 362 641 152 bytes (1.36 GB), where nnb_render_fwd needs 32 N S
 *   bytes of sample records (8.5 GB at S = 128). */
typedef struct nnb_frame_args {
  nnb_render_args fwd;   /* the inputs and outputs of nnb_render_fwd; the workspace is sized by nnb_render_frame_workspace_bytes */
  float t_min;           /* a ray stops after the first 32-sample chunk that leaves its transmittance below t_min; 0 = never */
  int32_t* n_eval;       /* optional [N]: samples evaluated per ray (S when the ray was not stopped)                          */
  float* t_final;        /* optional [N]: transmittance after the last evaluated sample                                        */
} nnb_frame_args;
size_t nnb_render_frame_workspace_bytes(int32_t N, int32_t S, int32_t hidden_dim);   /* 0 on bad sizes or an unsupported width */
int nnb_render_frame(const nnb_frame_args* f, void* stream);

/* nnb_render_frame on f->fwd.engine.  NNB_ENGINE_TC is exactly nnb_render_frame.  NNB_ENGINE_SIMT renders the frame on the exact-fp32
 * engine with the same chunk rule, outputs, flags and early ray termination, at any S from 2 to 1024: a 64-row tile holds 64 / R
 * ray-chunks of R = min(S, 32) rows, so a ray with fewer than 32 samples takes only its own rows.  No version bump: the symbols mark the
 * capability.
 * On NNB_ENGINE_SIMT:
 *   Bit-equality: at t_min = 0 every output is bit-identical to nnb_render_fwd on NNB_ENGINE_SIMT without NNB_STASH (an exact-engine
 *   sample result does not depend on its tile or row, and the lane terms of a ray are summed in composite_fwd's order).  For any t_min, a
 *   ray with n_eval == S has exactly the bits of the t_min = 0 call, and a ray's outputs depend on that ray alone.
 *   Error bound for t_min > 0: the bound stated above for the tensor-core frame, unchanged.  n_eval is a multiple of 32, or S.
 * Errors: those of nnb_render_frame in the same order, except that an engine other than NNB_ENGINE_TC and NNB_ENGINE_SIMT is the -4, S in
 *   2..15 is accepted on NNB_ENGINE_SIMT, and the workspace is sized by nnb_render_frame_workspace_bytes_engine.
 * Workspace: nnb_render_frame_workspace_bytes_engine(N, S, hidden_dim, engine) is nnb_render_frame_workspace_bytes on NNB_ENGINE_TC; on
 *   NNB_ENGINE_SIMT it is that layout without the weight image, 1 360 281 856 bytes at N = 1080 x 1920 for every width and every S, where
 *   nnb_render_fwd needs 32 N S bytes of sample records.  0 on bad sizes, an unsupported width or another engine. */
int nnb_render_frame_engine(const nnb_frame_args* f, void* stream);
size_t nnb_render_frame_workspace_bytes_engine(int32_t N, int32_t S, int32_t hidden_dim, int32_t engine);

/* The differentiable frame on the tensor-core engine: what nnb_render_fwd (NNB_STASH) + nnb_render_bwd compute, at t_min = 0 and without
 * jitter, in a workspace whose only part that grows with S is one float per ray and 32-sample chunk.  No version bump: the symbols mark
 * the capability.
 *   b->fwd: the inputs of nnb_render_frame with its flags (NNB_STASH is rejected: nothing is kept between calls), engine NNB_ENGINE_TC,
 *   the workspace sized by nnb_render_frame_bwd_workspace_bytes.  The call runs the forward again and writes rgb, depth_pred, depth_gt and
 *   mask: bit-identical to nnb_render_fwd on NNB_ENGINE_TC with the same arguments.  The gradient fields of b are those of
 *   nnb_render_bwd, with its rules: g_weights (NULL: no MLP gradient), g_c2w, g_cam, g_scale_shift ACCUMULATED, g_depth overwritten.
 * Method: the forward stores each ray's transmittance after every chunk but the last.  Then, for each chunk from the last to the first,
 *   the chunk of every ray is evaluated again with a training stash of 32 N rows, its compositing adjoint runs with the suffix of the
 *   later chunks carried in, then the data-gradient chain and the weight-gradient stage of nnb_render_bwd, whose reduce adds the
 *   chunk's dW / db into g_weights.  The chunks' point and direction adjoints are summed per ray, chunk by chunk, and the pose adjoint
 *   follows as in nnb_render_bwd.
 * Reproducible: every sum runs in a fixed order (no float atomics but the one add per element of g_c2w, g_cam and g_scale_shift), so the
 *   same inputs give the same bits on every run, whatever the workspace held.  Against nnb_render_fwd + nnb_render_bwd the gradients
 *   differ in the order of their sums only (the weight gradients are summed chunk by chunk, the ray sums from the last chunk).
 * Errors, with nothing launched: b == NULL (rc -1); an engine other than NNB_ENGINE_TC (-4); then nnb_render_frame's checks and codes
 *   without t_min, n_eval and t_final; a NULL g_rgb or g_c2w (-3); a workspace smaller than nnb_render_frame_bwd_workspace_bytes(N, S,
 *   hidden_dim) or not 256-byte aligned (-5).
 * Workspace, each section 256-byte aligned: nnb_render_frame's workspace | the transmittance checkpoints (4 N (ceil(S / 32) - 1) bytes) |
 *   suffix carries (4 N) | per-ray lane partials of the pose adjoint (1152 N) | nnb_workspace_bytes_dim(N, 32, NNB_STASH, NNB_ENGINE_TC,
 *   hidden_dim) without its weight images (the chunk stash of 32 N rows) | the transposed weight image.  About 650 KB per ray at D = 256.
 *   nnb_render_frame_bwd_workspace_bytes: 0 on bad sizes (N <= 0, S outside 16..1024) or an unsupported width. */
size_t nnb_render_frame_bwd_workspace_bytes(int32_t N, int32_t S, int32_t hidden_dim);
int nnb_render_frame_bwd(const nnb_render_bwd_args* b, void* stream);

/* nnb_render_frame_bwd as a forward / backward pair for training, with jitter: the forward's outputs feed the loss, and the backward starts
 * from the checkpoints the forward left, so the field is evaluated twice per step, not three times.  Both calls use one workspace sized
 * by nnb_render_frame_bwd_workspace_bytes(N, S, hidden_dim), in its layout.  No version bump: the symbols mark the capability.
 * nnb_render_frame_train_fwd(a): a as b->fwd of nnb_render_frame_bwd, and noise is accepted ([N][S] jitter in [0, 1), read as
 *   nnb_render_fwd reads it; ignored under NNB_NDC).  Writes rgb, depth_pred, depth_gt and mask, bit-identical to nnb_render_fwd on
 *   NNB_ENGINE_TC with the same arguments (noise included), and leaves the forward weight image and the per-chunk transmittance
 *   checkpoints in the workspace.
 * nnb_render_frame_train_bwd(b): b->fwd must be the train_fwd call's arguments, the same pointers with unchanged contents (weights, c2w,
 *   cam, ray_idx, depth_map / depth, scale, shift, noise), and its workspace as that call left it, on the same stream.  Runs the reverse
 *   half of nnb_render_frame_bwd only (the transposed weight image, the reverse rounds, the per-ray pose adjoint and its reduction); the
 *   forward outputs are not written.  The gradient fields and their accumulate / overwrite rules are nnb_render_frame_bwd's.  Its results
 *   are defined only after a train_fwd into that workspace.  Of what train_fwd wrote it reads the forward weight image and the
 *   checkpoints, which are data, never an index or a counter: a missing forward gives wrong numbers, not an access outside the workspace.
 *   Without noise, train_fwd + train_bwd give nnb_render_frame_bwd's outputs and gradients bit for bit.
 * Neither call synchronises, reads anything back to the host or allocates, so both can be captured in a CUDA graph once an eager call of
 * the same width has run the library's one-time set-up.
 * Errors, with nothing launched: a == NULL / b == NULL (rc -1); then nnb_render_frame_bwd's checks and codes in its order, except that
 *   noise is accepted (z_vals, alpha, pts and dirs stay -6, as do NNB_STASH, NNB_HVP, NNB_OCC_ONLY and NNB_RAW_DENSITY); the NULL g_rgb
 *   or g_c2w check (-3) applies to train_bwd only.  nnb_render_frame_bwd, nnb_render_frame and nnb_render_frame_engine keep rejecting
 *   noise (-6). */
int nnb_render_frame_train_fwd(const nnb_render_args* a, void* stream);
int nnb_render_frame_train_bwd(const nnb_render_bwd_args* b, void* stream);

/* The training pair with early ray termination, on the tensor-core engine.  No version bump: the symbols mark the capability.
 * nnb_render_frame_train_fwd_tmin(f): f->fwd as nnb_render_frame_train_fwd's argument (noise accepted), plus f->t_min and the optional
 *   f->n_eval / f->t_final of nnb_render_frame.  Ray n evaluates chunks 0 .. c_n - 1 under nnb_render_frame's stop rule (it stops after
 *   the first chunk that leaves its transmittance below t_min, or after the last chunk).  Without noise, rgb, depth_pred, depth_gt, mask,
 *   n_eval and t_final are bit-identical to nnb_render_frame at the same t_min; with noise, a ray with n_eval == S has the bits of
 *   nnb_render_frame_train_fwd, and a stopped ray keeps nnb_render_frame's bound on the weight it dropped (below 1.002 t_final).  At
 *   t_min = 0 every output is nnb_render_frame_train_fwd's.  Leaves the weight image, the checkpoints and the chunk counts c_n in the
 *   workspace.
 * nnb_render_frame_train_bwd_tmin(b): after that call, with nnb_render_frame_train_bwd's rules for b and the workspace.  The gradients are
 *   the exact gradients of the truncated outputs with every c_n held constant (the stop decision is piecewise constant): reverse round k
 *   visits only the rays with c_n > k, and a ray's suffix carry into composite_chunk_bwd is 0 at its own last chunk.  Before round k the
 *   list {n : c_n > k} is built in increasing n by a block scan into the forward's first ray list and round counter (free once the
 *   forward has ended), and the data-gradient and weight-gradient kernels take their row count, 32 per listed ray, from the device.  So
 *   both calls can be captured in a CUDA graph and replayed when the stop pattern changes.  At t_min = 0 every list is 0 .. N - 1, and
 *   the outputs and gradients are nnb_render_frame_train_bwd's bit for bit, after either forward.
 *   Every c_n read is clamped to 1..C (C = ceil(S / 32)) and every device count to 0..N: a backward without its forward gives wrong
 *   numbers, never an access outside the workspace.  Every sum runs in a fixed order, so the same inputs give the same bits whatever the
 *   workspace held.  Neither call synchronises, reads back or allocates.
 * Workspace: nnb_render_frame_bwd_workspace_bytes(N, S, hidden_dim), in its layout; nothing is added.
 * Errors, with nothing launched: NULL args (rc -1); an engine other than NNB_ENGINE_TC (-4, also when nnb_render_frame_bwd_engine would
 *   take it); then nnb_render_frame_train_fwd / _bwd's checks and codes in their order, with, on the forward, a negative or NaN t_min (-2)
 *   after the flag and size checks and misaligned n_eval / t_final (-3) after the output pointers, as in nnb_render_frame. */
int nnb_render_frame_train_fwd_tmin(const nnb_frame_args* f, void* stream);
int nnb_render_frame_train_bwd_tmin(const nnb_render_bwd_args* b, void* stream);

/* Training with early ray termination on the per-sample stash, on the tensor-core engine: each sample is evaluated once, and the backward
 * runs one weight-gradient stage over the rows the forward evaluated.  It trades the memory of nnb_render_frame_train_fwd_tmin's pair
 * (the stash path's worst case here) for time.  No version bump: the symbols mark the capability.
 * nnb_render_fwd_tmin(f): f->fwd as nnb_render_frame_train_fwd_tmin's (nnb_render_fwd's training arguments without NNB_STASH, which is
 *   implied; noise accepted), f->t_min, and the optional f->n_eval / f->t_final.  Ray n evaluates chunks 0 .. c_n - 1 under
 *   nnb_render_frame's stop rule; round k evaluates chunk k of the rays {n : c_n > k}, listed in increasing n by a block scan, with the
 *   training stash, and composites them with nnb_render_frame's statements.  rgb, depth_pred, depth_gt, mask and n_eval are
 *   nnb_render_frame_train_fwd_tmin's bits at the same t_min, noise or not (t_final is formed by the same statements); at t_min = 0 the
 *   outputs are nnb_render_fwd's (NNB_STASH).
 *   Every round's rows go into one packed stash: round k's start at R_k, the rows of the rounds before padded to the 128-row tile, formed
 *   on the device from the rounds' counts.  The workspace keeps the stash, the chunk counts, the lists and the checkpoints.
 * nnb_render_bwd_tmin(b): after that call, with nnb_render_bwd's cotangents and outputs (g_weights may be NULL: pose, camera, depth and
 *   scale-shift gradients only).  The gradients are the exact gradients of the truncated render with every c_n held constant, the
 *   definition of nnb_render_frame_train_bwd_tmin: the compositing adjoint of ray n runs from its chunk c_n - 1, with a zero suffix there,
 *   to chunk 0; the data-gradient chain runs on the packed rows and the weight-gradient stage once over them, with the row count read on
 *   the device.  The pose, camera, depth and scale-shift gradients are nnb_render_frame_train_bwd_tmin's bits; the MLP gradients differ
 *   from it in the order of their sums.  Every c_n read is clamped to 1..C (C = ceil(S / 32)) and every device count to 0..N: a backward
 *   without its forward gives wrong numbers, never an access outside the workspace.  Every sum runs in a fixed order, padding rows get a
 *   zero cotangent, and no count is read back, so the same inputs give the same bits whatever the workspace held, and both calls can be
 *   captured in a CUDA graph and replayed when the stop pattern changes.  Neither call synchronises or allocates.
 * nnb_render_tmin_workspace_bytes(N, S, hidden_dim): the workspace of both calls, for every ray running every chunk: the training stash of
 *   C 128 ceil(N / 4) rows (at least nnb_workspace_bytes_dim(N, S, NNB_STASH, NNB_ENGINE_TC, hidden_dim)) and the per-ray state.  0 for
 *   N <= 0, S outside 16..1024 or an unsupported width.
 * Errors, with nothing launched: NULL args (rc -1); an engine other than NNB_ENGINE_TC (-4); then the checks and codes of
 *   nnb_render_frame_train_fwd_tmin / _bwd_tmin in their order (sizes -2, with S below 16 -4 as on that pair; a negative or NaN t_min -2;
 *   misaligned n_eval / t_final -3; non-NULL z_vals, alpha, pts or dirs -6; NNB_STASH -6), with this workspace's size (-5). */
size_t nnb_render_tmin_workspace_bytes(int32_t N, int32_t S, int32_t hidden_dim);
int nnb_render_fwd_tmin(const nnb_frame_args* f, void* stream);
int nnb_render_bwd_tmin(const nnb_render_bwd_args* b, void* stream);

/* nnb_render_fwd_tmin, nnb_render_bwd_tmin and nnb_render_tmin_workspace_bytes on fwd.engine (on `engine` for the size).  NNB_ENGINE_TC
 * is exactly the call without the suffix (its checks, codes, bits and workspace).  NNB_ENGINE_SIMT runs the same method on the exact-fp32
 * engine at any S from 2 to 1024, with every flag, density head, width, NDC / uniform setting, eval mode and jitter the tensor-core pair
 * accepts.  Its packed stash holds R = min(S, 32) rows per listed ray and round, each round padded to the 64-row tile: round k's rows start
 * at base_k, formed on the device from the rounds' counts, and row base_k + R slot + j is sample 32 k + j of the round's ray `slot`.  At
 * S <= 32 (one round) the rows are nnb_render_fwd's, in its order: outputs and gradients are nnb_render_fwd / nnb_render_bwd's (NNB_STASH,
 * NNB_ENGINE_SIMT) bits, and n_eval is S.  At t_min = 0 the outputs are nnb_render_fwd's at every S, and the pose, camera and scale-shift
 * gradients are nnb_render_frame_train_bwd_engine's on NNB_ENGINE_SIMT.  The compositing adjoint takes composite_bwd's fused d L / d alpha.
 * The data-gradient chain and one weight-gradient stage run on the packed rows, with the row count and the stage's split count read on the
 * device (at S <= 32: nnb_render_bwd's M and splits).  No count is read back, no float atomic is used, every chunk count read is clamped to
 * 1..C and every device count to 0..N, as on the tensor-core pair.
 * Workspace: nnb_render_tmin_workspace_bytes_engine(N, S, hidden_dim, NNB_ENGINE_SIMT): the packed stash for every ray running every chunk
 * (at least nnb_workspace_bytes_dim(N, S, NNB_STASH, NNB_ENGINE_SIMT, hidden_dim)), then carry, chunk counts, lane partials, checkpoints,
 * lists, counts and ray lane partials; no weight images.  0 for N <= 0, S outside 2..1024 (16..1024 on NNB_ENGINE_TC), an unsupported
 * width or an unknown engine.
 * Errors, with nothing launched: NULL args (-1); an engine other than NNB_ENGINE_TC and NNB_ENGINE_SIMT (-4); then the checks and codes of
 * nnb_render_fwd_tmin / _bwd_tmin in their order (flags, width, sizes -2, per-sample outputs -6, t_min -2, pointers -3, workspace -5).
 * g_weights may be NULL (pose only). */
size_t nnb_render_tmin_workspace_bytes_engine(int32_t N, int32_t S, int32_t hidden_dim, int32_t engine);
int nnb_render_fwd_tmin_engine(const nnb_frame_args* f, void* stream);
int nnb_render_bwd_tmin_engine(const nnb_render_bwd_args* b, void* stream);

/* nnb_render_frame_bwd, nnb_render_frame_train_fwd and nnb_render_frame_train_bwd on fwd.engine.  NNB_ENGINE_TC is exactly the call
 * without the suffix (its checks, codes, bits and workspace).  NNB_ENGINE_SIMT runs the same method on the exact-fp32 engine at any S from
 * 2 to 1024, with a chunk stash that packs R = min(S, 32) rows per ray (row R n + j is sample 32 k + j of ray n), so a round at S < 32
 * evaluates N S rows.  The four calls without the suffix keep their contracts.  No version bump: the symbols mark the capability.
 * On NNB_ENGINE_SIMT:
 *   Forward bits: the outputs of nnb_render_frame_bwd_engine and nnb_render_frame_train_fwd_engine are bit-identical to nnb_render_fwd on
 *   NNB_ENGINE_SIMT with the same arguments (noise included, for the train pair).
 *   Gradients at S <= 32 (one chunk): the chunk stash holds nnb_render_fwd's rows in its order and the weight-gradient stage splits them
 *   as nnb_render_bwd does, so the gradients are those of nnb_render_fwd (NNB_STASH) + nnb_render_bwd on NNB_ENGINE_SIMT, bit for bit.
 *   At S > 32 they differ from them in the order of their sums only (weight gradients chunk by chunk, the ray sums from the last chunk);
 *   every dW / db, g_c2w and the other pose outputs stay within 1e-4 of the largest magnitude of their tensor.
 *   Without noise, train_fwd_engine + train_bwd_engine give nnb_render_frame_bwd_engine's outputs and gradients bit for bit.  Every sum
 *   runs in a fixed order, so the same inputs give the same bits whatever the workspace held.  Neither call of the pair synchronises,
 *   reads back or allocates.  Of what train_fwd_engine wrote, train_bwd_engine reads the checkpoints only.
 * Errors, with nothing launched: NULL args (rc -1); an engine other than NNB_ENGINE_TC and NNB_ENGINE_SIMT (-4); then the checks and codes
 *   of the call without the suffix in its order, except that S in 2..15 is accepted on NNB_ENGINE_SIMT and the workspace is sized by
 *   nnb_render_frame_bwd_workspace_bytes_engine.  noise is accepted by the train pair only (-6 on nnb_render_frame_bwd_engine).
 * Workspace: nnb_render_frame_bwd_workspace_bytes_engine(N, S, hidden_dim, engine) is nnb_render_frame_bwd_workspace_bytes on
 *   NNB_ENGINE_TC.  On NNB_ENGINE_SIMT it is that layout without weight images and with the chunk stash nnb_workspace_bytes_dim(N, R,
 *   NNB_STASH, NNB_ENGINE_SIMT, hidden_dim): 2.66 GB at N = 4096, D = 256 for every S >= 32, where nnb_render_fwd's stash needs about
 *   19.9 KB per sample (83.7 GB at S = 1024).  At S <= 32 the chunk stash is the stash path's, so the workspace is about 1.8 KB per ray
 *   larger than nnb_workspace_bytes_dim(N, S, NNB_STASH, NNB_ENGINE_SIMT, hidden_dim).  0 on bad sizes (N <= 0, S outside 2..1024 on
 *   NNB_ENGINE_SIMT), an unsupported width or another engine. */
size_t nnb_render_frame_bwd_workspace_bytes_engine(int32_t N, int32_t S, int32_t hidden_dim, int32_t engine);
int nnb_render_frame_bwd_engine(const nnb_render_bwd_args* b, void* stream);
int nnb_render_frame_train_fwd_engine(const nnb_render_args* a, void* stream);
int nnb_render_frame_train_bwd_engine(const nnb_render_bwd_args* b, void* stream);

/* LearnPose.forward (model/poses.py:23-31): c2w = [Exp(r[id]) t[id]; 0 1] @ init_c2w[id] */
int nnb_pose_fwd(const float* r, const float* t, const float* init_c2w /*[V,16] or NULL*/, int32_t cam_id,
                 float* c2w /*[16]*/, void* stream);
/* adjoint: g_r[cam_id], g_t[cam_id] += ... ; g_r/g_t are [V,3] (either may be NULL) */
int nnb_pose_bwd(const float* r, const float* t, const float* init_c2w, int32_t cam_id, const float* g_c2w,
                 float* g_r, float* g_t, void* stream);

/* CUDA-graph friendly variants: per-step host scalars (camera index, Adam step, learning rate, frame pointer) are read
 * from DEVICE memory so one captured graph of the whole training step can be replayed for every frame. */
int nnb_pose_fwd_dev(const float* r, const float* t, const float* init_c2w, const int32_t* cam_id_dev, float* c2w, void* stream);
int nnb_pose_bwd_dev(const float* r, const float* t, const float* init_c2w, const int32_t* cam_id_dev, const float* g_c2w, float* g_r,
                     float* g_t, void* stream);
/* Learn_Distortion.forward (model/distortions.py:19-27): out2 = {scale_eff, shift} of view *cam_id_dev; and its adjoint */
int nnb_distortion_fwd_dev(const float* scales, const float* shifts, int32_t V, const int32_t* cam_id_dev, int32_t fix_scaleN, float* out2,
                           void* stream);
int nnb_distortion_bwd_dev(const float* scales, int32_t V, const int32_t* cam_id_dev, int32_t fix_scaleN, const float* g_scale_shift,
                           float* g_scales, float* g_shifts, void* stream);
int nnb_adam_step_dev(float* p, const float* g, float* m, float* v, int64_t n, const int32_t* step_dev, const float* lr_dev, float beta1,
                      float beta2, float eps, void* stream);
int nnb_counter_incr(int32_t* counters, int32_t n, void* stream);
/* N distinct pixel ids uniform in [0,HW) from 2N uniforms u in [0,1): same distribution as torch.randperm(HW)[:N]
 * (model/training.py:257) without sorting HW keys.  0 < N <= min(HW/2, 8192). */
int nnb_sample_pixels(const float* u2n, int32_t HW, int32_t N, int64_t* out, void* stream);
/* w_dev (optional): device {w_rgb, w_depth} overriding the host weights -- the annealed weights of training.py:208-217 change per
 * epoch without re-capturing the graph */
int nnb_loss_rgb_depth_indirect(const float* rgb, const float* const* img_pp /* device pointer to the frame pointer */, const int64_t* ray_idx,
                                int32_t HW, const float* depth_pred, const float* depth_gt, const uint8_t* mask, int32_t N, float w_rgb,
                                float w_depth, int32_t rgb_l2, float grad_scale, float* out_losses, float* g_rgb, float* g_depth_pred,
                                float* g_depth_gt, const float* w_dev, void* stream);

/* Loss.forward photometric + depth-L1 terms (model/losses.py:27-32,59-61,192,196-202) fused with
 * the cotangent seeds of nnb_render_bwd.  rgb_gt is either explicit [N,3] or gathered from a planar
 * image [3,H*W] at ray_idx (training.py:258-259).  out_losses = {loss, loss_rgb, loss_depth, l2_mean}. */
int nnb_loss_rgb_depth(const float* rgb, const float* rgb_gt, const float* img, const int64_t* ray_idx, int32_t HW,
                       const float* depth_pred, const float* depth_gt, const uint8_t* mask, int32_t N,
                       float w_rgb, float w_depth, int32_t rgb_l2, float grad_scale, float* out_losses /*[4]*/,
                       float* g_rgb, float* g_depth_pred, float* g_depth_gt, void* stream);

/* Loss.get_pc_loss 'dense' (model/losses.py:114-148): symmetric mean nearest-neighbour distance (brute force, argmin ties ->
 * first index like torch.argmin).  X [P,3], Y [Q,3]; keys: scratch of nnb_chamfer_workspace_bytes(P, Q) bytes when the adjoints
 * are requested, [P+Q] 64-bit otherwise; idx_xy [P], idx_yx [Q] optional int32 nearest-neighbour outputs (both or neither);
 * loss [1] (+=); optional adjoints gX, gY (+=, both or neither).
 * Reproducible: the same inputs give the same bits on every run.  The loss is summed from block partials in block order; each
 * adjoint element collects the terms of the pairs whose nearest neighbour it is in 64-bit fixed point (integer adds, so their order
 * does not matter) and rounds that sum to float once.  Each term is first rounded to a quantum of 2^-F |weight| / n, n the size of
 * its cloud and F = 62 - bits(n) (2^-48 at n = 16 128): far below float resolution for the large terms, coarser than a float sum
 * for components many orders of magnitude below |weight| / n.  A component that receives a non-finite term comes out NaN.
 * loss, gX and gY get plain (non-atomic) adds: no other work may write them while the call runs. */
int nnb_chamfer(const float* X, int32_t P, const float* Y, int32_t Q, uint64_t* keys, int32_t* idx_xy, int32_t* idx_yx,
                float* loss, float weight, float* gX, float* gY, void* stream);
/* bytes of `keys` scratch nnb_chamfer needs with adjoints (search keys, fixed-point group sums); 0 on bad sizes.  The call cannot
 * check the size it is given: a smaller buffer is written out of bounds. */
size_t nnb_chamfer_workspace_bytes(int32_t P, int32_t Q);

/* Reference-image stage of Trainer.compute_loss (model/training.py:280-365): point-cloud (dense chamfer) + warped-RGB terms
 * between the current view and one reference view, forward AND adjoint in one call.
 *   img_* (3,H,W) planar fp32; dpt_* (h_d,w_d) raw DPT maps; c2w_* (4,4) row-major; dist_* = {effective scale, shift}
 *   (Learn_Distortion.forward) -- all device pointers.  flags: 1 = scale_pcs, 2 = detach_rgbs_scale, 4 = shift_first,
 *   8 = with_ssim (warped-RGB loss 0.15 L1 + 0.85 SSIM, losses.py:150-157; needs nnb_refstage_workspace_bytes_flags),
 *   16 = gradients into the reference view too (training.detach_ref_img = False; needs g_c2w_ref and g_dist_ref).
 *   losses[2] = {loss_pc, loss_rgb_s}; g_c2w[16] / g_dist[2] / g_kxy[2] ACCUMULATE grad_scale * d(w_pc*loss_pc + w_rgb_s*loss_rgb_s) /
 *   d(c2w_cur, dist_cur, (kx, ky)); loss_total (optional) += the weighted sum.
 * CUDA-graph replay: per-step values may come from device memory instead of the host fields -- img_pp (device array of the two
 * frame pointers {cur, ref}, replaces img_cur / img_ref), cam (device camera_mat [16]: kx = cam[0], ky = cam[5]), cam_idx_dev +
 * num_cams (is_last = *cam_idx_dev == num_cams - 1), weights_dev ({w_pc, w_rgb_s}).
 * Reproducible: every sum over the points runs in a fixed order (per-block partials in the workspace, added in block order), so the
 * same inputs give the same bits on every run.  losses is overwritten.  g_c2w, g_dist, g_kxy, loss_total, g_c2w_ref and g_dist_ref
 * each get one atomic add per element from one thread: other work may add into the same buffers concurrently (the sums stay
 * correct), but the bits are reproducible only when that work is ordered before or after the call (same stream, or an event). */
typedef struct nnb_refstage_args {
  const float* img_cur; const float* img_ref; const float* dpt_cur; const float* dpt_ref;
  const float* c2w_cur; const float* c2w_ref; const float* dist_cur; const float* dist_ref;
  int32_t H, W, h_d, w_d, pc_ratio, is_last;
  uint32_t flags;
  float kx, ky, nearest_limit, w_pc, w_rgb_s;
  float* losses; float* g_c2w; float* g_dist;
  void* workspace; size_t workspace_bytes;       /* >= nnb_refstage_workspace_bytes(h_d, w_d, pc_ratio) */
  /* optional (NULL / 0 = unused) */
  const float* const* img_pp; const float* cam; const int32_t* cam_idx_dev; int32_t num_cams; const float* weights_dev;
  float* g_kxy; float* loss_total; float grad_scale;   /* grad_scale 0 is read as 1 */
  /* flag 16: ACCUMULATE grad_scale * d(...) / d(c2w_ref) (rows 0-2 of the 4x4) and d / d(dist_ref) */
  float* g_c2w_ref; float* g_dist_ref;
} nnb_refstage_args;
size_t nnb_refstage_workspace_bytes(int32_t h_d, int32_t w_d, int32_t pc_ratio);          /* flags 1 | 2 | 4 */
size_t nnb_refstage_workspace_bytes_flags(int32_t h_d, int32_t w_d, int32_t pc_ratio, uint32_t flags);
int nnb_refstage(const nnb_refstage_args* args, void* stream);

/* ---- data-parallel exchange over NVLink peer memory (new component, SURVEY.md 8(e)) --------------------------------------
 * The reference has no distributed code; the design shards a step's rays (or views) over the GPUs of one box and needs ONE
 * sum of the flat gradient buffer per step.  nnb_allreduce_adam does that sum with P2P loads from every rank's buffer and applies
 * the three torch.optim.Adam updates (train.py:58,99,117) in the same kernel; it is captured in the step's CUDA graph.
 * Buffers come from nnb_ipc_alloc (cudaMalloc + CUDA IPC handle); peers map them with nnb_ipc_open. */
#define NNB_MAX_RANKS 8
#define NNB_FLAG_PAD_BYTES 256      /* per-rank flag pad: uint32 [2][NNB_MAX_RANKS] + local counters; zero it once after allocation */
int nnb_ipc_alloc(size_t bytes, void** dev_ptr, unsigned char handle_out[64]);
int nnb_ipc_open(const unsigned char handle[64], void** peer_ptr);
int nnb_ipc_close(void* peer_ptr);
int nnb_ipc_free(void* dev_ptr);
typedef struct nnb_adam_seg {       /* one parameter tensor (or flat group) inside the gradient buffer */
  float* p; float* m; float* v;     /* parameters and Adam moments (local) */
  int64_t offset, count;            /* position of its gradient in the flat buffer */
  const float* lr_dev; const int32_t* step_dev;   /* device-resident learning rate and 1-based step (as nnb_adam_step_dev) */
  float beta1, beta2, eps;
} nnb_adam_seg;
typedef struct nnb_allreduce_adam_args {
  const float* peer_grads[NNB_MAX_RANKS];   /* every rank's flat gradient buffer (own entry = local buffer), pre-scaled by 1/world */
  uint32_t* peer_flags[NNB_MAX_RANKS];      /* every rank's flag pad (NNB_FLAG_PAD_BYTES) */
  int32_t world, rank;
  int64_t n_total;                  /* floats in the buffer (multiple of 4) */
  float* reduced_out;               /* [n_total] local copy of the summed gradient (what .grad shows) or NULL */
  nnb_adam_seg segs[8]; int32_t nsegs;
} nnb_allreduce_adam_args;
/* Sums the buffers of all ranks (rank order: bit-identical on every rank), applies Adam to every segment, writes the sum to
 * reduced_out and ZEROES the local gradient buffer for the next step.  Every rank must call it the same number of times. */
int nnb_allreduce_adam(const nnb_allreduce_adam_args* args, void* stream);

/* ---- training options of the whole-step CUDA graph ------------------------------------------------------------------------
 * Each is one single-CTA launch.  Per-step values (loss weights, parameters) are read from device memory, nothing synchronises or
 * allocates, and every sum runs in a fixed order without float atomics: the same inputs give the same bits on every run. */

/* Scale / shift invariant depth term (training.depth_loss_type = invariant; Loss.depth_loss_dpt, model/losses.py:34-57) over the rays
 * with mask[i] != 0 of the dense depth_pred / depth_gt / mask that nnb_render_fwd writes, forward and adjoint:
 *   t = lower median (sorted position (n-1)/2 of the n masked values, as torch.median), s = mean |x - t|,
 *   L = mean ((p - t_p) / s_p - (g - t_g) / s_g)^2.
 * w = *w_dev (the annealed depth weight).  w == 0: nothing is read or written.  n == 0: nothing is written.  Otherwise
 * out_losses[2] = L (overwritten) and out_losses[0] += w * L, and the seeds are ADDED (plain adds, one writer per element) on the masked
 * rays: g_depth_pred += grad_scale * w * dL/dp, g_depth_gt (NULL = not wanted: training.detach_gt_depth) += grad_scale * w * dL/dg.
 * The adjoint follows torch's autograd through every path: through the two mean absolute deviations (|x - t| has gradient
 * sign(x - t), 0 at the median itself) and through the medians.  Ties at the median: like torch.median's backward, the median's
 * gradient is split evenly over ALL masked rays whose value equals the median (+0 and -0 compare equal).  n == 1 or all masked values
 * equal gives s = 0 and NaN, as in torch.  The masked count n lives on the device only.  One CTA: meant for the N <= 8192 rays of a
 * training step; N <= NNB_INVARIANT_MAX_N. */
#define NNB_INVARIANT_MAX_N 16777216
int nnb_depth_invariant(const float* depth_pred, const float* depth_gt, const uint8_t* mask, int32_t N, const float* w_dev, float grad_scale,
                        float* out_losses /*[4]*/, float* g_depth_pred, float* g_depth_gt, void* stream);
/* LearnFocal.forward (model/intrinsics.py) as the camera matrix of the step (training.py:247-252): cam[16] = diag(fx', -fy', -1, 1)
 * with (fx', fy') = (*fx, *fy) at order 1 and their squares at order 2; fy = NULL means fx_only (fy' = fx'). */
int nnb_focal_fwd(const float* fx, const float* fy, int32_t order, float* cam, void* stream);
/* its adjoint, ADDED into *g_fx / *g_fy: d/dfx' = g_cam[0] + g_kxy[0], d/dfy' = -(g_cam[5] + g_kxy[1]), chained through the square at
 * order 2; with fy = g_fy = NULL (fx_only) both terms go to *g_fx.  g_cam[16] is nnb_render_bwd's camera-matrix gradient, g_kxy[2]
 * nnb_refstage's (NULL when the reference-image stage does not run). */
int nnb_focal_bwd(const float* fx, const float* fy, int32_t order, const float* g_cam, const float* g_kxy, float* g_fx, float* g_fy, void* stream);
/* Pose-smoothness terms (Loss.get_weight_dist_loss, model/losses.py:103-112) of the translations t[V,3], V >= 2:
 *   dist_i = |t_i - t_{i-1}| (i = 1..V-1), out2[0] = loss_dist_1st = mean dist, out2[1] = loss_dist_2nd = mean_{j=2..V-1} (dist_j - dist_{j-1})^2
 * (NaN at V = 2, torch's mean over no element).  With {w1, w2} = w_dev[0..1]: loss_total (optional) += grad_scale (w1 1st + w2 2nd),
 * g_t[V,3] (optional) += grad_scale d(w1 1st + w2 2nd)/dt (plain adds, one writer per row; a zero-length step has gradient 0, like
 * the norm's autograd).  While w1 == w2 == 0 nothing is written. */
int nnb_pose_smooth(const float* t, int32_t V, const float* w_dev, float grad_scale, float* out2, float* loss_total, float* g_t, void* stream);

/* torch.optim.Adam step (train.py:58,99,117 defaults) over one flat buffer. step_count is the
 * 1-based step; lr/betas/eps as torch. */
int nnb_adam_step(float* p, const float* g, float* m, float* v, int64_t n, int32_t step, float lr, float beta1,
                  float beta2, float eps, void* stream);

#ifdef __cplusplus
}
#endif
#endif
