// extern "C" boundary (include/nope_nerf_b200.h): argument validation, workspace carving,
// engine dispatch.  No torch types, no allocation, no synchronisation.
#include <cstdio>
#include <cstdarg>
#include <cstring>
#include <initializer_list>
#include "nnb_workspace.cuh"

cudaError_t simt_render_fwd(const nnb_render_args& a, const WsLayout& L, cudaStream_t st);
cudaError_t simt_render_bwd(const nnb_render_bwd_args& b, const WsLayout& L, cudaStream_t st);
cudaError_t simt_field_fwd(const nnb_render_args& a, const WsLayout& L, float* out_rgba, cudaStream_t st);
cudaError_t simt_field_bwd(const nnb_render_args& a, const WsLayout& L, const float* g_rgba, float* g_pts, float* g_dirs, float* g_weights,
                           cudaStream_t st);
cudaError_t simt_field_hvp(const nnb_render_args& a, const WsLayout& L, const float* u, float* g_pts, float* g_weights, cudaStream_t st);
cudaError_t simt_wgrad_stage(const nnb_render_args& a, const WsLayout& L, float* gw, cudaStream_t st);
size_t simt_ray_march_workspace(int N, int n_steps);
cudaError_t simt_ray_march(const nnb_ray_march_args& r, int D, cudaStream_t st);
size_t simt_geometry_frame_workspace(int N, int n_steps, int D);
cudaError_t simt_geometry_frame(const nnb_geometry_args& g, int D, cudaStream_t st);
size_t simt_render_frame_workspace(int N);
cudaError_t simt_render_frame(const nnb_render_args& a, float t_min, int* n_eval, float* t_final, int D, cudaStream_t st);
size_t simt_render_frame_bwd_workspace(int N, int S, int D);
cudaError_t simt_render_frame_bwd(const nnb_render_bwd_args& b, int D, cudaStream_t st);
cudaError_t simt_render_frame_train_fwd(const nnb_render_args& a, int D, cudaStream_t st);
cudaError_t simt_render_frame_train_bwd(const nnb_render_bwd_args& b, int D, cudaStream_t st);
size_t simt_render_tmin_workspace(int N, int S, int D);
cudaError_t simt_render_fwd_tmin(const nnb_frame_args& f, int D, cudaStream_t st);
cudaError_t simt_render_bwd_tmin(const nnb_render_bwd_args& b, int D, cudaStream_t st);
#ifdef NNB_WITH_TC
cudaError_t tc_render_fwd(const nnb_render_args& a, const WsLayout& L, cudaStream_t st);
cudaError_t tc_render_bwd(const nnb_render_bwd_args& b, const WsLayout& L, cudaStream_t st);
cudaError_t tc_wgrad_stage(const nnb_render_args& a, const WsLayout& L, float* gw, cudaStream_t st);
cudaError_t tc_field_fwd_points(const nnb_render_args& a, const WsLayout& L, float* out_rgba, cudaStream_t st);
size_t tc_workspace_extra(int N, int S, uint32_t flags, int D);
size_t tc_ray_march_workspace(int N, int n_steps, int D);
cudaError_t tc_ray_march(const nnb_ray_march_args& r, int D, cudaStream_t st);
size_t tc_field_vjp_workspace(int N, uint32_t flags, int D);
cudaError_t tc_field_vjp(const nnb_render_args& a, const float* g_rgba, float* out_rgba, float* g_pts, float* g_dirs, int D, cudaStream_t st);
size_t tc_field_grad_workspace(int N, uint32_t flags, int D);
cudaError_t tc_field_grad(const nnb_render_args& a, const float* g_rgba, float* out_rgba, float* g_pts, float* g_dirs, float* g_weights, int D,
                          cudaStream_t st);
size_t tc_field_hvp_workspace(int N, int D);
cudaError_t tc_field_hvp(const nnb_render_args& a, const float* u, float* g_pts, float* g_weights, int D, cudaStream_t st);
size_t tc_geometry_frame_workspace(int N, int n_steps, int D);
size_t tc_render_frame_workspace(int N, int D);
cudaError_t tc_render_frame(const nnb_render_args& a, float t_min, int* n_eval, float* t_final, int D, cudaStream_t st);
size_t tc_render_frame_bwd_workspace(int N, int S, int D);
cudaError_t tc_render_frame_bwd(const nnb_render_bwd_args& b, int D, cudaStream_t st);
cudaError_t tc_render_frame_train_fwd(const nnb_render_args& a, int D, cudaStream_t st);
cudaError_t tc_render_frame_train_bwd(const nnb_render_bwd_args& b, int D, cudaStream_t st);
cudaError_t tc_render_frame_train_fwd_tmin(const nnb_frame_args& f, int D, cudaStream_t st);
cudaError_t tc_render_frame_train_bwd_tmin(const nnb_render_bwd_args& b, int D, cudaStream_t st);
size_t tc_render_tmin_workspace(int N, int S, int D);
cudaError_t tc_render_fwd_tmin(const nnb_frame_args& f, int D, cudaStream_t st);
cudaError_t tc_render_bwd_tmin(const nnb_render_bwd_args& b, int D, cudaStream_t st);
cudaError_t tc_geometry_frame(const nnb_geometry_args& g, int D, cudaStream_t st);
bool tc_supports(int S);
#endif
cudaError_t launch_pose_fwd(const float*, const float*, const float*, int, const int*, float*, cudaStream_t);
cudaError_t launch_pose_bwd(const float*, const float*, const float*, int, const int*, const float*, float*, float*, cudaStream_t);
cudaError_t launch_distortion_fwd(const float*, const float*, int, const int*, int, float*, cudaStream_t);
cudaError_t launch_distortion_bwd(const float*, int, const int*, int, const float*, float*, float*, cudaStream_t);
cudaError_t launch_adam_dev(float*, const float*, float*, float*, int64_t, const int*, const float*, float, float, float, cudaStream_t);
cudaError_t launch_incr(int*, int, cudaStream_t);
cudaError_t launch_sample_pixels(const float*, int, int, long long*, cudaStream_t);
cudaError_t launch_loss(const float*, const float*, const float*, const float* const*, const int64_t*, int, const float*, const float*, const uint8_t*,
                        int, float, float, int, float, float*, float*, float*, float*, const float*, cudaStream_t);
cudaError_t launch_chamfer_full(const float*, int, const float*, int, void*, float*, float, const float*, float*, float*, int*, int*, cudaStream_t);
size_t chamfer_workspace_bytes(int P, int Q);
cudaError_t launch_adam(float*, const float*, float*, float*, int64_t, int, float, float, float, float, cudaStream_t);
size_t refstage_workspace_bytes(int hd, int wd, int ratio);
size_t refstage_workspace_bytes_flags(int hd, int wd, int ratio, unsigned flags);
cudaError_t launch_refstage(const nnb_refstage_args& a, cudaStream_t st);
cudaError_t launch_allreduce_adam(const nnb_allreduce_adam_args& a, cudaStream_t st);
cudaError_t launch_depth_invariant(const float*, const float*, const uint8_t*, int, const float*, float, float*, float*, float*, cudaStream_t);
cudaError_t launch_focal_fwd(const float*, const float*, int, float*, cudaStream_t);
cudaError_t launch_focal_bwd(const float*, const float*, int, const float*, const float*, float*, float*, cudaStream_t);
cudaError_t launch_pose_smooth(const float*, int, const float*, float, float*, float*, float*, cudaStream_t);

// optional profiling hook (bench.py): CUDA events recorded between the kernels of one call
static cudaEvent_t* g_prof_events = nullptr;
static int g_prof_n = 0, g_prof_i = 0;
void nnb_prof_mark(cudaStream_t st) {
  if (g_prof_events && g_prof_i < g_prof_n) cudaEventRecord(g_prof_events[g_prof_i++], st);
}

static thread_local char g_err[512] = "";
static int fail(int code, const char* fmt, ...) {
  va_list ap; va_start(ap, fmt); vsnprintf(g_err, sizeof(g_err), fmt, ap); va_end(ap);
  return code;
}
static int cuda_fail(cudaError_t e, const char* where) {
  return fail(-100 - (int)e, "%s: CUDA error %d (%s)", where, (int)e, cudaGetErrorString(e));
}

extern "C" {

const char* nnb_last_error(void) { return g_err; }
// 101: nnb_chamfer with adjoints needs nnb_chamfer_workspace_bytes(P, Q) of keys; 102: nnb_field_hvp; 103: nnb_field_fwd on NNB_ENGINE_TC;
// 104: nnb_ray_march; 105: one-call backward, undefined flag bits rejected (see the header)
int nnb_version(void) { return 105; }
int nnb_profile_events(void** events, int32_t count) {
  g_prof_events = reinterpret_cast<cudaEvent_t*>(events); g_prof_n = events ? count : 0; g_prof_i = 0;
  return 0;
}
int nnb_profile_cursor(void) { return g_prof_i; }
// test/debug aid: byte offsets of the workspace sections {rec, h0..h7, feat, hr, enc, denc, total}
int nnb_debug_layout(int32_t N, int32_t S, uint32_t flags, int32_t engine, size_t* out14) {
  if (!out14 || N <= 0 || S <= 0) return fail(-3, "nnb_debug_layout: bad arguments");
  WsLayout L = make_layout(N, S, flags, engine);
  out14[0] = L.rec;
  for (int l = 0; l < 8; ++l) out14[1 + l] = L.h[l];
  out14[9] = L.feat; out14[10] = L.hr; out14[11] = L.enc; out14[12] = L.denc; out14[13] = L.total;
  return 0;
}

// model.hidden_dim of a call: 0 means 256
static int hidden_of(int32_t hidden_dim) { return hidden_dim == 0 ? 256 : hidden_dim; }

// every rendering flag the header defines; any other bit (among them those of options removed in version 105) is an error
static constexpr uint32_t KNOWN_FLAGS = NNB_DIST_ALPHA | NNB_NDC | NNB_NORMALISE | NNB_USE_DIR | NNB_WHITE_BG | NNB_EVAL | NNB_SOFTPLUS |
                                        NNB_SHIFT_FIRST | NNB_STASH | NNB_RAW_DENSITY | NNB_HVP | NNB_OCC_ONLY;
static int check_flags(uint32_t flags) {
  if (flags & ~KNOWN_FLAGS) return fail(-7, "flags 0x%x: bits 0x%x are not defined by this library", flags, flags & ~KNOWN_FLAGS);
  return 0;
}

size_t nnb_num_params(int32_t hidden_dim) {
  const int D = hidden_of(hidden_dim);
  return nnb::dim_supported(D) ? (size_t)nnb::num_params(D) : 0;
}

size_t nnb_workspace_bytes_dim(int32_t N, int32_t S, uint32_t flags, int32_t engine, int32_t hidden_dim) {
  const int D = hidden_of(hidden_dim);
  if (N <= 0 || S <= 0 || !nnb::dim_supported(D) || (flags & ~KNOWN_FLAGS)) return 0;
  WsLayout L = make_layout(N, S, flags, engine, D);
  size_t tot = L.total;
#ifdef NNB_WITH_TC
  if (engine == NNB_ENGINE_TC) tot += tc_workspace_extra(N, S, flags, D);
#endif
  return tot;
}

size_t nnb_workspace_bytes(int32_t N, int32_t S, uint32_t flags, int32_t engine) { return nnb_workspace_bytes_dim(N, S, flags, engine, 256); }

static int check_dim(const nnb_render_args* a) {
  if (!nnb::dim_supported(hidden_of(a->hidden_dim)))
    return fail(-8, "hidden_dim %d is not supported (supported: 64, 128, 256; 0 means 256)", a->hidden_dim);
  return 0;
}

static int check_engine_ws(const nnb_render_args* a);
static int check_args(const nnb_render_args* a) {
  if (!a) return fail(-1, "null args");
  if (a->N <= 0) return fail(-2, "N must be positive (got %d)", a->N);
  if (a->S < 2 || a->S > 1024) return fail(-2, "S must be in [2,1024] (got %d)", a->S);
  if (!a->weights || !a->c2w || !a->cam) return fail(-3, "weights / c2w / cam must be non-null");
  if (!a->ray_idx && !a->pixels) return fail(-3, "need ray_idx or pixels");
  if (!a->pixels && (a->H < 2 || a->W < 2)) return fail(-3, "H,W needed to derive pixels from ray_idx");
  if (!a->depth && !(a->depth_map && a->ray_idx && a->h_d > 0 && a->w_d > 0 && a->H > 0 && a->W > 0))
    return fail(-3, "need depth[N] or (depth_map,h_d,w_d,H,W,ray_idx)");
  if (!a->rgb || !a->depth_pred || !a->depth_gt || !a->mask) return fail(-3, "output pointers must be non-null");
  return check_engine_ws(a);
}

// flags, engine, width, the engine's S range, and the workspace's size and alignment
static int check_engine_ws(const nnb_render_args* a) {
  if (int rc = check_flags(a->flags)) return rc;
  if (a->engine != NNB_ENGINE_SIMT && a->engine != NNB_ENGINE_TC) return fail(-4, "unknown engine %d", a->engine);
  if (int rc = check_dim(a)) return rc;
#ifndef NNB_WITH_TC
  if (a->engine == NNB_ENGINE_TC) return fail(-4, "library built without the tensor-core engine");
#else
  if (a->engine == NNB_ENGINE_TC && !tc_supports(a->S))
    return fail(-4, "tensor-core engine needs S in [16,1024] (got %d); use NNB_ENGINE_SIMT", a->S);
#endif
  size_t need = nnb_workspace_bytes_dim(a->N, a->S, a->flags, a->engine, a->hidden_dim);
  if (!a->workspace || a->workspace_bytes < need)
    return fail(-5, "workspace too small: have %zu need %zu", a->workspace_bytes, need);
  if ((reinterpret_cast<uintptr_t>(a->workspace) & 255) != 0) return fail(-5, "workspace must be 256-byte aligned");
  return 0;
}

int nnb_render_fwd(const nnb_render_args* a, void* stream) {
  int rc = check_args(a); if (rc) return rc;
  WsLayout L = make_layout(a->N, a->S, a->flags, a->engine, hidden_of(a->hidden_dim));
  // pts / dirs belong to the nnb_field_* calls; the render kernels would take a non-NULL pts for N * S explicit points
  nnb_render_args r = *a; r.pts = nullptr; r.dirs = nullptr;
  cudaError_t e;
#ifdef NNB_WITH_TC
  if (r.engine == NNB_ENGINE_TC) e = tc_render_fwd(r, L, (cudaStream_t)stream); else
#endif
  e = simt_render_fwd(r, L, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : cuda_fail(e, "nnb_render_fwd");
}

int nnb_render_bwd(const nnb_render_bwd_args* b, void* stream) {
  if (!b) return fail(-1, "null args");
  int rc = check_args(&b->fwd); if (rc) return rc;
  if (!(b->fwd.flags & NNB_STASH)) return fail(-6, "nnb_render_bwd needs the forward call to have run with NNB_STASH");
  if (!b->g_rgb || !b->g_c2w) return fail(-3, "g_rgb and g_c2w must be non-null");
  WsLayout L = make_layout(b->fwd.N, b->fwd.S, b->fwd.flags, b->fwd.engine, hidden_of(b->fwd.hidden_dim));
  nnb_render_bwd_args r = *b; r.fwd.pts = nullptr; r.fwd.dirs = nullptr;   // as in nnb_render_fwd
  cudaError_t e;
#ifdef NNB_WITH_TC
  if (r.fwd.engine == NNB_ENGINE_TC) e = tc_render_bwd(r, L, (cudaStream_t)stream); else
#endif
  e = simt_render_bwd(r, L, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : cuda_fail(e, "nnb_render_bwd");
}

// test aid: the weight-gradient stage of nnb_render_bwd for a->engine alone, on whatever the workspace's stash holds
int nnb_debug_wgrad(const nnb_render_args* a, float* g_weights, void* stream) {
  if (!a || !g_weights) return fail(-3, "nnb_debug_wgrad: need args and g_weights");
  if (a->N <= 0) return fail(-2, "N must be positive (got %d)", a->N);
  if (a->S < 2 || a->S > 1024) return fail(-2, "S must be in [2,1024] (got %d)", a->S);
  if (!(a->flags & NNB_STASH)) return fail(-6, "nnb_debug_wgrad needs the stash (NNB_STASH)");
  if (int rc = check_engine_ws(a)) return rc;
  WsLayout L = make_layout(a->N, a->S, a->flags, a->engine, hidden_of(a->hidden_dim));
  cudaError_t e;
#ifdef NNB_WITH_TC
  if (a->engine == NNB_ENGINE_TC) e = tc_wgrad_stage(*a, L, g_weights, (cudaStream_t)stream); else
#endif
  e = simt_wgrad_stage(*a, L, g_weights, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : cuda_fail(e, "nnb_debug_wgrad");
}

static int check_field(const nnb_render_args* a) {
  if (!a || !a->pts || !a->weights || a->N <= 0) return fail(-3, "nnb_field_*: need pts, weights, N > 0");
  if (int rc = check_flags(a->flags)) return rc;
  if (int rc = check_dim(a)) return rc;
  size_t need = make_layout(a->N, 1, a->flags, NNB_ENGINE_SIMT, hidden_of(a->hidden_dim)).total;
  if (!a->workspace || a->workspace_bytes < need) return fail(-5, "workspace too small: have %zu need %zu", a->workspace_bytes, need);
  return 0;
}
int nnb_field_fwd(const nnb_render_args* a, float* out_rgba, void* stream) {
  int rc = check_field(a); if (rc) return rc;
  if (!out_rgba) return fail(-3, "nnb_field_fwd: out_rgba is null");
  if (a->engine == NNB_ENGINE_TC) {
#ifndef NNB_WITH_TC
    return fail(-4, "library built without the tensor-core engine");
#else
    if (a->flags & NNB_STASH)
      return fail(-6, "nnb_field_fwd: NNB_STASH needs NNB_ENGINE_SIMT (the tensor-core field query is inference only; gradients run on the exact-fp32 engine)");
    const size_t need = nnb_workspace_bytes_dim(a->N, 1, a->flags, NNB_ENGINE_TC, a->hidden_dim);
    if (a->workspace_bytes < need) return fail(-5, "workspace too small: have %zu need %zu", a->workspace_bytes, need);
    if ((reinterpret_cast<uintptr_t>(a->workspace) & 255) != 0) return fail(-5, "workspace must be 256-byte aligned");
    if ((reinterpret_cast<uintptr_t>(out_rgba) & 15) != 0) return fail(-3, "nnb_field_fwd: out_rgba must be 16-byte aligned");
    nnb_render_args b = *a; b.S = 1;
    cudaError_t e = tc_field_fwd_points(b, make_layout(b.N, 1, b.flags, NNB_ENGINE_TC, hidden_of(b.hidden_dim)), out_rgba, (cudaStream_t)stream);
    return e == cudaSuccess ? 0 : cuda_fail(e, "nnb_field_fwd");
#endif
  }
  if (a->flags & NNB_OCC_ONLY) return fail(-6, "nnb_field_fwd: NNB_OCC_ONLY needs NNB_ENGINE_TC");
  nnb_render_args b = *a; b.S = 1; b.engine = NNB_ENGINE_SIMT;
  cudaError_t e = simt_field_fwd(b, make_layout(b.N, 1, b.flags, NNB_ENGINE_SIMT, hidden_of(b.hidden_dim)), out_rgba, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : cuda_fail(e, "nnb_field_fwd");
}
size_t nnb_ray_march_workspace_bytes(int32_t N, int32_t n_steps, int32_t hidden_dim) {
  return nnb_ray_march_workspace_bytes_engine(N, n_steps, hidden_dim, NNB_ENGINE_TC);
}
size_t nnb_ray_march_workspace_bytes_engine(int32_t N, int32_t n_steps, int32_t hidden_dim, int32_t engine) {
  const int D = hidden_of(hidden_dim);
  if (N <= 0 || n_steps < 2 || !nnb::dim_supported(D)) return 0;
  if (engine == NNB_ENGINE_SIMT) return simt_ray_march_workspace(N, n_steps);
#ifdef NNB_WITH_TC
  if (engine == NNB_ENGINE_TC) return tc_ray_march_workspace(N, n_steps, D);
#endif
  return 0;
}
// the engines of nnb_ray_march_engine / nnb_geometry_frame_engine: NNB_ENGINE_TC (when built with it) and NNB_ENGINE_SIMT
static int check_march_engine(int32_t engine, const char* call) {
  if (engine != NNB_ENGINE_TC && engine != NNB_ENGINE_SIMT)
    return fail(-4, "%s: engine %d has no fused march (NNB_ENGINE_TC or NNB_ENGINE_SIMT)", call, engine);
#ifndef NNB_WITH_TC
  if (engine == NNB_ENGINE_TC) return fail(-4, "library built without the tensor-core engine");
#endif
  return 0;
}
// the checks after the engine's and the call, on a->engine (validated by the caller)
static int ray_march_on(const nnb_ray_march_args* a, void* stream) {
  const int D = hidden_of(a->hidden_dim);
  if (!nnb::dim_supported(D)) return fail(-8, "hidden_dim %d is not supported (supported: 64, 128, 256; 0 means 256)", a->hidden_dim);
  if (a->N < 0) return fail(-2, "nnb_ray_march: N must not be negative (got %d)", a->N);
  if (a->n_steps < 2 || a->n_secant < 0) return fail(-2, "nnb_ray_march: need n_steps >= 2 and n_secant >= 0 (got %d, %d)", a->n_steps, a->n_secant);
  if (a->N == 0) return 0;
  if (!a->weights || !a->ray0 || !a->ray_dir || !a->far_ || !a->frac || !a->depth)
    return fail(-3, "nnb_ray_march: weights, ray0, ray_dir, far_, frac and depth must be non-null");
  const size_t need = nnb_ray_march_workspace_bytes_engine(a->N, a->n_steps, a->hidden_dim, a->engine);
  if (!a->workspace || a->workspace_bytes < need) return fail(-5, "workspace too small: have %zu need %zu", a->workspace_bytes, need);
  if ((reinterpret_cast<uintptr_t>(a->workspace) & 255) != 0) return fail(-5, "workspace must be 256-byte aligned");
  if ((reinterpret_cast<uintptr_t>(a->bracket) & 15) != 0) return fail(-3, "nnb_ray_march: bracket must be 16-byte aligned");
  cudaError_t e;
#ifdef NNB_WITH_TC
  if (a->engine == NNB_ENGINE_TC) e = tc_ray_march(*a, D, (cudaStream_t)stream); else
#endif
  e = simt_ray_march(*a, D, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : cuda_fail(e, "nnb_ray_march");
}
int nnb_ray_march(const nnb_ray_march_args* a, void* stream) {
  if (!a) return fail(-1, "null args");
  if (a->engine != NNB_ENGINE_TC)
    return fail(-4, "nnb_ray_march: engine %d has no fused march here (NNB_ENGINE_TC only; nnb_ray_march_engine runs NNB_ENGINE_SIMT)", a->engine);
#ifndef NNB_WITH_TC
  return fail(-4, "library built without the tensor-core engine");
#else
  return ray_march_on(a, stream);
#endif
}
int nnb_ray_march_engine(const nnb_ray_march_args* a, void* stream) {
  if (!a) return fail(-1, "null args");
  if (int rc = check_march_engine(a->engine, "nnb_ray_march_engine")) return rc;
  return ray_march_on(a, stream);
}
size_t nnb_field_vjp_workspace_bytes(int32_t N, uint32_t flags, int32_t hidden_dim) {
#ifdef NNB_WITH_TC
  const int D = hidden_of(hidden_dim);
  if (N > 0 && nnb::dim_supported(D) && !(flags & ~KNOWN_FLAGS)) return tc_field_vjp_workspace(N, flags, D);
#endif
  return 0;
}
static inline bool misaligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) != 0; }
int nnb_field_vjp(const nnb_render_args* a, const float* g_rgba, float* out_rgba, float* g_pts, float* g_dirs, void* stream) {
  if (!a) return fail(-3, "nnb_field_vjp: null args");
  if (a->engine != NNB_ENGINE_TC)
    return fail(-4, "nnb_field_vjp: engine %d has no explicit-point data gradient here (NNB_ENGINE_TC only; the exact-fp32 engine has nnb_field_bwd)",
                a->engine);
#ifndef NNB_WITH_TC
  return fail(-4, "library built without the tensor-core engine");
#else
  if (int rc = check_flags(a->flags)) return rc;
  if (a->flags & (NNB_STASH | NNB_HVP))
    return fail(-6, "nnb_field_vjp: NNB_STASH and NNB_HVP are not accepted (nothing is stashed; weight gradients and nnb_field_hvp need the exact-fp32 engine)");
  if (int rc = check_dim(a)) return rc;
  if (a->N < 0) return fail(-3, "nnb_field_vjp: N must not be negative (got %d)", a->N);
  if ((a->flags & NNB_OCC_ONLY) && g_dirs) return fail(-6, "nnb_field_vjp: g_dirs must be NULL with NNB_OCC_ONLY (the colour branch is not evaluated)");
  if (a->N == 0) return 0;
  if (!a->pts || !a->weights || !g_rgba || !g_pts) return fail(-3, "nnb_field_vjp: need pts, weights, g_rgba and g_pts");
  if (misaligned16(g_rgba) || misaligned16(out_rgba) || misaligned16(g_pts) || misaligned16(g_dirs))
    return fail(-3, "nnb_field_vjp: g_rgba, out_rgba, g_pts and g_dirs must be 16-byte aligned [N][4] arrays");
  const size_t need = nnb_field_vjp_workspace_bytes(a->N, a->flags, a->hidden_dim);
  if (!a->workspace || a->workspace_bytes < need) return fail(-5, "workspace too small: have %zu need %zu", a->workspace_bytes, need);
  if ((reinterpret_cast<uintptr_t>(a->workspace) & 255) != 0) return fail(-5, "workspace must be 256-byte aligned");
  nnb_render_args b = *a; b.S = 1;
  cudaError_t e = tc_field_vjp(b, g_rgba, out_rgba, g_pts, g_dirs, hidden_of(a->hidden_dim), (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : cuda_fail(e, "nnb_field_vjp");
#endif
}
size_t nnb_field_grad_workspace_bytes(int32_t N, uint32_t flags, int32_t hidden_dim) {
#ifdef NNB_WITH_TC
  const int D = hidden_of(hidden_dim);
  if (N > 0 && nnb::dim_supported(D) && !(flags & ~KNOWN_FLAGS)) return tc_field_grad_workspace(N, flags, D);
#endif
  return 0;
}
// the arguments of nnb_field_vjp, plus g_weights (4-byte aligned floats, ACCUMULATED); the same checks in the same order
int nnb_field_grad(const nnb_render_args* a, const float* g_rgba, float* out_rgba, float* g_pts, float* g_dirs, float* g_weights, void* stream) {
  if (!a) return fail(-3, "nnb_field_grad: null args");
  if (a->engine != NNB_ENGINE_TC)
    return fail(-4, "nnb_field_grad: engine %d has no tensor-core field gradient (NNB_ENGINE_TC only; the exact-fp32 engine has nnb_field_bwd)",
                a->engine);
#ifndef NNB_WITH_TC
  return fail(-4, "library built without the tensor-core engine");
#else
  if (int rc = check_flags(a->flags)) return rc;
  if (a->flags & (NNB_STASH | NNB_HVP))
    return fail(-6, "nnb_field_grad: NNB_STASH and NNB_HVP are not accepted (the call keeps its own stash; nnb_field_hvp needs the exact-fp32 engine)");
  if (int rc = check_dim(a)) return rc;
  if (a->N < 0) return fail(-3, "nnb_field_grad: N must not be negative (got %d)", a->N);
  if ((a->flags & NNB_OCC_ONLY) && g_dirs) return fail(-6, "nnb_field_grad: g_dirs must be NULL with NNB_OCC_ONLY (the colour branch is not evaluated)");
  if (a->N == 0) return 0;
  if (!a->pts || !a->weights || !g_rgba || !g_pts) return fail(-3, "nnb_field_grad: need pts, weights, g_rgba and g_pts");
  if (misaligned16(g_rgba) || misaligned16(out_rgba) || misaligned16(g_pts) || misaligned16(g_dirs))
    return fail(-3, "nnb_field_grad: g_rgba, out_rgba, g_pts and g_dirs must be 16-byte aligned [N][4] arrays");
  if ((reinterpret_cast<uintptr_t>(g_weights) & 3) != 0) return fail(-3, "nnb_field_grad: g_weights must be 4-byte aligned");
  const size_t need = nnb_field_grad_workspace_bytes(a->N, a->flags, a->hidden_dim);
  if (!a->workspace || a->workspace_bytes < need) return fail(-5, "workspace too small: have %zu need %zu", a->workspace_bytes, need);
  if ((reinterpret_cast<uintptr_t>(a->workspace) & 255) != 0) return fail(-5, "workspace must be 256-byte aligned");
  nnb_render_args b = *a; b.S = 1;
  cudaError_t e = tc_field_grad(b, g_rgba, out_rgba, g_pts, g_dirs, g_weights, hidden_of(a->hidden_dim), (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : cuda_fail(e, "nnb_field_grad");
#endif
}
size_t nnb_field_hvp_tc_workspace_bytes(int32_t N, uint32_t flags, int32_t hidden_dim) {
#ifdef NNB_WITH_TC
  const int D = hidden_of(hidden_dim);
  if (N > 0 && nnb::dim_supported(D) && !(flags & ~KNOWN_FLAGS)) return tc_field_hvp_workspace(N, D);
#endif
  return 0;
}
// the checks of nnb_field_grad in its order; u takes g_rgba's place and g_pts is optional when g_weights is given
int nnb_field_hvp_tc(const nnb_render_args* a, const float* u, float* g_pts, float* g_weights, void* stream) {
  if (!a) return fail(-3, "nnb_field_hvp_tc: null args");
  if (a->engine != NNB_ENGINE_TC)
    return fail(-4, "nnb_field_hvp_tc: engine %d has no tensor-core second-order backward (NNB_ENGINE_TC only; the exact-fp32 engine has "
                "nnb_field_hvp)", a->engine);
#ifndef NNB_WITH_TC
  return fail(-4, "library built without the tensor-core engine");
#else
  if (int rc = check_flags(a->flags)) return rc;
  if (a->flags & (NNB_STASH | NNB_HVP))
    return fail(-6, "nnb_field_hvp_tc: NNB_STASH and NNB_HVP are not accepted (the call keeps its own stash; they size nnb_field_hvp's)");
  if (int rc = check_dim(a)) return rc;
  if (a->N < 0) return fail(-3, "nnb_field_hvp_tc: N must not be negative (got %d)", a->N);
  if (a->N == 0) return 0;
  if (!a->pts || !a->weights || !u || (!g_pts && !g_weights))
    return fail(-3, "nnb_field_hvp_tc: need pts, weights, u and at least one of g_pts, g_weights");
  if (misaligned16(u) || misaligned16(g_pts)) return fail(-3, "nnb_field_hvp_tc: u and g_pts must be 16-byte aligned [N][4] arrays");
  if ((reinterpret_cast<uintptr_t>(g_weights) & 3) != 0) return fail(-3, "nnb_field_hvp_tc: g_weights must be 4-byte aligned");
  const size_t need = nnb_field_hvp_tc_workspace_bytes(a->N, a->flags, a->hidden_dim);
  if (!a->workspace || a->workspace_bytes < need) return fail(-5, "workspace too small: have %zu need %zu", a->workspace_bytes, need);
  if ((reinterpret_cast<uintptr_t>(a->workspace) & 255) != 0) return fail(-5, "workspace must be 256-byte aligned");
  nnb_render_args b = *a; b.S = 1; b.dirs = nullptr; b.flags |= NNB_RAW_DENSITY | NNB_OCC_ONLY;
  cudaError_t e = tc_field_hvp(b, u, g_pts, g_weights, hidden_of(a->hidden_dim), (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : cuda_fail(e, "nnb_field_hvp_tc");
#endif
}
size_t nnb_geometry_frame_workspace_bytes(int32_t N, int32_t n_steps, int32_t hidden_dim) {
  return nnb_geometry_frame_workspace_bytes_engine(N, n_steps, hidden_dim, NNB_ENGINE_TC);
}
size_t nnb_geometry_frame_workspace_bytes_engine(int32_t N, int32_t n_steps, int32_t hidden_dim, int32_t engine) {
  const int D = hidden_of(hidden_dim);
  if (N <= 0 || n_steps < 2 || !nnb::dim_supported(D)) return 0;
  if (engine == NNB_ENGINE_SIMT) return simt_geometry_frame_workspace(N, n_steps, D);
#ifdef NNB_WITH_TC
  if (engine == NNB_ENGINE_TC) return tc_geometry_frame_workspace(N, n_steps, D);
#endif
  return 0;
}
static inline bool misaligned4(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 3) != 0; }
// the checks after the engine's and the call, on a->engine (validated by the caller)
static int geometry_frame_on(const nnb_geometry_args* a, void* stream) {
  if (int rc = check_flags(a->flags)) return rc;
  if (a->flags & ~(NNB_DIST_ALPHA | NNB_SOFTPLUS))
    return fail(-6, "nnb_geometry_frame: flags 0x%x: only NNB_DIST_ALPHA and NNB_SOFTPLUS are accepted", a->flags);
  const int D = hidden_of(a->hidden_dim);
  if (!nnb::dim_supported(D)) return fail(-8, "hidden_dim %d is not supported (supported: 64, 128, 256; 0 means 256)", a->hidden_dim);
  if (a->N < 0) return fail(-2, "nnb_geometry_frame: N must not be negative (got %d)", a->N);
  if (a->n_steps < 2 || a->n_secant < 0)
    return fail(-2, "nnb_geometry_frame: need n_steps >= 2 and n_secant >= 0 (got %d, %d)", a->n_steps, a->n_secant);
  if (a->N == 0) return 0;
  if (!a->weights || !a->T || !a->pixels || !a->frac || !a->rgb || !a->rgb_surf)
    return fail(-3, "nnb_geometry_frame: weights, T, pixels, frac, rgb and rgb_surf must be non-null");
  for (const void* p : {(const void*)a->weights, (const void*)a->T, (const void*)a->pixels, (const void*)a->frac, (const void*)a->rgb,
                        (const void*)a->rgb_surf, (const void*)a->ray0, (const void*)a->ray_dir, (const void*)a->far_, (const void*)a->depth})
    if (misaligned4(p)) return fail(-3, "nnb_geometry_frame: float arrays must be 4-byte aligned");
  if (misaligned16(a->grad)) return fail(-3, "nnb_geometry_frame: grad must be a 16-byte aligned [N][4] array");
  const size_t need = nnb_geometry_frame_workspace_bytes_engine(a->N, a->n_steps, a->hidden_dim, a->engine);
  if (!a->workspace || a->workspace_bytes < need) return fail(-5, "workspace too small: have %zu need %zu", a->workspace_bytes, need);
  if ((reinterpret_cast<uintptr_t>(a->workspace) & 255) != 0) return fail(-5, "workspace must be 256-byte aligned");
  cudaError_t e;
#ifdef NNB_WITH_TC
  if (a->engine == NNB_ENGINE_TC) e = tc_geometry_frame(*a, D, (cudaStream_t)stream); else
#endif
  e = simt_geometry_frame(*a, D, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : cuda_fail(e, "nnb_geometry_frame");
}
int nnb_geometry_frame(const nnb_geometry_args* a, void* stream) {
  if (!a) return fail(-1, "null args");
  if (a->engine != NNB_ENGINE_TC)
    return fail(-4, "nnb_geometry_frame: engine %d has no geometry frame here (NNB_ENGINE_TC only; nnb_geometry_frame_engine runs NNB_ENGINE_SIMT)",
                a->engine);
#ifndef NNB_WITH_TC
  return fail(-4, "library built without the tensor-core engine");
#else
  return geometry_frame_on(a, stream);
#endif
}
int nnb_geometry_frame_engine(const nnb_geometry_args* a, void* stream) {
  if (!a) return fail(-1, "null args");
  if (int rc = check_march_engine(a->engine, "nnb_geometry_frame_engine")) return rc;
  return geometry_frame_on(a, stream);
}
size_t nnb_render_frame_workspace_bytes(int32_t N, int32_t S, int32_t hidden_dim) {
#ifdef NNB_WITH_TC
  const int D = hidden_of(hidden_dim);
  if (N > 0 && tc_supports(S) && nnb::dim_supported(D)) return tc_render_frame_workspace(N, D);
#endif
  return 0;
}
size_t nnb_render_frame_workspace_bytes_engine(int32_t N, int32_t S, int32_t hidden_dim, int32_t engine) {
  if (engine == NNB_ENGINE_TC) return nnb_render_frame_workspace_bytes(N, S, hidden_dim);
  if (engine == NNB_ENGINE_SIMT && N > 0 && S >= 2 && S <= 1024 && nnb::dim_supported(hidden_of(hidden_dim)))
    return simt_render_frame_workspace(N);
  return 0;
}
// the checks of the frame's render arguments after the engine's, in nnb_render_frame's order up to the output pointers; `noise` is
// accepted with allow_noise only (nnb_render_frame_train_fwd / _bwd)
static int check_frame(const nnb_render_args* a, bool allow_noise = false) {
  if (int rc = check_flags(a->flags)) return rc;
  if (a->flags & (NNB_STASH | NNB_HVP | NNB_OCC_ONLY | NNB_RAW_DENSITY))
    return fail(-6, "nnb_render_frame: NNB_STASH, NNB_HVP, NNB_OCC_ONLY and NNB_RAW_DENSITY are not accepted (flags 0x%x)", a->flags);
  if (int rc = check_dim(a)) return rc;
  if (a->N <= 0) return fail(-2, "N must be positive (got %d)", a->N);
  if (a->S < 2 || a->S > 1024) return fail(-2, "S must be in [2,1024] (got %d)", a->S);
#ifdef NNB_WITH_TC
  if (a->engine == NNB_ENGINE_TC && !tc_supports(a->S))
    return fail(-4, "tensor-core engine needs S in [16,1024] (got %d); use nnb_render_fwd on NNB_ENGINE_SIMT", a->S);
#endif
  if ((a->noise && !allow_noise) || a->z_vals || a->alpha || a->pts || a->dirs)
    return fail(-6, allow_noise ? "nnb_render_frame_train: z_vals, alpha, pts and dirs must be NULL (no per-sample outputs)"
                                : "nnb_render_frame: noise, z_vals, alpha, pts and dirs must be NULL (no jitter, no per-sample outputs)");
  return 0;
}
// the render arguments' checks after the t_min check
static int check_frame_io(const nnb_render_args* a) {
  if (!a->weights || !a->c2w || !a->cam) return fail(-3, "weights / c2w / cam must be non-null");
  if (!a->ray_idx && !a->pixels) return fail(-3, "need ray_idx or pixels");
  if (!a->pixels && (a->H < 2 || a->W < 2)) return fail(-3, "H,W needed to derive pixels from ray_idx");
  if (!a->depth && !(a->depth_map && a->ray_idx && a->h_d > 0 && a->w_d > 0 && a->H > 0 && a->W > 0))
    return fail(-3, "need depth[N] or (depth_map,h_d,w_d,H,W,ray_idx)");
  if (!a->rgb || !a->depth_pred || !a->depth_gt || !a->mask) return fail(-3, "output pointers must be non-null");
  return 0;
}
// the checks after the engine's and the call, on f->fwd.engine (NNB_ENGINE_TC or NNB_ENGINE_SIMT, validated by the caller)
static int render_frame_on(const nnb_frame_args* f, void* stream) {
  const nnb_render_args* a = &f->fwd;
  if (int rc = check_frame(a)) return rc;
  if (!(f->t_min >= 0.f)) return fail(-2, "nnb_render_frame: t_min must be >= 0 (got %g)", (double)f->t_min);
  if (int rc = check_frame_io(a)) return rc;
  if (misaligned4(f->n_eval) || misaligned4(f->t_final)) return fail(-3, "nnb_render_frame: n_eval and t_final must be 4-byte aligned");
  const int D = hidden_of(a->hidden_dim);
  const size_t need = nnb_render_frame_workspace_bytes_engine(a->N, a->S, a->hidden_dim, a->engine);
  if (!a->workspace || a->workspace_bytes < need) return fail(-5, "workspace too small: have %zu need %zu", a->workspace_bytes, need);
  if ((reinterpret_cast<uintptr_t>(a->workspace) & 255) != 0) return fail(-5, "workspace must be 256-byte aligned");
  cudaError_t e;
#ifdef NNB_WITH_TC
  if (a->engine == NNB_ENGINE_TC) e = tc_render_frame(*a, f->t_min, f->n_eval, f->t_final, D, (cudaStream_t)stream); else
#endif
  e = simt_render_frame(*a, f->t_min, f->n_eval, f->t_final, D, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : cuda_fail(e, "nnb_render_frame");
}
int nnb_render_frame(const nnb_frame_args* f, void* stream) {
  if (!f) return fail(-1, "null args");
  const nnb_render_args* a = &f->fwd;
  if (a->engine != NNB_ENGINE_TC)
    return fail(-4, "nnb_render_frame: engine %d has no frame renderer here (NNB_ENGINE_TC only; nnb_render_frame_engine runs NNB_ENGINE_SIMT)",
                a->engine);
#ifndef NNB_WITH_TC
  return fail(-4, "library built without the tensor-core engine");
#else
  return render_frame_on(f, stream);
#endif
}
int nnb_render_frame_engine(const nnb_frame_args* f, void* stream) {
  if (!f) return fail(-1, "null args");
  const int32_t engine = f->fwd.engine;
  if (engine != NNB_ENGINE_TC && engine != NNB_ENGINE_SIMT)
    return fail(-4, "nnb_render_frame_engine: engine %d has no frame renderer (NNB_ENGINE_TC or NNB_ENGINE_SIMT)", engine);
#ifndef NNB_WITH_TC
  if (engine == NNB_ENGINE_TC) return fail(-4, "library built without the tensor-core engine");
#endif
  return render_frame_on(f, stream);
}
size_t nnb_render_frame_bwd_workspace_bytes(int32_t N, int32_t S, int32_t hidden_dim) {
#ifdef NNB_WITH_TC
  const int D = hidden_of(hidden_dim);
  if (N > 0 && tc_supports(S) && nnb::dim_supported(D)) return tc_render_frame_bwd_workspace(N, S, D);
#endif
  return 0;
}
int nnb_render_frame_bwd(const nnb_render_bwd_args* b, void* stream) {
  if (!b) return fail(-1, "null args");
  const nnb_render_args* a = &b->fwd;
  if (a->engine != NNB_ENGINE_TC)
    return fail(-4, "nnb_render_frame_bwd: engine %d has no differentiable frame (NNB_ENGINE_TC only)", a->engine);
#ifndef NNB_WITH_TC
  return fail(-4, "library built without the tensor-core engine");
#else
  if (int rc = check_frame(a)) return rc;
  if (int rc = check_frame_io(a)) return rc;
  if (!b->g_rgb || !b->g_c2w) return fail(-3, "nnb_render_frame_bwd: g_rgb and g_c2w must be non-null");
  const int D = hidden_of(a->hidden_dim);
  const size_t need = nnb_render_frame_bwd_workspace_bytes(a->N, a->S, a->hidden_dim);
  if (!a->workspace || a->workspace_bytes < need) return fail(-5, "workspace too small: have %zu need %zu", a->workspace_bytes, need);
  if ((reinterpret_cast<uintptr_t>(a->workspace) & 255) != 0) return fail(-5, "workspace must be 256-byte aligned");
  const cudaError_t e = tc_render_frame_bwd(*b, D, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : cuda_fail(e, "nnb_render_frame_bwd");
#endif
}
// the checks of nnb_render_frame_train_fwd / _bwd on b->fwd up to the workspace's, nnb_render_frame_bwd's with noise accepted
static int check_frame_train(const nnb_render_args* a, const char* name) {
  if (a->engine != NNB_ENGINE_TC) return fail(-4, "%s: engine %d has no differentiable frame (NNB_ENGINE_TC only)", name, a->engine);
#ifndef NNB_WITH_TC
  return fail(-4, "library built without the tensor-core engine");
#else
  if (int rc = check_frame(a, true)) return rc;
  return check_frame_io(a);
#endif
}
static int check_frame_train_ws(const nnb_render_args* a) {
  const size_t need = nnb_render_frame_bwd_workspace_bytes(a->N, a->S, a->hidden_dim);
  if (!a->workspace || a->workspace_bytes < need) return fail(-5, "workspace too small: have %zu need %zu", a->workspace_bytes, need);
  if ((reinterpret_cast<uintptr_t>(a->workspace) & 255) != 0) return fail(-5, "workspace must be 256-byte aligned");
  return 0;
}
int nnb_render_frame_train_fwd(const nnb_render_args* a, void* stream) {
  if (!a) return fail(-1, "null args");
  if (int rc = check_frame_train(a, "nnb_render_frame_train_fwd")) return rc;
  if (int rc = check_frame_train_ws(a)) return rc;
#ifdef NNB_WITH_TC
  const cudaError_t e = tc_render_frame_train_fwd(*a, hidden_of(a->hidden_dim), (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : cuda_fail(e, "nnb_render_frame_train_fwd");
#else
  return fail(-4, "library built without the tensor-core engine");
#endif
}
int nnb_render_frame_train_bwd(const nnb_render_bwd_args* b, void* stream) {
  if (!b) return fail(-1, "null args");
  const nnb_render_args* a = &b->fwd;
  if (int rc = check_frame_train(a, "nnb_render_frame_train_bwd")) return rc;
  if (!b->g_rgb || !b->g_c2w) return fail(-3, "nnb_render_frame_train_bwd: g_rgb and g_c2w must be non-null");
  if (int rc = check_frame_train_ws(a)) return rc;
#ifdef NNB_WITH_TC
  const cudaError_t e = tc_render_frame_train_bwd(*b, hidden_of(a->hidden_dim), (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : cuda_fail(e, "nnb_render_frame_train_bwd");
#else
  return fail(-4, "library built without the tensor-core engine");
#endif
}
int nnb_render_frame_train_fwd_tmin(const nnb_frame_args* f, void* stream) {
  if (!f) return fail(-1, "null args");
  const nnb_render_args* a = &f->fwd;
  if (a->engine != NNB_ENGINE_TC)
    return fail(-4, "nnb_render_frame_train_fwd_tmin: engine %d has no differentiable frame with early termination (NNB_ENGINE_TC only)",
                a->engine);
#ifndef NNB_WITH_TC
  return fail(-4, "library built without the tensor-core engine");
#else
  if (int rc = check_frame(a, true)) return rc;
  if (!(f->t_min >= 0.f)) return fail(-2, "nnb_render_frame_train_fwd_tmin: t_min must be >= 0 (got %g)", (double)f->t_min);
  if (int rc = check_frame_io(a)) return rc;
  if (misaligned4(f->n_eval) || misaligned4(f->t_final))
    return fail(-3, "nnb_render_frame_train_fwd_tmin: n_eval and t_final must be 4-byte aligned");
  if (int rc = check_frame_train_ws(a)) return rc;
  const cudaError_t e = tc_render_frame_train_fwd_tmin(*f, hidden_of(a->hidden_dim), (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : cuda_fail(e, "nnb_render_frame_train_fwd_tmin");
#endif
}
int nnb_render_frame_train_bwd_tmin(const nnb_render_bwd_args* b, void* stream) {
  if (!b) return fail(-1, "null args");
  const nnb_render_args* a = &b->fwd;
  if (a->engine != NNB_ENGINE_TC)
    return fail(-4, "nnb_render_frame_train_bwd_tmin: engine %d has no differentiable frame with early termination (NNB_ENGINE_TC only)",
                a->engine);
#ifndef NNB_WITH_TC
  return fail(-4, "library built without the tensor-core engine");
#else
  if (int rc = check_frame(a, true)) return rc;
  if (int rc = check_frame_io(a)) return rc;
  if (!b->g_rgb || !b->g_c2w) return fail(-3, "nnb_render_frame_train_bwd_tmin: g_rgb and g_c2w must be non-null");
  if (int rc = check_frame_train_ws(a)) return rc;
  const cudaError_t e = tc_render_frame_train_bwd_tmin(*b, hidden_of(a->hidden_dim), (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : cuda_fail(e, "nnb_render_frame_train_bwd_tmin");
#endif
}
size_t nnb_render_tmin_workspace_bytes(int32_t N, int32_t S, int32_t hidden_dim) {
#ifdef NNB_WITH_TC
  const int D = hidden_of(hidden_dim);
  if (N > 0 && tc_supports(S) && nnb::dim_supported(D)) return tc_render_tmin_workspace(N, S, D);
#endif
  return 0;
}
static int check_tmin_ws(const nnb_render_args* a) {
  const size_t need = nnb_render_tmin_workspace_bytes(a->N, a->S, a->hidden_dim);
  if (!a->workspace || a->workspace_bytes < need) return fail(-5, "workspace too small: have %zu need %zu", a->workspace_bytes, need);
  if ((reinterpret_cast<uintptr_t>(a->workspace) & 255) != 0) return fail(-5, "workspace must be 256-byte aligned");
  return 0;
}
int nnb_render_fwd_tmin(const nnb_frame_args* f, void* stream) {
  if (!f) return fail(-1, "null args");
  const nnb_render_args* a = &f->fwd;
  if (a->engine != NNB_ENGINE_TC)
    return fail(-4, "nnb_render_fwd_tmin: engine %d has no stash render with early termination (NNB_ENGINE_TC only)", a->engine);
#ifndef NNB_WITH_TC
  return fail(-4, "library built without the tensor-core engine");
#else
  if (int rc = check_frame(a, true)) return rc;
  if (!(f->t_min >= 0.f)) return fail(-2, "nnb_render_fwd_tmin: t_min must be >= 0 (got %g)", (double)f->t_min);
  if (int rc = check_frame_io(a)) return rc;
  if (misaligned4(f->n_eval) || misaligned4(f->t_final)) return fail(-3, "nnb_render_fwd_tmin: n_eval and t_final must be 4-byte aligned");
  if (int rc = check_tmin_ws(a)) return rc;
  const cudaError_t e = tc_render_fwd_tmin(*f, hidden_of(a->hidden_dim), (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : cuda_fail(e, "nnb_render_fwd_tmin");
#endif
}
int nnb_render_bwd_tmin(const nnb_render_bwd_args* b, void* stream) {
  if (!b) return fail(-1, "null args");
  const nnb_render_args* a = &b->fwd;
  if (a->engine != NNB_ENGINE_TC)
    return fail(-4, "nnb_render_bwd_tmin: engine %d has no stash render with early termination (NNB_ENGINE_TC only)", a->engine);
#ifndef NNB_WITH_TC
  return fail(-4, "library built without the tensor-core engine");
#else
  if (int rc = check_frame(a, true)) return rc;
  if (int rc = check_frame_io(a)) return rc;
  if (!b->g_rgb || !b->g_c2w) return fail(-3, "nnb_render_bwd_tmin: g_rgb and g_c2w must be non-null");
  if (int rc = check_tmin_ws(a)) return rc;
  const cudaError_t e = tc_render_bwd_tmin(*b, hidden_of(a->hidden_dim), (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : cuda_fail(e, "nnb_render_bwd_tmin");
#endif
}
// The _engine forms of the stash pair with early termination: NNB_ENGINE_TC is the call without the suffix (its checks, codes, bits and
// workspace); NNB_ENGINE_SIMT runs the exact engine at any S from 2 to 1024 with the same checks in the same order.
size_t nnb_render_tmin_workspace_bytes_engine(int32_t N, int32_t S, int32_t hidden_dim, int32_t engine) {
  if (engine == NNB_ENGINE_TC) return nnb_render_tmin_workspace_bytes(N, S, hidden_dim);
  const int D = hidden_of(hidden_dim);
  if (engine == NNB_ENGINE_SIMT && N > 0 && S >= 2 && S <= 1024 && nnb::dim_supported(D)) return simt_render_tmin_workspace(N, S, D);
  return 0;
}
static int check_tmin_engine(int32_t engine, const char* name) {
  if (engine != NNB_ENGINE_TC && engine != NNB_ENGINE_SIMT)
    return fail(-4, "%s: engine %d has no stash render with early termination (NNB_ENGINE_TC or NNB_ENGINE_SIMT)", name, engine);
#ifndef NNB_WITH_TC
  if (engine == NNB_ENGINE_TC) return fail(-4, "library built without the tensor-core engine");
#endif
  return 0;
}
static int check_tmin_ws_engine(const nnb_render_args* a) {
  const size_t need = nnb_render_tmin_workspace_bytes_engine(a->N, a->S, a->hidden_dim, a->engine);
  if (!a->workspace || a->workspace_bytes < need) return fail(-5, "workspace too small: have %zu need %zu", a->workspace_bytes, need);
  if ((reinterpret_cast<uintptr_t>(a->workspace) & 255) != 0) return fail(-5, "workspace must be 256-byte aligned");
  return 0;
}
int nnb_render_fwd_tmin_engine(const nnb_frame_args* f, void* stream) {
  if (!f) return fail(-1, "null args");
  const nnb_render_args* a = &f->fwd;
  if (int rc = check_tmin_engine(a->engine, "nnb_render_fwd_tmin_engine")) return rc;
#ifdef NNB_WITH_TC
  if (a->engine == NNB_ENGINE_TC) return nnb_render_fwd_tmin(f, stream);
#endif
  if (int rc = check_frame(a, true)) return rc;
  if (!(f->t_min >= 0.f)) return fail(-2, "nnb_render_fwd_tmin_engine: t_min must be >= 0 (got %g)", (double)f->t_min);
  if (int rc = check_frame_io(a)) return rc;
  if (misaligned4(f->n_eval) || misaligned4(f->t_final))
    return fail(-3, "nnb_render_fwd_tmin_engine: n_eval and t_final must be 4-byte aligned");
  if (int rc = check_tmin_ws_engine(a)) return rc;
  const cudaError_t e = simt_render_fwd_tmin(*f, hidden_of(a->hidden_dim), (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : cuda_fail(e, "nnb_render_fwd_tmin_engine");
}
int nnb_render_bwd_tmin_engine(const nnb_render_bwd_args* b, void* stream) {
  if (!b) return fail(-1, "null args");
  const nnb_render_args* a = &b->fwd;
  if (int rc = check_tmin_engine(a->engine, "nnb_render_bwd_tmin_engine")) return rc;
#ifdef NNB_WITH_TC
  if (a->engine == NNB_ENGINE_TC) return nnb_render_bwd_tmin(b, stream);
#endif
  if (int rc = check_frame(a, true)) return rc;
  if (int rc = check_frame_io(a)) return rc;
  if (!b->g_rgb || !b->g_c2w) return fail(-3, "nnb_render_bwd_tmin_engine: g_rgb and g_c2w must be non-null");
  if (int rc = check_tmin_ws_engine(a)) return rc;
  const cudaError_t e = simt_render_bwd_tmin(*b, hidden_of(a->hidden_dim), (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : cuda_fail(e, "nnb_render_bwd_tmin_engine");
}
size_t nnb_render_frame_bwd_workspace_bytes_engine(int32_t N, int32_t S, int32_t hidden_dim, int32_t engine) {
  if (engine == NNB_ENGINE_TC) return nnb_render_frame_bwd_workspace_bytes(N, S, hidden_dim);
  const int D = hidden_of(hidden_dim);
  if (engine == NNB_ENGINE_SIMT && N > 0 && S >= 2 && S <= 1024 && nnb::dim_supported(D)) return simt_render_frame_bwd_workspace(N, S, D);
  return 0;
}
// the engine check of the _engine forms of the differentiable frame: NNB_ENGINE_TC (when built with it) or NNB_ENGINE_SIMT
static int check_frame_bwd_engine(int32_t engine, const char* name) {
  if (engine != NNB_ENGINE_TC && engine != NNB_ENGINE_SIMT)
    return fail(-4, "%s: engine %d has no differentiable frame (NNB_ENGINE_TC or NNB_ENGINE_SIMT)", name, engine);
#ifndef NNB_WITH_TC
  if (engine == NNB_ENGINE_TC) return fail(-4, "library built without the tensor-core engine");
#endif
  return 0;
}
static int check_frame_bwd_ws_engine(const nnb_render_args* a) {
  const size_t need = nnb_render_frame_bwd_workspace_bytes_engine(a->N, a->S, a->hidden_dim, a->engine);
  if (!a->workspace || a->workspace_bytes < need) return fail(-5, "workspace too small: have %zu need %zu", a->workspace_bytes, need);
  if ((reinterpret_cast<uintptr_t>(a->workspace) & 255) != 0) return fail(-5, "workspace must be 256-byte aligned");
  return 0;
}
// The _engine forms: NNB_ENGINE_TC is the call without the suffix (its checks, bits and workspace); NNB_ENGINE_SIMT runs the exact engine
// at any S from 2 to 1024 (check_frame accepts S < 16 there) with the same checks in the same order.
int nnb_render_frame_bwd_engine(const nnb_render_bwd_args* b, void* stream) {
  if (!b) return fail(-1, "null args");
  const nnb_render_args* a = &b->fwd;
  if (int rc = check_frame_bwd_engine(a->engine, "nnb_render_frame_bwd_engine")) return rc;
#ifdef NNB_WITH_TC
  if (a->engine == NNB_ENGINE_TC) return nnb_render_frame_bwd(b, stream);
#endif
  if (int rc = check_frame(a)) return rc;
  if (int rc = check_frame_io(a)) return rc;
  if (!b->g_rgb || !b->g_c2w) return fail(-3, "nnb_render_frame_bwd: g_rgb and g_c2w must be non-null");
  if (int rc = check_frame_bwd_ws_engine(a)) return rc;
  const cudaError_t e = simt_render_frame_bwd(*b, hidden_of(a->hidden_dim), (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : cuda_fail(e, "nnb_render_frame_bwd_engine");
}
int nnb_render_frame_train_fwd_engine(const nnb_render_args* a, void* stream) {
  if (!a) return fail(-1, "null args");
  if (int rc = check_frame_bwd_engine(a->engine, "nnb_render_frame_train_fwd_engine")) return rc;
#ifdef NNB_WITH_TC
  if (a->engine == NNB_ENGINE_TC) return nnb_render_frame_train_fwd(a, stream);
#endif
  if (int rc = check_frame(a, true)) return rc;
  if (int rc = check_frame_io(a)) return rc;
  if (int rc = check_frame_bwd_ws_engine(a)) return rc;
  const cudaError_t e = simt_render_frame_train_fwd(*a, hidden_of(a->hidden_dim), (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : cuda_fail(e, "nnb_render_frame_train_fwd_engine");
}
int nnb_render_frame_train_bwd_engine(const nnb_render_bwd_args* b, void* stream) {
  if (!b) return fail(-1, "null args");
  const nnb_render_args* a = &b->fwd;
  if (int rc = check_frame_bwd_engine(a->engine, "nnb_render_frame_train_bwd_engine")) return rc;
#ifdef NNB_WITH_TC
  if (a->engine == NNB_ENGINE_TC) return nnb_render_frame_train_bwd(b, stream);
#endif
  if (int rc = check_frame(a, true)) return rc;
  if (int rc = check_frame_io(a)) return rc;
  if (!b->g_rgb || !b->g_c2w) return fail(-3, "nnb_render_frame_train_bwd: g_rgb and g_c2w must be non-null");
  if (int rc = check_frame_bwd_ws_engine(a)) return rc;
  const cudaError_t e = simt_render_frame_train_bwd(*b, hidden_of(a->hidden_dim), (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : cuda_fail(e, "nnb_render_frame_train_bwd_engine");
}
int nnb_field_bwd(const nnb_render_args* a, const float* g_rgba, float* g_pts, float* g_dirs, float* g_weights, void* stream) {
  int rc = check_field(a); if (rc) return rc;
  if (!g_rgba || !(a->flags & NNB_STASH)) return fail(-3, "nnb_field_bwd: need g_rgba and a forward run with NNB_STASH");
  nnb_render_args b = *a; b.S = 1; b.engine = NNB_ENGINE_SIMT;
  cudaError_t e = simt_field_bwd(b, make_layout(b.N, 1, b.flags, NNB_ENGINE_SIMT, hidden_of(b.hidden_dim)), g_rgba, g_pts, g_dirs, g_weights,
                                 (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : cuda_fail(e, "nnb_field_bwd");
}
int nnb_field_hvp(const nnb_render_args* a, const float* u, float* g_pts, float* g_weights, void* stream) {
  int rc = check_field(a); if (rc) return rc;
  if (!u || (!g_pts && !g_weights)) return fail(-3, "nnb_field_hvp: need u and at least one of g_pts, g_weights");
  if (!(a->flags & NNB_STASH) || !(a->flags & NNB_HVP))
    return fail(-6, "nnb_field_hvp: flags must contain NNB_STASH | NNB_HVP, and the workspace be sized with them");
  if ((reinterpret_cast<uintptr_t>(a->workspace) & 255) != 0) return fail(-5, "workspace must be 256-byte aligned");
  if ((reinterpret_cast<uintptr_t>(u) & 15) != 0 || (reinterpret_cast<uintptr_t>(g_pts) & 15) != 0)
    return fail(-3, "nnb_field_hvp: u and g_pts must be 16-byte aligned [N][4] arrays");
  nnb_render_args b = *a; b.S = 1; b.engine = NNB_ENGINE_SIMT; b.flags |= NNB_RAW_DENSITY;
  cudaError_t e = simt_field_hvp(b, make_layout(b.N, 1, b.flags, NNB_ENGINE_SIMT, hidden_of(b.hidden_dim)), u, g_pts, g_weights,
                                 (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : cuda_fail(e, "nnb_field_hvp");
}

int nnb_pose_fwd(const float* r, const float* t, const float* init, int32_t cam, float* c2w, void* stream) {
  if (!r || !t || !c2w || cam < 0) return fail(-3, "nnb_pose_fwd: bad arguments");
  cudaError_t e = launch_pose_fwd(r, t, init, cam, nullptr, c2w, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : cuda_fail(e, "nnb_pose_fwd");
}
int nnb_pose_fwd_dev(const float* r, const float* t, const float* init, const int32_t* cam_dev, float* c2w, void* stream) {
  if (!r || !t || !c2w || !cam_dev) return fail(-3, "nnb_pose_fwd_dev: bad arguments");
  cudaError_t e = launch_pose_fwd(r, t, init, 0, cam_dev, c2w, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : cuda_fail(e, "nnb_pose_fwd_dev");
}
int nnb_pose_bwd_dev(const float* r, const float* t, const float* init, const int32_t* cam_dev, const float* g, float* gr, float* gt, void* stream) {
  if (!r || !t || !g || !cam_dev) return fail(-3, "nnb_pose_bwd_dev: bad arguments");
  cudaError_t e = launch_pose_bwd(r, t, init, 0, cam_dev, g, gr, gt, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : cuda_fail(e, "nnb_pose_bwd_dev");
}
int nnb_distortion_fwd_dev(const float* scales, const float* shifts, int32_t V, const int32_t* cam_dev, int32_t fix_last, float* out2, void* stream) {
  if (!scales || !shifts || !cam_dev || !out2 || V <= 0) return fail(-3, "nnb_distortion_fwd_dev: bad arguments");
  cudaError_t e = launch_distortion_fwd(scales, shifts, V, cam_dev, fix_last, out2, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : cuda_fail(e, "nnb_distortion_fwd_dev");
}
int nnb_distortion_bwd_dev(const float* scales, int32_t V, const int32_t* cam_dev, int32_t fix_last, const float* g_ss, float* g_scales,
                           float* g_shifts, void* stream) {
  if (!scales || !cam_dev || !g_ss || V <= 0) return fail(-3, "nnb_distortion_bwd_dev: bad arguments");
  cudaError_t e = launch_distortion_bwd(scales, V, cam_dev, fix_last, g_ss, g_scales, g_shifts, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : cuda_fail(e, "nnb_distortion_bwd_dev");
}
int nnb_adam_step_dev(float* p, const float* g, float* m, float* v, int64_t n, const int32_t* step_dev, const float* lr_dev, float b1, float b2,
                      float eps, void* stream) {
  if (!p || !g || !m || !v || n <= 0 || !step_dev || !lr_dev) return fail(-3, "nnb_adam_step_dev: bad arguments");
  cudaError_t e = launch_adam_dev(p, g, m, v, n, step_dev, lr_dev, b1, b2, eps, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : cuda_fail(e, "nnb_adam_step_dev");
}
int nnb_sample_pixels(const float* u2n, int32_t HW, int32_t N, int64_t* out, void* stream) {
  if (!u2n || !out || HW <= 0 || N <= 0 || N > HW / 2 || N > 8192) return fail(-3, "nnb_sample_pixels: bad arguments (need 0 < N <= min(HW/2, 8192))");
  cudaError_t e = launch_sample_pixels(u2n, HW, N, reinterpret_cast<long long*>(out), (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : cuda_fail(e, "nnb_sample_pixels");
}
int nnb_counter_incr(int32_t* counters, int32_t n, void* stream) {
  if (!counters || n <= 0 || n > 32) return fail(-3, "nnb_counter_incr: bad arguments");
  cudaError_t e = launch_incr(counters, n, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : cuda_fail(e, "nnb_counter_incr");
}
int nnb_pose_bwd(const float* r, const float* t, const float* init, int32_t cam, const float* g, float* gr, float* gt, void* stream) {
  if (!r || !t || !g || cam < 0) return fail(-3, "nnb_pose_bwd: bad arguments");
  cudaError_t e = launch_pose_bwd(r, t, init, cam, nullptr, g, gr, gt, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : cuda_fail(e, "nnb_pose_bwd");
}

int nnb_loss_rgb_depth(const float* rgb, const float* rgb_gt, const float* img, const int64_t* ray_idx, int32_t HW,
                       const float* dp, const float* dg, const uint8_t* mask, int32_t N, float w_rgb, float w_depth,
                       int32_t rgb_l2, float grad_scale, float* out, float* g_rgb, float* g_dp, float* g_dg, void* stream) {
  if (!rgb || !(rgb_gt || (img && ray_idx)) || !dp || !dg || !mask || !out || !g_rgb || !g_dp || !g_dg || N <= 0)
    return fail(-3, "nnb_loss_rgb_depth: bad arguments");
  cudaError_t e = launch_loss(rgb, rgb_gt, img, nullptr, ray_idx, HW, dp, dg, mask, N, w_rgb, w_depth, rgb_l2, grad_scale, out, g_rgb, g_dp, g_dg,
                              nullptr, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : cuda_fail(e, "nnb_loss_rgb_depth");
}
int nnb_loss_rgb_depth_indirect(const float* rgb, const float* const* img_pp, const int64_t* ray_idx, int32_t HW, const float* dp, const float* dg,
                                const uint8_t* mask, int32_t N, float w_rgb, float w_depth, int32_t rgb_l2, float grad_scale, float* out,
                                float* g_rgb, float* g_dp, float* g_dg, const float* w_dev, void* stream) {
  if (!rgb || !img_pp || !ray_idx || !dp || !dg || !mask || !out || !g_rgb || !g_dp || !g_dg || N <= 0)
    return fail(-3, "nnb_loss_rgb_depth_indirect: bad arguments");
  cudaError_t e = launch_loss(rgb, nullptr, nullptr, img_pp, ray_idx, HW, dp, dg, mask, N, w_rgb, w_depth, rgb_l2, grad_scale, out, g_rgb, g_dp,
                              g_dg, w_dev, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : cuda_fail(e, "nnb_loss_rgb_depth_indirect");
}

int nnb_chamfer(const float* X, int32_t P, const float* Y, int32_t Q, uint64_t* keys, int32_t* ixy, int32_t* iyx, float* loss, float weight,
                float* gX, float* gY, void* stream) {
  if (!X || !Y || !keys || !loss || P <= 0 || Q <= 0 || ((gX == nullptr) != (gY == nullptr)) || ((ixy == nullptr) != (iyx == nullptr)))
    return fail(-3, "nnb_chamfer: bad arguments");
  cudaError_t e = launch_chamfer_full(X, P, Y, Q, keys, loss, weight, nullptr, gX, gY, ixy, iyx, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : cuda_fail(e, "nnb_chamfer");
}

size_t nnb_chamfer_workspace_bytes(int32_t P, int32_t Q) {
  if (P <= 0 || Q <= 0 || (int64_t)P + Q > INT32_MAX) return 0;
  return chamfer_workspace_bytes(P, Q);
}

size_t nnb_refstage_workspace_bytes(int32_t h_d, int32_t w_d, int32_t pc_ratio) {
  if (h_d <= 0 || w_d <= 0 || pc_ratio <= 0 || h_d / pc_ratio < 2 || w_d / pc_ratio < 2) return 0;
  return refstage_workspace_bytes(h_d, w_d, pc_ratio);
}

size_t nnb_refstage_workspace_bytes_flags(int32_t h_d, int32_t w_d, int32_t pc_ratio, uint32_t flags) {
  if (h_d <= 0 || w_d <= 0 || pc_ratio <= 0 || h_d / pc_ratio < 2 || w_d / pc_ratio < 2) return 0;
  return refstage_workspace_bytes_flags(h_d, w_d, pc_ratio, flags);
}

int nnb_refstage(const nnb_refstage_args* a, void* stream) {
  if (!a) return fail(-1, "null args");
  if ((!a->img_pp && (!a->img_cur || !a->img_ref)) || !a->dpt_cur || !a->dpt_ref || !a->c2w_cur || !a->c2w_ref || !a->dist_cur || !a->dist_ref ||
      !a->losses)
    return fail(-3, "nnb_refstage: null pointer");
  if (a->cam_idx_dev && a->num_cams <= 0) return fail(-3, "nnb_refstage: cam_idx_dev needs num_cams");
  if (a->H < 2 || a->W < 2 || a->pc_ratio <= 0 || a->h_d / a->pc_ratio < 2 || a->w_d / a->pc_ratio < 2)
    return fail(-2, "nnb_refstage: bad sizes");
  if ((a->flags & 16u) && (!a->g_c2w_ref || !a->g_dist_ref))
    return fail(-3, "nnb_refstage: flag 16 (gradients into the reference view) needs g_c2w_ref and g_dist_ref");
  if (!a->workspace || a->workspace_bytes < refstage_workspace_bytes_flags(a->h_d, a->w_d, a->pc_ratio, a->flags))
    return fail(-4, "nnb_refstage: workspace too small");
  cudaError_t e = launch_refstage(*a, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : cuda_fail(e, "nnb_refstage");
}

int nnb_ipc_alloc(size_t bytes, void** dev_ptr, unsigned char handle_out[64]) {
  if (!dev_ptr || !handle_out || bytes == 0) return fail(-3, "nnb_ipc_alloc: bad arguments");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  void* p = nullptr;
  cudaError_t e = cudaMalloc(&p, bytes);
  if (e != cudaSuccess) return cuda_fail(e, "nnb_ipc_alloc: cudaMalloc");
  e = cudaMemset(p, 0, bytes);
  cudaIpcMemHandle_t h;
  if (e == cudaSuccess) e = cudaIpcGetMemHandle(&h, p);
  if (e != cudaSuccess) { cudaFree(p); return cuda_fail(e, "nnb_ipc_alloc: cudaIpcGetMemHandle"); }
  memcpy(handle_out, &h, 64);
  *dev_ptr = p;
  return 0;
}
int nnb_ipc_open(const unsigned char handle[64], void** peer_ptr) {
  if (!handle || !peer_ptr) return fail(-3, "nnb_ipc_open: bad arguments");
  cudaIpcMemHandle_t h; memcpy(&h, handle, 64);
  cudaError_t e = cudaIpcOpenMemHandle(peer_ptr, h, cudaIpcMemLazyEnablePeerAccess);
  return e == cudaSuccess ? 0 : cuda_fail(e, "nnb_ipc_open");
}
int nnb_ipc_close(void* peer_ptr) {
  cudaError_t e = cudaIpcCloseMemHandle(peer_ptr);
  return e == cudaSuccess ? 0 : cuda_fail(e, "nnb_ipc_close");
}
int nnb_ipc_free(void* dev_ptr) {
  cudaError_t e = cudaFree(dev_ptr);
  return e == cudaSuccess ? 0 : cuda_fail(e, "nnb_ipc_free");
}
int nnb_allreduce_adam(const nnb_allreduce_adam_args* a, void* stream) {
  if (!a) return fail(-1, "null args");
  if (a->world < 1 || a->world > NNB_MAX_RANKS || a->rank < 0 || a->rank >= a->world || a->n_total <= 0 || (a->n_total & 3) || a->nsegs < 0 || a->nsegs > 8)
    return fail(-2, "nnb_allreduce_adam: bad sizes");
  for (int r = 0; r < a->world; ++r) if (!a->peer_grads[r] || !a->peer_flags[r]) return fail(-3, "nnb_allreduce_adam: null peer pointer");
  for (int q = 0; q < a->nsegs; ++q) {
    const nnb_adam_seg& s = a->segs[q];
    if (!s.p || !s.m || !s.v || !s.lr_dev || !s.step_dev || s.offset < 0 || s.count <= 0 || s.offset + s.count > a->n_total)
      return fail(-3, "nnb_allreduce_adam: bad segment");
  }
  cudaError_t e = launch_allreduce_adam(*a, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : cuda_fail(e, "nnb_allreduce_adam");
}

int nnb_depth_invariant(const float* dp, const float* dg, const uint8_t* mask, int32_t N, const float* w_dev, float grad_scale, float* out_losses,
                        float* g_dp, float* g_dg, void* stream) {
  if (!dp || !dg || !mask || !w_dev || !out_losses || !g_dp || N <= 0 || N > NNB_INVARIANT_MAX_N)
    return fail(-3, "nnb_depth_invariant: bad arguments (need 0 < N <= %d)", NNB_INVARIANT_MAX_N);
  cudaError_t e = launch_depth_invariant(dp, dg, mask, N, w_dev, grad_scale, out_losses, g_dp, g_dg, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : cuda_fail(e, "nnb_depth_invariant");
}
int nnb_focal_fwd(const float* fx, const float* fy, int32_t order, float* cam, void* stream) {
  if (!fx || !cam || (order != 1 && order != 2)) return fail(-3, "nnb_focal_fwd: bad arguments (order must be 1 or 2)");
  cudaError_t e = launch_focal_fwd(fx, fy, order, cam, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : cuda_fail(e, "nnb_focal_fwd");
}
int nnb_focal_bwd(const float* fx, const float* fy, int32_t order, const float* g_cam, const float* g_kxy, float* g_fx, float* g_fy, void* stream) {
  if (!fx || !g_cam || !g_fx || ((fy == nullptr) != (g_fy == nullptr)) || (order != 1 && order != 2))
    return fail(-3, "nnb_focal_bwd: bad arguments (fy and g_fy both or neither; order 1 or 2)");
  cudaError_t e = launch_focal_bwd(fx, fy, order, g_cam, g_kxy, g_fx, g_fy, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : cuda_fail(e, "nnb_focal_bwd");
}
int nnb_pose_smooth(const float* t, int32_t V, const float* w_dev, float grad_scale, float* out2, float* loss_total, float* g_t, void* stream) {
  if (!t || !w_dev || !out2 || V < 2) return fail(-3, "nnb_pose_smooth: bad arguments (need V >= 2)");
  cudaError_t e = launch_pose_smooth(t, V, w_dev, grad_scale, out2, loss_total, g_t, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : cuda_fail(e, "nnb_pose_smooth");
}

int nnb_adam_step(float* p, const float* g, float* m, float* v, int64_t n, int32_t step, float lr, float b1, float b2, float eps,
                  void* stream) {
  if (!p || !g || !m || !v || n <= 0 || step < 1) return fail(-3, "nnb_adam_step: bad arguments");
  cudaError_t e = launch_adam(p, g, m, v, n, step, lr, b1, b2, eps, (cudaStream_t)stream);
  return e == cudaSuccess ? 0 : cuda_fail(e, "nnb_adam_step");
}

}  // extern "C"
