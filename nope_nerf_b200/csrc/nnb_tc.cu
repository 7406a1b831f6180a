// Tensor-core engine (NNB_ENGINE_TC), Hopper (sm_90a): the whole field of a 128-sample tile evaluated by one persistent CTA
// per SM.
//
// Every kernel is a template on the hidden width D (64 | 128 | 256), one instantiation per width, dispatched on WsLayout::D.
//
//   warps 0..7: two consumer warpgroups, each owning 64 sample rows of the tile.  Prologue: ray generation, sampling, the
//               63-column positional encoding -> E operand, direction encoding -> per-ray bias of rgb_layers.0.  Per layer the
//               warpgroup issues wgmma.m64n{D}k16 (m64n{D/2}k16 for the rgb hidden layer) with both operands in shared memory;
//               every logical product runs as three MMAs a_lo*b_hi + a_hi*b_lo + a_hi*b_hi (split-fp16, 22-bit operands, fp32
//               accumulation in registers) so results match the fp32 reference.  The epilogue (bias, ReLU, re-split into
//               hi | lo halves) writes the next layer's A operand IN PLACE: a warpgroup's MMAs read only its own 64 rows, and
//               they have completed (wgmma.wait_group 0) before the epilogue starts.  Density / colour heads, the per-sample
//               record, the fp32 training stash and the ReLU gate bits of the backward come out of the same registers.
//   warp 8   : weight producer (in the third warpgroup, whose registers go to the consumers) - cp.async.bulk of pre-imaged
//               fp16 hi | lo weight stages (all output rows x 16 k) from L2 into a 3-deep shared-memory ring, mbarrier tx-count;
//               a stage is released once both warpgroups' MMAs have read it.
//
// tc_points_fwd is the same kernel on explicit points (nnb_field_fwd with NNB_ENGINE_TC): the row's point and view direction are
// read instead of generated, the direction term of rgb_layers.0 is two more K-steps of its GEMM (every row has its own direction),
// the output is one float4 per point, and NNB_OCC_ONLY ends the tile after the density head.
//
// tc_march / tc_secant (nnb_ray_march, the geometry view's fused ray march) are the occupancy-only kernel again with points made from
// (ray origin, direction, depth) in the prologue and a reduction instead of an output: the first sign change of a ray's 128-step block,
// or the update of a hit ray's secant bracket (see MarchPtrs).
//
// nnb_geometry_frame (the geometry view of a frame in one call) runs that march on rays made per pixel (geo_rays), compacts the object
// rays (geo_compact), runs the points kernels on them with the row count read on the device (the DEVN forms of the bodies), and shades
// (geo_shade).
//
// The backward of this engine (tc_render_bwd) runs tc_dgrad (the same skeleton through the transposed weights, gated by the
// forward's ReLU bits) and tc_wgrad (the MLP weight-gradient GEMMs on the fp32 stash), between the compositing and ray adjoints of
// nnb_simt.cu.
//
// Shared-memory operand layout (no swizzle, "interleave"): element (row, k) of a [rows x K] fp16 operand lives at byte
// (k / 8) * rows * 16 + row * 16 + (k % 8) * 2: 8 x 8 core matrices of 128 contiguous bytes, SBO = 128 B between row groups,
// LBO = rows * 16 B between the two k-halves of one MMA.
#include "nnb_tc_common.cuh"
#include "nnb_march.cuh"
#include "nnb_frame.cuh"
#include <cuda.h>            // CUtensorMap (types only: the driver entry point is obtained at run time)
#include <cudaTypedefs.h>    // PFN_cuTensorMapEncodeTiled

cudaError_t launch_composite_fwd(const nnb_render_args& a, const SampleRec* recs, cudaStream_t st);
cudaError_t simt_render_bwd_with(const nnb_render_bwd_args& b, const WsLayout& L, cudaStream_t st, DgradFn dgrad, WgradFn wgrad);
cudaError_t launch_ray_reduce(const nnb_render_bwd_args& b, const float* rayred, cudaStream_t st);
cudaError_t launch_head_wgrad(const SmallJob* jobs, int njobs, size_t M, int D, float* part, size_t off, RedJob* R, cudaStream_t st,
                              const int* mcount = nullptr);

void nnb_prof_mark(cudaStream_t st);

namespace {

constexpr int TILE = 128;
constexpr int NST = 3;                      // weight ring depth
constexpr int N_GEMM = 10;                  // L0..L7, feature, rgb-hidden
struct StageDesc { int w_off, ldw, kcol0, kvalid, nrows, img_off; };
struct StageDescT { int w_off, ldw, coloff, nvalid, k0, kvalid, nrows, img_off; };
constexpr int N_THREADS = 384;              // two consumer warpgroups + the producer warpgroup (one thread of it issues the copies)

// sizes and shared-memory maps (bytes) of the field kernels at hidden width D
template <int D> struct Tc {
  static constexpr int LOG_D = D == 256 ? 8 : (D == 128 ? 7 : 6);
  static constexpr int KS = D / 16;                       // K-steps of a D-wide input
  static constexpr int STAGE_BYTES = D * 64;              // D output rows x 16 k x (hi + lo) 16-bit = one K-step of a D-wide layer
  // ---- forward stage table: the order in which weight stages are consumed for one tile (152 stages at D = 256) ----
  static constexpr int N_STAGES = 4 + 3 * KS + (4 + KS) + 3 * KS + KS + KS;
  static constexpr size_t IMG_BYTES = (size_t)(N_STAGES - KS) * STAGE_BYTES + KS * (STAGE_BYTES / 2);   // rgb hidden layer: D/2 rows
  // The producer's and the consumers' loop bounds both come from gemm_steps: K-steps (= weight stages) of GEMM g.  Points mode (pts)
  // appends the two direction K-steps of the rgb hidden layer; an occupancy-only tile (occ) ends after GEMM 7.
  static constexpr int enc_steps(int g) { return (g == 0 || g == 4) ? 4 : 0; }   // of them, the leading K-steps from the encoding operand E
  static constexpr int gemm_steps(int g, bool pts) { return enc_steps(g) + (g == 0 ? 0 : KS) + (pts && g == 9 ? 2 : 0); }
  static constexpr int n_gemm(bool occ) { return occ ? 8 : N_GEMM; }
  static constexpr int tile_stages(bool pts, bool occ) {
    int n = 0;
    for (int g = 0; g < n_gemm(occ); ++g) n += gemm_steps(g, pts);
    return n;
  }
  static_assert(tile_stages(false, false) == N_STAGES, "ray-mode stage count");
  // points mode: the direction stages (D/2 rows each) follow the ray-mode table and image
  static constexpr int N_STAGES_PTS = tile_stages(true, false), N_STAGES_OCC = tile_stages(true, true);
  static constexpr size_t IMG_PTS_BYTES = IMG_BYTES + 2 * (STAGE_BYTES / 2);
  static_assert(N_STAGES_PTS == N_STAGES + 2 && N_STAGES_OCC == N_STAGES - 2 * KS && IMG_PTS_BYTES == IMG_BYTES + 64 * D, "points-mode stages");
  static constexpr int SM_AHI = 0, SM_ALO = D * 256, SM_EHI = 2 * D * 256, SM_ELO = SM_EHI + 16384, SM_W = SM_ELO + 16384;
  static constexpr int SM_BIAS = SM_W + NST * STAGE_BYTES;
  static constexpr int BIAS_FLOATS = 8 * D + D + D + 3 * (D / 2) + 4;   // trunk, feat, w_sigma, W_rgb, (b_sigma, b_rgb[3])
  static constexpr int SM_RAYB = SM_BIAS + ((BIAS_FLOATS * 4 + 127) / 128) * 128;
  // per warpgroup: per-ray bias [RAYB_RAYS][D/2] + direction encodings [RAYB_RAYS][32].  A 64-row block that starts at a multiple of 64
  // overlaps at most ceil(63 / S) + 1 rays: 5 at the smallest S of this engine (16), 2 for S >= 64
  static constexpr int RAYB_RAYS = 5;
  static constexpr int RAYB_FLOATS = RAYB_RAYS * (D / 2) + RAYB_RAYS * 32;
  static constexpr int SM_BAR = SM_RAYB + 2 * RAYB_FLOATS * 4;
  static constexpr int SM_TOTAL = SM_BAR + 2 * NST * 8;
  // ---- data-gradient chain (176 transposed stages at D = 256) ----
  static constexpr int N_STAGES_T = D / 32 + D / 32 + KS + 7 * KS + KS + KS;
  static constexpr size_t IMG_T_BYTES = (size_t)34 * D * D + (size_t)576 * D;
  // The producer's and the consumers' bounds of the chain come from dg_steps: K-steps (= transposed stages) of chain GEMM j: 0 g_de,
  // 1 g_feat, 2 g_h7 (W_feat), 3 + i (i = 0..6) g_h(6 - i) = dY_(7 - i) W_(7 - i), 10 the encoding slice of layer 4, 11 the encoding
  // gradient of layer 0.  An occupancy-only chain (occ, nnb_field_vjp) starts at g_h7 = g_s w_sigma: GEMMs 0..2 (the colour prefix of the
  // stage table) have no stages, and it walks the table from dg_first_stage(true) on.
  static constexpr int N_DG_GEMM = 12;
  static constexpr int dg_steps(int j, bool occ) { return j < 2 ? (occ ? 0 : D / 32) : (j == 2 && occ ? 0 : KS); }
  static constexpr int dg_tile_stages(bool occ) {
    int n = 0;
    for (int j = 0; j < N_DG_GEMM; ++j) n += dg_steps(j, occ);
    return n;
  }
  static constexpr int dg_first_stage(bool occ) { return dg_tile_stages(false) - dg_tile_stages(occ); }
  static constexpr size_t IMG_T_PREFIX_BYTES = (size_t)(D / 32) * 32 * 64 + (size_t)(D / 32 + KS) * STAGE_BYTES;   // g_de, g_feat, W_feat
  static_assert(dg_tile_stages(false) == N_STAGES_T && dg_first_stage(true) == D / 16 + KS, "chain stage count");
  static_assert(dg_steps(3, false) == KS && dg_steps(9, false) == KS && dg_steps(3, true) == KS && dg_steps(9, true) == KS,
                "the trunk layers of the chain share one K-step count");
  static constexpr int DG_AHI = 0, DG_ALO = D * 256, DG_W = 2 * D * 256, DG_GENC = DG_W + NST * STAGE_BYTES;
  static constexpr int DG_SMALL = DG_GENC + 2 * 64 * 64 * 4;     // W_rgb [3][D/2] | w_sigma [D]
  static constexpr int DG_GYC = DG_SMALL + (5 * D / 2) * 4;      // per row: d/d(rgb logits), d/d density logit
  static constexpr int DG_BAR = DG_GYC + 128 * 4 * 4;
  static constexpr int DG_TOTAL = DG_BAR + 2 * NST * 8;
  static_assert(SM_TOTAL <= 232448 && DG_TOTAL <= 232448, "shared memory budget");
  // a field query's workspace is sized like a render's: the direction stages spill into the transposed-image region behind the
  // forward image, which only the backward uses
  static_assert(IMG_PTS_BYTES <= (IMG_BYTES + 255) / 256 * 256 + IMG_T_BYTES, "points-mode weight image fits the workspace");
  static_assert(RAYB_FLOATS >= D / 2, "points mode keeps the bias of the rgb hidden layer in the per-ray bias area");
};
static_assert(Tc<256>::N_STAGES == 152 && Tc<256>::SM_BIAS == 212992 && Tc<256>::BIAS_FLOATS == 2948 && Tc<256>::N_STAGES_T == 176 &&
              Tc<256>::IMG_T_BYTES == (size_t)136 * 16384 + 8 * 2048 + 32 * 4096 && Tc<256>::DG_GENC == 180224, "D = 256 layout");

// stage tables, one per width
__constant__ StageDesc c_stages_256[Tc<256>::N_STAGES_PTS], c_stages_128[Tc<128>::N_STAGES_PTS], c_stages_64[Tc<64>::N_STAGES_PTS];
__constant__ StageDescT c_stages_t_256[Tc<256>::N_STAGES_T], c_stages_t_128[Tc<128>::N_STAGES_T], c_stages_t_64[Tc<64>::N_STAGES_T];
template <int D> __device__ __forceinline__ const StageDesc& stage(int s) {
  if constexpr (D == 256) return c_stages_256[s]; else if constexpr (D == 128) return c_stages_128[s]; else return c_stages_64[s];
}
template <int D> __device__ __forceinline__ const StageDescT& stage_t(int s) {
  if constexpr (D == 256) return c_stages_t_256[s]; else if constexpr (D == 128) return c_stages_t_128[s]; else return c_stages_t_64[s];
}

using namespace tcu;

// ---- weight imaging: fp32 (out,in) matrices -> per-stage shared-memory images (hi | lo) --------
template <int D, bool BF16>
__device__ __forceinline__ void prep_stage(const float* __restrict__ w, unsigned char* __restrict__ img) {
  const StageDesc sd = stage<D>(blockIdx.x);
  unsigned char* hi = img + sd.img_off;       // [k-octet 0..1][nrows][8] fp16 (bf16)
  unsigned char* lo = hi + sd.nrows * 32;
  for (int idx = threadIdx.x; idx < sd.nrows * 2; idx += blockDim.x) {
    const int n = idx % sd.nrows, ko = idx / sd.nrows;
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int k = sd.kcol0 + ko * 8 + j;
      v[j] = (k < sd.kvalid) ? __ldg(w + sd.w_off + (size_t)n * sd.ldw + k) : 0.f;
    }
    if constexpr (BF16) split_store8_bf16(v, hi + ko * sd.nrows * 16 + n * 16, lo + ko * sd.nrows * 16 + n * 16);
    else split_store8(v, hi + ko * sd.nrows * 16 + n * 16, lo + ko * sd.nrows * 16 + n * 16);
  }
}
template <int D>
__global__ void tc_prep_weights(const float* __restrict__ w, unsigned char* __restrict__ img) { prep_stage<D, false>(w, img); }
// the same stages as bf16 hi | lo (the tangent chain of nnb_field_hvp_tc, whose operands span the range of gradients)
template <int D>
__global__ void tc_prep_weights_bf16(const float* __restrict__ w, unsigned char* __restrict__ img) { prep_stage<D, true>(w, img); }

// fp32 [sample][feature] stash, layout of nnb_simt.cu, and the ReLU gate bits of h0..h7 and hr (gate_bits_off).  This and DgPtrs are
// __grid_constant__ kernel parameters: indexed by layer in parameter space, not copied to local memory (which would also leave the
// pointers generic instead of global)
struct TcStash { float *h[8], *feat, *hr, *enc, *denc; unsigned char* gates; };

// this thread's NB ReLU gate bits of one tile and layer (NB = 16 | 32 | 64 | 128, see gate_bits_off): one vector access.  In
// registers, bit b of the set is bit 31 - b % 32 of word b / 32 (a 16-bit set is loaded into the upper half of its word).  Stored
// like the stash (st.global.cs, evict-first).
template <int NB> __device__ __forceinline__ void store_gates(unsigned char* p, const uint32_t* w) {
  if constexpr (NB == 128) __stcs(reinterpret_cast<uint4*>(p), make_uint4(w[0], w[1], w[2], w[3]));
  else if constexpr (NB == 64) __stcs(reinterpret_cast<uint2*>(p), make_uint2(w[0], w[1]));
  else if constexpr (NB == 32) __stcs(reinterpret_cast<unsigned int*>(p), w[0]);
  else __stcs(reinterpret_cast<unsigned short*>(p), (unsigned short)w[0]);
}
template <int NB> __device__ __forceinline__ void load_gates(const unsigned char* p, uint32_t* w) {
  if constexpr (NB == 128) { const uint4 v = __ldg(reinterpret_cast<const uint4*>(p)); w[0] = v.x; w[1] = v.y; w[2] = v.z; w[3] = v.w; }
  else if constexpr (NB == 64) { const uint2 v = __ldg(reinterpret_cast<const uint2*>(p)); w[0] = v.x; w[1] = v.y; }
  else if constexpr (NB == 32) w[0] = __ldg(reinterpret_cast<const unsigned int*>(p));
  else w[0] = (uint32_t)__ldg(reinterpret_cast<const unsigned short*>(p)) << 16;
}
// shifts the gate bit of v (a ReLU output, so v >= 0 or -0) in at the bottom of w: w = (w << 1) | (v > 0).  0 - v is negative exactly
// when v > 0 (0 - (-0) = +0), so the bit is its sign: one FADD and one funnel shift per bit.
__device__ __forceinline__ uint32_t push_gate(uint32_t w, float v) { return __funnelshift_l(__float_as_uint(0.f - v), w, 1); }

__device__ __forceinline__ void split2_bf16(float a, float b, uint32_t& hi, uint32_t& lo) {
  __nv_bfloat162 hh = __floats2bfloat162_rn(a, b);
  hi = *reinterpret_cast<uint32_t*>(&hh);
  __nv_bfloat162 ll = __floats2bfloat162_rn(a - __uint_as_float(hi << 16), b - __uint_as_float(hi & 0xffff0000u));
  lo = *reinterpret_cast<uint32_t*>(&ll);
}

__device__ __forceinline__ void row_geometry_tc(const nnb_render_args& a, size_t m, size_t M, Ray& ray, float& z, float p[3]) {
  const size_t mm = m < M ? m : M - 1;
  const int n = (int)(mm / a.S), i = (int)(mm % a.S);
  setup_ray(a, n, ray);
  z = sample_z(a, n, i);
  sample_point(a, ray, z, p);
}

// x, opaque to the compiler: an address formed from it is computed where it is used, not once per tile and held (or spilled) across the MMAs
__device__ __forceinline__ uint32_t computed_here(uint32_t x) { asm volatile("" : "+r"(x)); return x; }

__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// ---- fused ray marching (nnb_ray_march): tc_march / tc_secant are tc_fwd_body with a front end that makes each row's point from
// (origin, direction, depth) and a back end that reduces the tile's occupancies instead of writing them (nnb_march.cuh) ----
static_assert(TILE == MARCH_BLOCK, "a march tile is one block of a ray's steps");

// nnb_render_frame (tc_frame): a tile is 4 ray-chunks x 32 rows, composited by frame_step (nnb_frame.cuh) in the tile's back end.
// workspace row of tile row `row` of a frame tile: sample i = 32 k + row % 32 of ray list[4 tile + row / 32].  Ray-chunks past the end of
// the list repeat its last ray and rows past the ray's last sample evaluate that sample; frame_step ignores both.
__device__ __forceinline__ size_t frame_sample(const nnb_render_args& a, const FramePtrs& f, int tile, int row, int n_live) {
  const int slot = min(4 * tile + row / 32, n_live - 1);
  const int n = f.list ? f.list[slot] : slot;
  return (size_t)n * a.S + min(32 * f.k + row % 32, a.S - 1);
}
// nnb_render_frame_bwd (tc_frame_stash, tc_dgrad_frame): (ray, sample) of row m of chunk k's stash (row 32 n + j: sample 32 k + j of ray n;
// rows past the last ray take its last ray, rows past the ray's last sample that sample; their cotangent is zero).  32-bit: m < 32 N + 128.
__device__ __forceinline__ int2 chunk_sample(const nnb_render_args& a, int k, size_t m) {
  return make_int2(min((int)(m >> 5), a.N - 1), min(32 * k + (int)(m & 31), a.S - 1));
}
// nnb_render_frame_train_bwd_tmin (the live-list forms, DEVN): row m of round k's stash is sample 32 k + m % 32 of ray list[m / 32], over
// the n_live rays of the list (rows past the last slot take its ray, rows past the ray's last sample that sample; their cotangent is zero)
__device__ __forceinline__ int2 live_sample(const nnb_render_args& a, int k, const int* list, int n_live, size_t m) {
  return make_int2(list[min((int)(m >> 5), n_live - 1)], min(32 * k + (int)(m & 31), a.S - 1));
}
// row_geometry_tc of a sample (ray, index)
__device__ __forceinline__ void sample_geometry(const nnb_render_args& a, int2 ni, Ray& ray, float& z, float p[3]) {
  setup_ray(a, ni.x, ray);
  z = sample_z(a, ni.x, ni.y);
  sample_point(a, ray, z, p);
}
__device__ __forceinline__ void chunk_geometry(const nnb_render_args& a, int k, size_t m, Ray& ray, float& z, float p[3]) {
  sample_geometry(a, chunk_sample(a, k, m), ray, z, p);
}

// ---- nnb_render_fwd_tmin / nnb_render_bwd_tmin (early ray termination on the per-sample stash, tensor-core engine) ----------------
// Round k evaluates chunk k of the rays {n : c_n > k}, listed in increasing n by frame_live_list into lists[k] ([C][N]) with their count
// in counts[k]; the forward writes c_n (FramePtrs::chunks) as C while a ray is live and k + 1 when it stops in round k, so the lists of
// the rounds after round 0 (whose list is every ray whatever chunks holds) come from the chunk counts the rounds before wrote.  Every
// round's training stash goes into one packed stash: round k's rows start at R_k = sum over j < k of 128 ceil(count_j / 4) (each round
// padded to the 128-row tile, the unit of the gate bits), and row R_k + 32 slot + j is sample 32 k + j of ray lists[k][slot].  counts[C]
// holds R_C / 32, the stash's row count for the weight-gradient stage.  Every count is clamped to 0..N where it is read, so every row
// index stays below the packed stash's C 128 ceil(N / 4) rows.
__device__ __forceinline__ size_t stash_round_base(const int* counts, int k, int N) {
  size_t r = 0;
  for (int j = 0; j < k; ++j) r += (size_t)128 * ((frame_live_count(counts + j, N) + 3) / 4);
  return r;
}
// (ray, sample) of packed row m: the round whose rows hold m (the last round past them), the slot's ray (padding slots take the list's
// last ray, rows past the ray's last sample that sample: their cotangent is zero)
__device__ __forceinline__ int2 stash_row_sample(const nnb_render_args& a, const int* lists, const int* counts, int C, size_t m) {
  size_t r = 0;
  int k = 0;
  for (; k < C - 1; ++k) {
    const size_t rows = (size_t)128 * ((frame_live_count(counts + k, a.N) + 3) / 4);
    if (m < r + rows) break;
    r += rows;
  }
  const int slot = min((int)((m - r) >> 5), max(frame_live_count(counts + k, a.N) - 1, 0));
  return make_int2(min(max(lists[(size_t)k * a.N + slot], 0), a.N - 1), min(32 * k + (int)(m & 31), a.S - 1));
}
// slot of ray n in a round's list (increasing n): the first slot whose ray is not below n, clamped to the list
__device__ __forceinline__ int stash_slot(const int* list, int count, int n) {
  int lo = 0, hi = count;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (list[mid] < n) lo = mid + 1; else hi = mid;
  }
  return min(lo, max(count - 1, 0));
}

// Back end of forward round f.k (f.list = lists[k], f.count = counts + k): one warp per slot, frame_step's arithmetic on the (r, g, b, a)
// of the round's packed records, from the ray's carry and lane partials of the rounds before.  Lane 0 stores the carry, its checkpoint
// ckpt[k][n] (transmittance into chunk k + 1) and c_n: k + 1 when the ray stops (frame_step's rule), C while it stays live.
__global__ void stash_frame_step(nnb_render_args a, const __grid_constant__ FramePtrs f, const SampleRec* __restrict__ rec,
                                 float* __restrict__ ckpt, int C) {
  const int lane = threadIdx.x & 31, slot = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (slot >= frame_live_count(f.count, a.N)) return;
  const int n = f.list[slot];
  const int i = 32 * f.k + lane;
  const bool valid = i < a.S;
  float4 me = make_float4(0.f, 0.f, 0.f, 0.f);
  float z = 0.f, alpha = 0.f;
  if (valid) {
    const SampleRec r = rec[stash_round_base(f.count - f.k, f.k, a.N) + (size_t)slot * 32 + lane];
    me = make_float4(r.r, r.g, r.b, r.a);
    z = sample_z(a, n, i);
    alpha = composite_alpha(a, i, me.w, z, [&] { return sample_z(a, n, i + 1); });
  }
  float* part = f.part + (size_t)n * 160 + lane;
  float carry = 1.f, C0 = 0.f, C1 = 0.f, C2 = 0.f, Dist = 0.f, acc = 0.f;
  if (f.k > 0) { carry = f.carry[n]; C0 = part[0]; C1 = part[32]; C2 = part[64]; Dist = part[96]; acc = part[128]; }
  composite_chunk(alpha, valid, me.x, me.y, me.z, z, lane, carry, C0, C1, C2, Dist, acc);
  part[0] = C0; part[32] = C1; part[64] = C2; part[96] = Dist; part[128] = acc;
  if (lane == 0) {
    f.carry[n] = carry;
    if (f.k + 1 < C) ckpt[(size_t)f.k * a.N + n] = carry;
    f.chunks[n] = carry < f.t_min || 32 * (f.k + 1) >= a.S ? f.k + 1 : C;
  }
}

// Compositing adjoint of the packed stash, one warp per ray: frame_chunk_adjoint_live's statements for chunks c_n - 1 .. 0, the suffix
// carry starting at 0 in the ray's last chunk and held in a register between chunks.  Warps N .. N + 3 C - 1 zero the cotangents of
// round (w - N) / 3's padding slots count .. 4 ceil(count / 4) - 1, so those rows give zero dY.  Thread 0 stores counts[C] = R_C / 32.
__global__ void stash_chunk_adjoint(nnb_render_bwd_args b, const __grid_constant__ FrameBwdPtrs f, const int* __restrict__ chunks,
                                    const int* __restrict__ lists, int* __restrict__ counts) {
  const nnb_render_args& a = b.fwd;
  const int C = f.rounds;
  const int lane = threadIdx.x & 31, w = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (w == 0 && lane == 0) counts[C] = (int)(stash_round_base(counts, C, a.N) / 32);
  if (w >= a.N) {
    const int k = (w - a.N) / 3;
    if (k >= C) return;
    const int cnt = frame_live_count(counts + k, a.N), slot = cnt + (w - a.N) % 3;
    if (slot < (cnt + 3) / 4 * 4) f.gs[stash_round_base(counts, k, a.N) + (size_t)slot * 32 + lane] = make_float4(0.f, 0.f, 0.f, 0.f);
    return;
  }
  const int n = w;
  Ray ray; setup_ray(a, n, ray);
  float gD = b.g_depth_pred ? __ldg(b.g_depth_pred + n) : 0.f;
  if ((a.flags & NNB_EVAL) && (a.flags & NNB_NORMALISE)) gD = gD / ray.nrm;
  const float gC0 = __ldg(b.g_rgb + 3 * n), gC1 = __ldg(b.g_rgb + 3 * n + 1), gC2 = __ldg(b.g_rgb + 3 * n + 2);
  const float gsum = (a.flags & NNB_WHITE_BG) ? (gC0 + gC1 + gC2) : 0.f;
  float carry_s = 0.f;
  for (int k = frame_ray_chunks(chunks, n, C) - 1; k >= 0; --k) {
    const int slot = stash_slot(lists + (size_t)k * a.N, frame_live_count(counts + k, a.N), n);
    const size_t m = stash_round_base(counts, k, a.N) + (size_t)slot * 32 + lane;
    const int i = 32 * k + lane;
    const bool valid = i < a.S;
    const SampleRec me = valid ? f.rec[m] : SampleRec{0, 0, 0, 0, 0, 0, 0, 0};
    float alpha = 0.f, df = 1.f;   // df = d alpha / d a
    if (valid) {
      alpha = composite_alpha(a, i, me.a, me.z, [&] { return sample_z(a, n, i + 1); });
      if (a.flags & NNB_DIST_ALPHA) {
        if (i >= a.S - 1) df = 0.f;
        else { const float delta = __fsub_rn(sample_z(a, n, i + 1), me.z); df = delta * expf(-me.a * delta); }
      }
    }
    const float carry = k > 0 ? f.ckpt[(size_t)(k - 1) * a.N + n] : 1.f;
    f.gs[m] = composite_chunk_bwd<false>(alpha, valid, me.r, me.g, me.b, me.z, df, lane, carry, gC0, gC1, gC2, gD, gsum, carry_s);
  }
}

// frame_ray_acc_live's sums on the packed stash, one warp per ray: the terms of chunks c_n - 1 .. 0 added in that order to lane partials
// that start at 0, stored once for frame_ray_finish
__global__ void stash_ray_acc(nnb_render_args a, const __grid_constant__ FrameBwdPtrs f, const int* __restrict__ chunks,
                              const int* __restrict__ lists, const int* __restrict__ counts) {
  const int lane = threadIdx.x & 31, n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (n >= a.N) return;
  float v[9];
#pragma unroll
  for (int c = 0; c < 9; ++c) v[c] = 0.f;
  for (int k = frame_ray_chunks(chunks, n, f.rounds) - 1; k >= 0; --k) {
    if (32 * k + lane >= a.S) continue;
    const int slot = stash_slot(lists + (size_t)k * a.N, frame_live_count(counts + k, a.N), n);
    const size_t m = stash_round_base(counts, k, a.N) + (size_t)slot * 32 + lane;
    const float4 g = f.gp[m], dv = f.gv[m];
    const float z = f.rec[m].z;
    v[0] += g.x; v[1] += g.y; v[2] += g.z;
    v[3] += z * g.x; v[4] += z * g.y; v[5] += z * g.z;
    v[6] += dv.x; v[7] += dv.y; v[8] += dv.z;
  }
  float* part = f.raypart + (size_t)n * 288 + lane;
#pragma unroll
  for (int c = 0; c < 9; ++c) part[32 * c] = v[c];
}

// MODE FWD_RAYS (tc_field_fwd): recs [Mpad], out unused.  FWD_POINTS: explicit points (tc_points_fwd): a.pts / a.dirs [M][3] ->
// out [M] = (r, g, b, a), or (0, 0, 0, a) with NNB_OCC_ONLY; nothing is stashed and recs is not written.  M = a.N there, so point indices
// are 32-bit.  FWD_VJP (tc_points_vjp_fwd, nnb_field_vjp): FWD_POINTS that also writes recs [Mpad] and the ReLU gate bits st.gates of
// the chain that follows (h0..h7, and the rgb hidden layer unless NNB_OCC_ONLY); out may be NULL; no fp32 stash.  FWD_MARCH /
// FWD_SECANT (tc_march / tc_secant): occupancy-only tiles of points made from q; n_tiles (and M, the hit count of tc_secant) are read
// from *q.count when the kernel starts and fixed from then on.
//   FWD_MARCH: tile = 128 consecutive steps of one ray; march_scan reduces them.
//   FWD_SECANT: tile = 128 hit rays, evaluated q.n_secant times in a row at the secant iterate of each ray's bracket, which the thread
//   that owns the row's logit then updates in q.brk1 (pass 0 reads q.brk0).  A row's prologue threads and that thread sit in the same
//   warpgroup, whose barrier at the top of the tile loop orders the update before the next pass reads it.
// DEVN (FWD_POINTS / FWD_VJP of nnb_geometry_frame): M = *q.count points, read when the kernel starts like FWD_SECANT's count; the
// launch is sized for the largest count and a CTA without a tile leaves at once.
// FWD_FRAME (tc_frame): FWD_RAYS on the rows frame_sample gives (M = N S), with ray-chunks of 32 rows in place of whole rays in the per-ray
// bias; nothing is stashed.  The colour head puts each row's (r, g, b, a) in this warpgroup's rows of the E operand (last read by layer
// 4) and frame_step composites them.  n_tiles is read from *fr.count (ray-chunks, 4 per tile) when the kernel starts, as in FWD_MARCH.
// FWD_CHUNK (tc_frame_stash, nnb_render_frame_bwd): FWD_RAYS with the training stash on the rows of chunk fr.k of every ray (M = 32 N,
// row m is sample chunk_sample(a, fr.k, m) of its ray), with ray-chunks of 32 rows in place of whole rays in the per-ray bias as in FWD_FRAME; records,
// stash and gate bits are indexed by the row.  With DEVN (tc_frame_stash_live): the rows of the rays of round fr.k's live list fr.list
// (live_sample), M = 32 n_live and n_tiles = ceil(n_live / 4) with n_live = *fr.count clamped to 0..N, read when the kernel starts; the
// launch is sized for N and a CTA without a tile leaves at once.
// FWD_GRAD (tc_points_grad_fwd, nnb_field_grad): FWD_VJP that also writes the fp32 training stash st of every row of every tile (rows
// past M hold the last point's values): h0..h7, feat, hr and enc as FWD_RAYS does, and denc per point (the direction encoding of
// a.dirs[m], or of the ones), which is a per-row operand of rgb_layers.0 here.  With NNB_OCC_ONLY the colour part (feat, hr, denc) is not
// written.
// FWD_PACK (tc_stash_pack, nnb_render_fwd_tmin): FWD_CHUNK with DEVN on round fr.k's list (fr.list, fr.count = counts + k), into the
// packed stash of nnb_frame.cuh: its rows go to packed rows R_k + m (R_k from counts[0 .. k - 1], read when the kernel starts), its gate
// bits to tiles R_k / 128 + tile of a stash of M rows.
// FWD_TANGENT (tc_points_tangent, nnb_field_hvp_tc): the tangent chain of the density logit along u on the trunk of an occupancy-only
// FWD_VJP forward: the prologue puts e' = J_enc(p) u in E (u = (*out)[m], read, never written; rows past M have u = 0), every layer is
// the bias-free z'_l = W_l x'_{l-1} ([h'3 | e'] into layer 4), gated with the forward's bits st.gates (read as tc_dgrad reads them)
// instead of a ReLU, and the tile ends after layer 7.  Operands are bf16 hi | lo (wimg is the bf16 image of the occupancy-only stages),
// because tangents span the range of gradients.  e' and h'0..h'7 of every row of every tile go to st.enc / st.h with the stash's
// streaming stores; nothing else is written.
enum : int { FWD_RAYS = 0, FWD_POINTS = 1, FWD_MARCH = 2, FWD_SECANT = 3, FWD_VJP = 4, FWD_FRAME = 5, FWD_GRAD = 6, FWD_TANGENT = 7,
             FWD_CHUNK = 8, FWD_PACK = 9 };
template <int D, int MODE, bool DEVN = false>
__device__ __forceinline__ void tc_fwd_body(const nnb_render_args& a, const unsigned char* __restrict__ wimg, SampleRec* __restrict__ recs,
                                            float4* __restrict__ out, const TcStash& st, const MarchPtrs& q, size_t M, int n_tiles,
                                            int stash, const FramePtrs& fr = FramePtrs{}) {
  using T = Tc<D>;
  constexpr bool PACK = MODE == FWD_PACK;
  constexpr bool FRAME = MODE == FWD_FRAME, GRAD = MODE == FWD_GRAD, TAN = MODE == FWD_TANGENT, CHUNK = MODE == FWD_CHUNK || PACK;
  static_assert(!PACK || DEVN, "the packed stash takes its rows from the round's list");
  constexpr bool PTS = MODE != FWD_RAYS && !FRAME && !CHUNK, MARCH = MODE == FWD_MARCH || MODE == FWD_SECANT, VJP = MODE == FWD_VJP || GRAD;
  constexpr bool XPTS = MODE == FWD_POINTS || VJP;   // points read from a.pts
  static_assert(!DEVN || XPTS || CHUNK, "a device count of explicit points or of a frame round's rays");
  if constexpr ((PTS && !GRAD && !TAN) || FRAME) stash = 0;
  if constexpr (GRAD || TAN || CHUNK) stash = 1;
  int n_live = 0;   // FWD_FRAME, FWD_CHUNK with DEVN: ray-chunks of this round
  if constexpr (FRAME) {
    n_live = fr.count ? *fr.count : a.N;
    n_tiles = (n_live + 3) / 4;
    if ((int)blockIdx.x >= n_tiles) return;   // a CTA without a tile leaves before any barrier exists
  }
  if constexpr (CHUNK && DEVN) {
    n_live = frame_live_count(fr.count, a.N);
    n_tiles = (n_live + 3) / 4;
    if ((int)blockIdx.x >= n_tiles) return;   // a CTA without a tile leaves before any barrier exists
  }
  const size_t mo = PACK ? stash_round_base(fr.count - fr.k, fr.k, a.N) : 0;   // FWD_PACK: packed row of the round's row 0
  const bool gates = !TAN && (VJP || stash);   // the ReLU gate bits are stored
  if constexpr (MARCH || (DEVN && !CHUNK)) {
    if (q.count) {
      const int c = *q.count;
      M = (size_t)c;
      n_tiles = MODE == FWD_MARCH ? c : (c + TILE - 1) / TILE;
    }
    if ((int)blockIdx.x >= n_tiles) return;   // a CTA without a tile leaves before any barrier exists
  }
  const bool occ = MARCH || TAN || (PTS && (a.flags & NNB_OCC_ONLY));
  constexpr int SM_AHI = T::SM_AHI, SM_ALO = T::SM_ALO, SM_EHI = T::SM_EHI, SM_ELO = T::SM_ELO, SM_W = T::SM_W, SM_BIAS = T::SM_BIAS;
  constexpr int SM_RAYB = T::SM_RAYB, SM_BAR = T::SM_BAR, BIAS_FLOATS = T::BIAS_FLOATS, RAYB_FLOATS = T::RAYB_FLOATS;
  constexpr int STAGE_BYTES = T::STAGE_BYTES, N_STAGES = T::N_STAGES, DR = D / 2;
  constexpr int B_FEAT0 = 8 * D, W_SIG0 = 9 * D, W_RGB0 = 10 * D, B_SIG0 = 10 * D + 3 * DR;   // s_bias sections
  extern __shared__ __align__(1024) unsigned char smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* s_bias = reinterpret_cast<float*>(smem + SM_BIAS);
  const uint32_t bar0 = smem_u32(smem + SM_BAR);
  auto FULL = [&](uint32_t i) { return bar0 + 8u * i; };
  auto EMPTY = [&](uint32_t i) { return bar0 + 8u * (NST + i); };

  if (threadIdx.x == 0) {
    for (int i = 0; i < NST; ++i) { mbar_init(FULL(i), 1); mbar_init(EMPTY(i), 2); }   // EMPTY: one arrival per warpgroup
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  {  // biases / small heads -> shared (weights are constant for the launch)
    const float* w = a.weights;
    for (int i = threadIdx.x; i < BIAS_FLOATS; i += blockDim.x) {
      float v;
      if (i < B_FEAT0) v = __ldg(w + nnb::b_off(D, i >> T::LOG_D) + (i & (D - 1)));
      else if (i < W_SIG0) v = __ldg(w + nnb::B_FEAT(D) + (i - B_FEAT0));
      else if (i < W_RGB0) v = __ldg(w + nnb::W_SIG(D) + (i - W_SIG0));
      else if (i < B_SIG0) v = __ldg(w + nnb::W_RGB(D) + (i - W_RGB0));
      else if (i == B_SIG0) v = __ldg(w + nnb::B_SIG(D));
      else v = __ldg(w + nnb::B_RGB(D) + (i - (B_SIG0 + 1)));
      s_bias[i] = v;
    }
  }
  __syncthreads();
  const int my_tiles = (n_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;   // tiles blockIdx.x, + gridDim.x, ...
  // tile evaluations of this CTA: the producer's and the consumers' common bound.  tc_secant evaluates each tile n_secant times in a row.
  const int my_evals = MODE == FWD_SECANT ? my_tiles * q.n_secant : my_tiles;

  if (warp >= 8) {
    // =============================== weight producer ===============================
    // registers move from the producer warpgroup to the consumers: 40 + 2 x 232 per SM sub-partition fits the register file
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
    if (warp == 8 && lane == 0) {
      uint32_t slot = 0, phase = 0;
      const int n_st = PTS ? (occ ? T::N_STAGES_OCC : T::N_STAGES_PTS) : N_STAGES;
      for (int t = 0; t < my_evals; ++t)
        for (int s = 0; s < n_st; ++s) {
          const uint32_t bytes = (uint32_t)stage<D>(s).nrows * 64u;
          mbar_wait(EMPTY(slot), phase ^ 1u);                 // both warpgroups released this slot
          mbar_expect_tx(FULL(slot), bytes);
          bulk_g2s(smem_u32(smem + SM_W + slot * STAGE_BYTES), wimg + stage<D>(s).img_off, bytes, FULL(slot));
          if (++slot == NST) { slot = 0; phase ^= 1u; }
        }
    }
    return;
  }
  // =============================== consumer warpgroups ===============================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
  const int wg = warp >> 2, tl = threadIdx.x & 127;
  const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);     // tile rows r0 and r0 + 8 hold this thread's accumulator fragment
  const int c0 = (lane & 3) * 2;                               // its column pair inside every 8-column block
  float* rayb = reinterpret_cast<float*>(smem + SM_RAYB) + wg * RAYB_FLOATS;
  const uint32_t a_hi = smem_u32(smem + SM_AHI) + wg * 1024, a_lo = smem_u32(smem + SM_ALO) + wg * 1024;
  const uint32_t e_hi = smem_u32(smem + SM_EHI) + wg * 1024, e_lo = smem_u32(smem + SM_ELO) + wg * 1024;
  const uint32_t w_base = smem_u32(smem + SM_W);
  const uint32_t bar_id = 1u + (uint32_t)wg;
  auto wg_sync = [&]() { asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory"); };
  constexpr int RAYB_DE = T::RAYB_RAYS * DR;   // direction encodings after the per-ray biases
  uint32_t slot = 0, phase = 0;
  float acc[D / 2];
  if constexpr (XPTS) {   // b_rgbh is a plain bias here; visible after the tile's first barrier
    if (tl < DR) rayb[tl] = __ldg(a.weights + nnb::B_RGBH(D) + tl);
  }
  const int n_gemm = T::n_gemm(occ);

  for (int t = 0; t < my_evals; ++t) {
    const int tile = blockIdx.x + (MODE == FWD_SECANT ? t / q.n_secant : t) * gridDim.x;
    const size_t mt = (size_t)tile * TILE;
    // sample index of this warpgroup's first row inside its ray: row rl reads the bias of the block's ray (ray_off() + rl) / S.  Computed
    // where it is used, not held across the MMAs.
    auto ray_off = [&]() { return (int)((mt + (size_t)wg * 64) % (size_t)a.S); };
    // rows per ray of the per-ray bias: a frame tile's ray-chunks take the place of rays
    auto ray_len = [&]() { return FRAME || CHUNK ? 32 : a.S; };
    wg_sync();   // the previous tile's epilogue (a frame tile: its frame_step) is done with the per-ray bias buffer and E
    {
      const int off0 = PTS || FRAME || CHUNK ? 0 : ray_off();
      // ---- prologue: thread (row rl, part) writes encoding columns [32 part, 32 part + 32) of its row ----
      const int rl = tl & 63, part = tl >> 6, row = wg * 64 + rl;
      const size_t m = FRAME ? frame_sample(a, fr, tile, row, n_live) : mt + row;
      Ray ray; float z, p[3];
      if constexpr (MODE == FWD_MARCH) {
        const int ray = q.list ? q.list[tile] : tile;
        march_point(q, ray, march_depth(q.near, __ldg(q.far + ray), __ldg(q.frac + min(q.block * TILE + row, q.n_steps - 1))), p);
      } else if constexpr (MODE == FWD_SECANT) {
        const uint32_t mp = tile * (uint32_t)TILE + row;
        p[0] = p[1] = p[2] = 0.f;   // rows past the last hit ray are evaluated and ignored
        if (mp < (uint32_t)M) {
          const int ray = q.list[mp];
          const float depth = secant_depth((t % q.n_secant == 0 ? q.brk0 : q.brk1)[ray]);
#pragma unroll
          for (int c = 0; c < 3; ++c) p[c] = __fadd_rn(__ldg(q.ray0 + (size_t)ray * 3 + c), __fmul_rn(depth, __ldg(q.dir + (size_t)ray * 3 + c)));
        }
      } else if constexpr (PTS) {
        const uint32_t mm = min(tile * (uint32_t)TILE + row, (uint32_t)M - 1u);
#pragma unroll
        for (int c = 0; c < 3; ++c) p[c] = __ldg(a.pts + (size_t)mm * 3 + c);
      } else {
        if constexpr (CHUNK && DEVN) sample_geometry(a, live_sample(a, fr.k, fr.list, n_live, m), ray, z, p);
        else if constexpr (CHUNK) chunk_geometry(a, fr.k, m, ray, z, p);
        else row_geometry_tc(a, m, M, ray, z, p);
      }
      float ee[64];
      if constexpr (TAN) {   // e' = J_enc(p) u, rounded as simt_field_tangent rounds it
        const uint32_t mp = tile * (uint32_t)TILE + row;
        const float4 uv = mp < (uint32_t)M ? out[mp] : make_float4(0.f, 0.f, 0.f, 0.f);
        const float u[3] = {uv.x, uv.y, uv.z};
#pragma unroll
        for (int c = 0; c < 3; ++c) ee[c] = u[c];
#pragma unroll
        for (int l = 0; l < 10; ++l) {
          const float f = (float)(1 << l);
#pragma unroll
          for (int c = 0; c < 3; ++c) {
            float sn, cs; sincosf(__fmul_rn(f, p[c]), &sn, &cs);
            ee[3 + 6 * l + c] = __fmul_rn(__fmul_rn(f, cs), u[c]); ee[6 + 6 * l + c] = -__fmul_rn(__fmul_rn(f, sn), u[c]);
          }
        }
      } else {
#pragma unroll
        for (int c = 0; c < 3; ++c) ee[c] = p[c];
#pragma unroll
        for (int l = 0; l < 10; ++l) {
          const float f = (float)(1 << l);
#pragma unroll
          for (int c = 0; c < 3; ++c) { float sn, cs; sincosf(__fmul_rn(f, p[c]), &sn, &cs); ee[3 + 6 * l + c] = sn; ee[6 + 6 * l + c] = cs; }
        }
      }
      ee[63] = 0.f;
#pragma unroll
      for (int kb = 0; kb < 8; ++kb) {
        if ((kb >> 2) != part) continue;   // static register indices: ee[] stays in registers
        if constexpr (TAN) split_store8_bf16(ee + kb * 8, smem + SM_EHI + kb * 2048 + row * 16, smem + SM_ELO + kb * 2048 + row * 16);
        else split_store8(ee + kb * 8, smem + SM_EHI + kb * 2048 + row * 16, smem + SM_ELO + kb * 2048 + row * 16);
        if (stash) {
          __stcs(reinterpret_cast<float4*>(st.enc + (mo + m) * 64 + kb * 8), make_float4(ee[kb * 8], ee[kb * 8 + 1], ee[kb * 8 + 2], ee[kb * 8 + 3]));
          __stcs(reinterpret_cast<float4*>(st.enc + (mo + m) * 64 + kb * 8 + 4), make_float4(ee[kb * 8 + 4], ee[kb * 8 + 5], ee[kb * 8 + 6], ee[kb * 8 + 7]));
        }
      }
      if constexpr (!PTS) if (part == 0) {   // direction-encoding term of rgb_layers.0 is constant per ray: folded into a per-ray bias below
        float v[3], de[32];
        view_dir(a, ray, v);
        encode<4>(v, [&](int k, float val) { de[k] = val; });
#pragma unroll
        for (int k = 27; k < 32; ++k) de[k] = 0.f;
        if (stash) {
#pragma unroll
          for (int k4 = 0; k4 < 8; ++k4)
            __stcs(reinterpret_cast<float4*>(st.denc + (mo + m) * 32 + k4 * 4), make_float4(de[4 * k4], de[4 * k4 + 1], de[4 * k4 + 2], de[4 * k4 + 3]));
        }
        if (rl == 0 || (off0 + rl) % ray_len() == 0) {   // the block's first row and every row that starts a ray publish its direction encoding
          const int r = (off0 + rl) / ray_len();
#pragma unroll
          for (int k = 0; k < 32; ++k) rayb[RAYB_DE + r * 32 + k] = de[k];
        }
      }
      fence_async_smem();
      wg_sync();
      const float* w = a.weights;
      const int n_rays = PTS ? 0 : (off0 + 63) / ray_len() + 1;
      for (int r = 0; r < n_rays; ++r) {   // thread tl = output column of the rgb hidden layer
        if (DR < 128 && tl >= DR) break;
        float b = __ldg(w + nnb::B_RGBH(D) + tl);
#pragma unroll
        for (int k = 0; k < 27; ++k) b = fmaf(__ldg(w + nnb::W_RGBH(D) + (size_t)tl * (D + 27) + D + k), rayb[RAYB_DE + r * 32 + k], b);
        rayb[r * DR + tl] = b;   // read after layer 0's epilogue barrier
      }
    }
    float s_logit[2] = {0.f, 0.f};
    for (int g = 0; g < n_gemm; ++g) {
      uint32_t gm[D / 64];   // FWD_TANGENT: the forward's gate bits of layer g, loaded before the MMAs so the load completes behind them
      if constexpr (TAN) load_gates<D / 2>(st.gates + gate_bits_off(g, tile, threadIdx.x, (size_t)n_tiles * TILE, D), gm);
      // ---- MMAs: K-steps from the encoding operand E (layers 0 and 4) first, then from the previous layer's output; in points mode
      //      the rgb hidden layer ends with the two K-steps of the direction operand, which took E's place after layer 4 ----
      const int n_e = T::enc_steps(g), ns = T::gemm_steps(g, PTS);
      const uint32_t nrows = (g == 9) ? (uint32_t)DR : (uint32_t)D;
      for (int s = 0; s < ns; ++s) {
        const bool from_dir = PTS && g == 9 && s >= T::KS;
        const bool from_e = s < n_e || from_dir;
        const uint32_t ko = (uint32_t)(from_dir ? s - T::KS : (from_e ? s : s - n_e)) * 4096u;   // two k-octets of 2048 B per K-step
        const uint64_t dah = gdesc((from_e ? e_hi : a_hi) + ko, 2048, 128), dal = gdesc((from_e ? e_lo : a_lo) + ko, 2048, 128);
        const uint32_t wb = w_base + slot * STAGE_BYTES;
        const uint64_t dbh = gdesc(wb, nrows * 16u, 128), dbl = gdesc(wb + nrows * 32u, nrows * 16u, 128);
        mbar_wait(FULL(slot), phase);
        wgmma_fence();
        if constexpr (TAN) {
          wgmma_bf16<D>(acc, dal, dbh, s > 0 ? 1u : 0u);
          wgmma_bf16<D>(acc, dah, dbl, 1u);
          wgmma_bf16<D>(acc, dah, dbh, 1u);
        } else if (g < 9) {
          wgmma_f16<D>(acc, dal, dbh, s > 0 ? 1u : 0u);
          wgmma_f16<D>(acc, dah, dbl, 1u);
          wgmma_f16<D>(acc, dah, dbh, 1u);
        } else {
          wgmma_f16<DR>(acc, dal, dbh, s > 0 ? 1u : 0u);
          wgmma_f16<DR>(acc, dah, dbl, 1u);
          wgmma_f16<DR>(acc, dah, dbh, 1u);
        }
        wgmma_commit();
        if (s > 0) {   // the previous K-step's MMAs have completed: release its weight stage
          wgmma_wait<1>();
          if (tl == 0) mbar_arrive(EMPTY(slot == 0 ? NST - 1 : slot - 1));
        }
        if (++slot == NST) { slot = 0; phase ^= 1u; }
      }
      wgmma_wait<0>();
      if (tl == 0) mbar_arrive(EMPTY(slot == 0 ? NST - 1 : slot - 1));
      // ---- epilogue ----
      if constexpr (TAN) {   // h'_g = [h_g > 0] z'_g: no bias, the forward's gate -> tangent stash and the next A operand (bf16 hi | lo)
#pragma unroll
        for (int j = 0; j < D / 8; ++j) {
          const int col = j * 8 + c0;
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            const int row = r0 + 8 * r;
            const uint32_t b = gm[j / 8] << (4 * (j & 7) + 2 * r);   // gate bits of columns c0 and c0 + 1 at bits 31 and 30
            const float v0 = (b & 0x80000000u) ? acc[4 * j + 2 * r] : 0.f, v1 = (b & 0x40000000u) ? acc[4 * j + 2 * r + 1] : 0.f;
            uint32_t hw, lw;
            split2_bf16(v0, v1, hw, lw);
            const int off = j * 2048 + row * 16 + c0 * 2;
            *reinterpret_cast<uint32_t*>(smem + SM_AHI + off) = hw;
            *reinterpret_cast<uint32_t*>(smem + SM_ALO + off) = lw;
            __stcs(reinterpret_cast<float2*>(st.h[g] + (mt + row) * D + col), make_float2(v0, v1));
          }
        }
        fence_async_smem();
        wg_sync();
      } else if (g < 9) {
        const float* bias = (g < 8) ? s_bias + g * D : s_bias + B_FEAT0;
        float* sp = stash ? (g < 8 ? st.h[g] : st.feat) : nullptr;
        uint32_t gw[D / 64] = {};   // ReLU gate bits of this thread's fragment, shifted in in the order b = 4j + 2r + e
#pragma unroll
        for (int j = 0; j < D / 8; ++j) {
          const int col = j * 8 + c0;
          const float2 b = *reinterpret_cast<const float2*>(bias + col);
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            const int row = r0 + 8 * r;
            float v0 = acc[4 * j + 2 * r] + b.x, v1 = acc[4 * j + 2 * r + 1] + b.y;
            if (g != 8) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
            uint32_t hw, lw;
            split2(v0, v1, hw, lw);
            const int off = j * 2048 + row * 16 + c0 * 2;
            *reinterpret_cast<uint32_t*>(smem + SM_AHI + off) = hw;
            *reinterpret_cast<uint32_t*>(smem + SM_ALO + off) = lw;
            if (g == 7) s_logit[r] = fmaf(v1, s_bias[W_SIG0 + col + 1], fmaf(v0, s_bias[W_SIG0 + col], s_logit[r]));
            if (sp) __stcs(reinterpret_cast<float2*>(sp + (mo + mt + row) * D + col), make_float2(v0, v1));
            gw[j / 8] = push_gate(push_gate(gw[j / 8], v0), v1);
          }
        }
        if (gates && g < 8) store_gates<D / 2>(st.gates + (PACK ? gate_bits_off(g, mo / TILE + tile, threadIdx.x, M, D)
                                                               : gate_bits_off(g, tile, threadIdx.x, (size_t)n_tiles * TILE, D)), gw);
        if constexpr (PTS) {
          // Layer 4 was the last reader of E.  The direction operand of the rgb hidden layer takes its place: enc4(dirs[m]), 27 columns
          // padded to 32 (two K-steps), as fp16 hi | lo in E's layout.  A warp writes the 16 rows its own MMAs read, like the A operand
          // above, and the barrier below orders the writes before the rgb hidden layer's MMAs.
          if (g == 4 && !occ) {
            const int row = wg * 64 + (warp & 3) * 16 + (lane & 15), part = lane >> 4;
            const uint32_t mm = computed_here(min(tile * (uint32_t)TILE + row, (uint32_t)M - 1u));
            float v[3], de[32];
#pragma unroll
            for (int c = 0; c < 3; ++c) v[c] = a.dirs ? __ldg(a.dirs + (size_t)mm * 3 + c) : 1.f;
            encode<4>(v, [&](int k, float val) { de[k] = val; });
#pragma unroll
            for (int k = 27; k < 32; ++k) de[k] = 0.f;
#pragma unroll
            for (int kb = 0; kb < 4; ++kb) {
              if ((kb >> 1) != part) continue;   // static register indices
              split_store8(de + kb * 8, smem + SM_EHI + kb * 2048 + row * 16, smem + SM_ELO + kb * 2048 + row * 16);
              if constexpr (GRAD) {   // the per-point direction encoding of the stash (the weight gradient of rgb_layers.0's last 27 columns)
                float* dp = st.denc + (mt + row) * 32 + kb * 8;
                __stcs(reinterpret_cast<float4*>(dp), make_float4(de[kb * 8], de[kb * 8 + 1], de[kb * 8 + 2], de[kb * 8 + 3]));
                __stcs(reinterpret_cast<float4*>(dp + 4), make_float4(de[kb * 8 + 4], de[kb * 8 + 5], de[kb * 8 + 6], de[kb * 8 + 7]));
              }
            }
          }
        }
        fence_async_smem();
        wg_sync();   // the whole A operand (and, after layer 0, the per-ray bias) is written before the next layer's MMAs
      } else {
        // rgb hidden layer (D/2 columns) -> colour head + per-sample record
        float c_acc[2][3] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
        uint32_t gw[D / 128 > 0 ? D / 128 : 1] = {};
        const int off0 = PTS || FRAME || CHUNK ? 0 : ray_off();
#pragma unroll
        for (int j = 0; j < DR / 8; ++j) {
          const int col = j * 8 + c0;
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            const int row = r0 + 8 * r;
            const float* rb = PTS ? rayb : rayb + ((off0 + row - wg * 64) / ray_len()) * DR;   // points mode: b_rgbh
            const float v0 = fmaxf(acc[4 * j + 2 * r] + rb[col], 0.f), v1 = fmaxf(acc[4 * j + 2 * r + 1] + rb[col + 1], 0.f);
#pragma unroll
            for (int c = 0; c < 3; ++c)
              c_acc[r][c] = fmaf(v1, s_bias[W_RGB0 + c * DR + col + 1], fmaf(v0, s_bias[W_RGB0 + c * DR + col], c_acc[r][c]));
            if (stash) __stcs(reinterpret_cast<float2*>(st.hr + (mo + mt + row) * DR + col), make_float2(v0, v1));
            gw[j / 8] = push_gate(push_gate(gw[j / 8], v0), v1);
          }
        }
        if (gates) store_gates<D / 4>(st.gates + (PACK ? gate_bits_off(8, mo / TILE + tile, threadIdx.x, M, D)
                                                               : gate_bits_off(8, tile, threadIdx.x, (size_t)n_tiles * TILE, D)), gw);
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const float sl = quad_sum(s_logit[r]);
          const float cr = quad_sum(c_acc[r][0]), cg = quad_sum(c_acc[r][1]), cb = quad_sum(c_acc[r][2]);
          if ((lane & 3) == 0) {
            const size_t m = mt + r0 + 8 * r, mm = m < M ? m : M - 1;
            const float s = sl + s_bias[B_SIG0];
            float sigma;
            SampleRec rec;
            rec.r = sigmoid_f(cr + s_bias[B_SIG0 + 1]); rec.g = sigmoid_f(cg + s_bias[B_SIG0 + 2]); rec.b = sigmoid_f(cb + s_bias[B_SIG0 + 3]);
            rec.a = density_act(s, a.flags, &sigma); rec.s = s;
            if constexpr (VJP) {   // every row of the tile has its record; the point of a row past M is the last point
              const uint32_t mp = computed_here(tile * (uint32_t)TILE + r0 + 8 * r);
              rec.z = 0.f; rec.pad0 = 0.f; rec.pad1 = 0.f;
              recs[mp] = rec;
              if (out && mp < (uint32_t)M) out[mp] = make_float4(rec.r, rec.g, rec.b, rec.a);
            } else if constexpr (PTS) {
              const uint32_t mp = computed_here(tile * (uint32_t)TILE + r0 + 8 * r);
              if (mp < (uint32_t)M) out[mp] = make_float4(rec.r, rec.g, rec.b, rec.a);
            } else if constexpr (FRAME) {   // E row r0 + 8 r, k-octet 0: this warpgroup's rows of E
              *reinterpret_cast<float4*>(smem + SM_EHI + (r0 + 8 * r) * 16) = make_float4(rec.r, rec.g, rec.b, rec.a);
            } else if constexpr (CHUNK) {
              const int2 ni = DEVN ? live_sample(a, fr.k, fr.list, n_live, m) : chunk_sample(a, fr.k, m);
              rec.z = sample_z(a, ni.x, ni.y);
              rec.pad0 = 0.f; rec.pad1 = 0.f;
              recs[mo + m] = rec;
            } else {
              rec.z = sample_z(a, (int)(mm / a.S), (int)(mm % a.S));
              rec.pad0 = 0.f; rec.pad1 = 0.f;
              recs[m] = rec;
            }
          }
        }
      }
    }
    if (occ) {   // the tile ended after layer 7 and the density head
      // an occupancy-only tile does not use the per-ray bias area: a march tile's 128 values (occupancy - tau) go there
      float* s_val = reinterpret_cast<float*>(smem + SM_RAYB);
      static_assert(2 * RAYB_FLOATS >= TILE, "a march tile's values fit the per-ray bias area");
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const float sl = quad_sum(s_logit[r]);
        const uint32_t mp = computed_here(tile * (uint32_t)TILE + r0 + 8 * r);
        float sigma;
        if constexpr (MODE == FWD_POINTS) {
          if ((lane & 3) == 0 && mp < (uint32_t)M) out[mp] = make_float4(0.f, 0.f, 0.f, density_act(sl + s_bias[B_SIG0], a.flags, &sigma));
        } else if constexpr (VJP) {
          if ((lane & 3) == 0) {
            SampleRec rec;
            rec.s = sl + s_bias[B_SIG0];
            rec.a = density_act(rec.s, a.flags, &sigma);
            rec.r = 0.f; rec.g = 0.f; rec.b = 0.f; rec.z = 0.f; rec.pad0 = 0.f; rec.pad1 = 0.f;
            recs[mp] = rec;
            if (out && mp < (uint32_t)M) out[mp] = make_float4(0.f, 0.f, 0.f, rec.a);
          }
        } else if constexpr (MODE == FWD_MARCH) {
          if ((lane & 3) == 0) s_val[r0 + 8 * r] = __fsub_rn(density_act(sl + s_bias[B_SIG0], a.flags, &sigma), q.tau);
        } else if constexpr (MODE == FWD_SECANT) {
          if ((lane & 3) == 0 && mp < (uint32_t)M) {
            const int ray = q.list[mp];
            float4 b = (t % q.n_secant == 0 ? q.brk0 : q.brk1)[ray];
            const float d_mid = secant_depth(b), f_mid = __fsub_rn(density_act(sl + s_bias[B_SIG0], a.flags, &sigma), q.tau);
            if (f_mid < 0.f) { b.x = d_mid; b.z = f_mid; } else { b.y = d_mid; b.w = f_mid; }
            q.brk1[ray] = b;
          }
        }
      }
      if constexpr (MODE == FWD_MARCH) {
        // both warpgroups' values are written before the scan, and the scan has read them before either warpgroup's next tile writes
        asm volatile("bar.sync 3, 256;" ::: "memory");
        if (warp == 0) march_scan(q, q.list ? q.list[tile] : tile, s_val, lane);
        asm volatile("bar.sync 3, 256;" ::: "memory");
      }
    }
    if constexpr (FRAME) {
      // the warpgroup's 64 rows (its two ray-chunks) are in E before its first two warps composite them; the barrier at the top of
      // the next tile orders their reads before the prologue writes E again
      static_assert(TILE * 16 <= 2048, "a frame tile's (r, g, b, a) rows fit k-octet 0 of E");
      wg_sync();
      if ((warp & 3) < 2) frame_step(a, fr, 4 * tile + 2 * wg + (warp & 3), n_live, smem + SM_EHI + (wg * 64 + 32 * (warp & 3)) * 16, lane);
    }
  }
}

template <int D>
__global__ void __launch_bounds__(N_THREADS, 1) tc_field_fwd(nnb_render_args a, const unsigned char* __restrict__ wimg,
                                              SampleRec* __restrict__ recs, const __grid_constant__ TcStash st, size_t M, int n_tiles,
                                              int stash) {
  tc_fwd_body<D, FWD_RAYS>(a, wimg, recs, nullptr, st, MarchPtrs{}, M, n_tiles, stash);
}

template <int D>
__global__ void __launch_bounds__(N_THREADS, 1) tc_points_fwd(nnb_render_args a, const unsigned char* __restrict__ wimg,
                                                              float4* __restrict__ out, size_t M, int n_tiles) {
  tc_fwd_body<D, FWD_POINTS>(a, wimg, nullptr, out, TcStash{}, MarchPtrs{}, M, n_tiles, 0);
}
// the same on the *count points that nnb_geometry_frame's compaction wrote (a separate name in profiles)
template <int D>
__global__ void __launch_bounds__(N_THREADS, 1) tc_points_fwd_n(nnb_render_args a, const unsigned char* __restrict__ wimg,
                                                                float4* __restrict__ out, const int* __restrict__ count) {
  MarchPtrs q{};
  q.count = count;
  tc_fwd_body<D, FWD_POINTS, true>(a, wimg, nullptr, out, TcStash{}, q, 0, 0, 0);
}

// one round of nnb_ray_march: block q.block of every ray of q.list (n_rays rays when q.count is NULL)
template <int D>
__global__ void __launch_bounds__(N_THREADS, 1) tc_march(nnb_render_args a, const unsigned char* __restrict__ wimg,
                                                         const __grid_constant__ MarchPtrs q, int n_rays) {
  tc_fwd_body<D, FWD_MARCH>(a, wimg, nullptr, nullptr, TcStash{}, q, 0, n_rays, 0);
}
// the q.n_secant secant passes of nnb_ray_march over the *q.count hit rays of q.list
template <int D>
__global__ void __launch_bounds__(N_THREADS, 1) tc_secant(nnb_render_args a, const unsigned char* __restrict__ wimg,
                                                          const __grid_constant__ MarchPtrs q) {
  tc_fwd_body<D, FWD_SECANT>(a, wimg, nullptr, nullptr, TcStash{}, q, 0, 0, 0);
}

// one round of nnb_render_frame: chunk f.k of every ray of f.list (of every ray when f.list is NULL)
template <int D>
__global__ void __launch_bounds__(N_THREADS, 1) tc_frame(nnb_render_args a, const unsigned char* __restrict__ wimg,
                                                         const __grid_constant__ FramePtrs f) {
  tc_fwd_body<D, FWD_FRAME>(a, wimg, nullptr, nullptr, TcStash{}, MarchPtrs{}, (size_t)a.N * a.S, 0, 0, f);
}
// one reverse round of nnb_render_frame_bwd: chunk f.k of every ray with records, the training stash and gate bits (n_tiles = ceil(N / 4))
template <int D>
__global__ void __launch_bounds__(N_THREADS, 1) tc_frame_stash(nnb_render_args a, const unsigned char* __restrict__ wimg,
                                                               SampleRec* __restrict__ recs, const __grid_constant__ TcStash st,
                                                               const __grid_constant__ FramePtrs f, int n_tiles) {
  tc_fwd_body<D, FWD_CHUNK>(a, wimg, recs, nullptr, st, MarchPtrs{}, (size_t)a.N * 32, n_tiles, 1, f);
}
// tc_frame_stash on the rays of round f.k's live list f.list (*f.count of them; the launch is sized for N)
template <int D>
__global__ void __launch_bounds__(N_THREADS, 1) tc_frame_stash_live(nnb_render_args a, const unsigned char* __restrict__ wimg,
                                                                    SampleRec* __restrict__ recs, const __grid_constant__ TcStash st,
                                                                    const __grid_constant__ FramePtrs f) {
  tc_fwd_body<D, FWD_CHUNK, true>(a, wimg, recs, nullptr, st, MarchPtrs{}, (size_t)a.N * 32, 0, 1, f);
}
// one forward round of nnb_render_fwd_tmin: tc_frame_stash_live into the packed stash of M rows (FWD_PACK)
template <int D>
__global__ void __launch_bounds__(N_THREADS, 1) tc_stash_pack(nnb_render_args a, const unsigned char* __restrict__ wimg,
                                                              SampleRec* __restrict__ recs, const __grid_constant__ TcStash st,
                                                              const __grid_constant__ FramePtrs f, size_t M) {
  tc_fwd_body<D, FWD_PACK, true>(a, wimg, recs, nullptr, st, MarchPtrs{}, M, 0, 1, f);
}

// ---- weight gradients: dW[n][k] += sum_m dY[m][n] X[m][k] (and db[n] += sum_m dY[m][n]) over the fp32 stash ----------------------
// CTA = one 128-row slice of dW (all KN columns) over a contiguous share of the samples, warp-specialized in 32-sample chunks:
//   warpgroup 2 (converter): one thread streams each chunk's fp32 rows into a staging ring with cp.async.bulk, completion on an
//     mbarrier tx-count: two copies per chunk, 32 contiguous rows of X and of dY (whole rows: the row slices of a job read the same
//     dY and X rows, and the second read of each comes from L2; 1D copies need no tensor map).  All 128 threads
//     then convert the staged chunk to bf16 hi | lo K-major operands dY^T / X^T (zeroing samples >= s_end, rows >= Nn, columns >= Kk,
//     and summing the bias partials), publish them to the MMA warpgroups through an mbarrier and refill the staging slot.
//   warpgroups 0, 1 (MMA): 64 rows of dW each, 128 fp32 accumulators in registers; per chunk 2 K-steps x three MMAs
//     (a_lo*b_hi + a_hi*b_lo + a_hi*b_hi), an operand buffer released once wgmma.wait_group shows its MMAs complete.
// A split covers whole 64-sample blocks (two chunks each; samples past s_end are zeros), so every output element sees the same MMA
// sequence for any chunking.  Bias slot h of a row sums samples 32h .. 32h + 31 of each 64-sample block in sample order.  Each split
// stores its partial dW and bias slots to the split buffer; wgrad_reduce adds the splits in a fixed order, so the result is the same
// every run.
// tc_wgrad_piece<KN> runs one job as column pieces: the CTA holds columns k0 .. k0 + KN - 1 of the job's dW and stages that column
// block of X through a 2-D tensor map (X rows are wider than KN).  An output element's K-steps, MMAs and operands are those of the
// whole-job CTA, and the piece stores exactly that CTA's floats of its columns; only the piece at k0 = 0 stores the bias slots.
struct WgJobT { const float* dY; const float* X; float* dW; float* db; int ldy, Nn, ldx, Kk, ldw, cta0; size_t part_off; int k0; };
constexpr int MAX_WG_JOBS = 10, WG_BLOCK = 64;
struct WgJobsT { WgJobT j[MAX_WG_JOBS]; int njobs, msplit, per_cta; };
constexpr int WG_MAX_LDY = 256;
template <int KN> struct Wg {   // shared-memory map (bytes) of tc_wgrad<KN>; X rows are KN floats (ldx == KN)
  static constexpr int CH = 32, NOP = 2;                                   // samples per chunk, operand buffers
  static constexpr int SY = CH * WG_MAX_LDY * 4, STG = SY + CH * KN * 4;   // fp32 staging: dY [CH][ldy] | X [CH][KN]
  static constexpr int A_BYTES = 128 * CH * 2, B_BYTES = KN * CH * 2; // one bf16 plane of dY^T / X^T
  static constexpr int OPB = 2 * A_BYTES + 2 * B_BYTES;
  static constexpr int NSTG = (232448 - 128 - NOP * OPB) / STG;      // staging ring: all the rest of shared memory (loads in flight)
  static constexpr int SM_OP = NSTG * STG, SM_BAR = SM_OP + NOP * OPB;
  static constexpr int SMEM = SM_BAR + (NSTG + 2 * NOP) * 8;
  static_assert(NSTG >= 2 && SMEM <= 232448, "shared memory budget");
};

// 2-D bulk tensor copy of box (c0, c1) of the map (innermost coordinate first), completion on `bar`
__device__ __forceinline__ void tma_g2s_2d(uint32_t dst, const CUtensorMap* map, int c0, int c1, uint32_t bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
               ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(bar) : "memory");
}

// KN = 256 | 128 | 64: columns of dW (features of X) held by one CTA.  XMAP: X column block k0 .. k0 + KN - 1 through xmap (box KN x CH).
// DEVM (tc_wgrad_live, tc_wgrad_piece_live: a reverse round of nnb_render_frame_train_bwd_tmin): M = min(32 *mcount, M), the rows of the
// round's live rays, read when the kernel starts, and per_cta formed from it as launch_wgrad forms it, with the launch's split count: at
// *mcount = N the splits are those of tc_wgrad on 32 N rows; splits past M store zeros.
template <int KN, bool XMAP, bool DEVM = false>
__device__ __forceinline__ void wgrad_body(const WgJobsT& J, const CUtensorMap* xmap, size_t M, float* __restrict__ part,
                                           const int* mcount = nullptr) {
  using W = Wg<KN>;
  constexpr int CH = W::CH, NSTG = W::NSTG, NOP = W::NOP, A_BYTES = W::A_BYTES, B_BYTES = W::B_BYTES;
  extern __shared__ __align__(1024) unsigned char smem[];
  int ji = 0;
  while (ji + 1 < J.njobs && (int)blockIdx.x >= J.j[ji + 1].cta0) ++ji;
  const WgJobT& jb = J.j[ji];
  const int local = blockIdx.x - jb.cta0, n0 = (local / J.msplit) * 128;
  size_t s_begin, s_end;
  if constexpr (DEVM) {
    const size_t m = (size_t)max(*mcount, 0) * 32, Md = m < M ? m : M;
    const size_t per_cta = ((Md + J.msplit - 1) / J.msplit + WG_BLOCK - 1) / WG_BLOCK * WG_BLOCK;
    s_begin = (size_t)(local % J.msplit) * per_cta;
    s_end = (s_begin + per_cta < Md) ? s_begin + per_cta : Md;   // an empty split stores zeros
  } else {
    s_begin = (size_t)(local % J.msplit) * J.per_cta;
    s_end = (s_begin + J.per_cta < M) ? s_begin + J.per_cta : M;   // an empty split stores zeros
  }
  const int nch = s_begin < s_end ? (int)((s_end - s_begin + WG_BLOCK - 1) / WG_BLOCK) * (WG_BLOCK / CH) : 0;
  float* pp = part + jb.part_off + (size_t)(local % J.msplit) * ((size_t)jb.Nn * jb.Kk + 2 * jb.Nn);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const uint32_t bar0 = smem_u32(smem + W::SM_BAR);
  auto SFULL = [&](int i) { return bar0 + 8u * i; };                    // staging slot filled (tx-count)
  auto OPFULL = [&](int i) { return bar0 + 8u * (NSTG + i); };          // operand buffer written by the converter
  auto OPEMPTY = [&](int i) { return bar0 + 8u * (NSTG + NOP + i); };   // operand buffer read by both MMA warpgroups
  if (tid == 0) {
    for (int i = 0; i < NSTG; ++i) mbar_init(SFULL(i), 1);
    for (int i = 0; i < NOP; ++i) { mbar_init(OPFULL(i), 1); mbar_init(OPEMPTY(i), 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  pdl_launch_dependents();   // the next grid of the stage starts only once every CTA of this one is resident (see tc_wgrad_all)
  const bool last_cta = blockIdx.x == gridDim.x - 1;

  if (warp >= 8) {
    // =============================== converter warpgroup ===============================
    // 104 + 2 x 200 = 3 x 168 registers per thread: the MMA warpgroups get what the converter gives up
    asm volatile("setmaxnreg.dec.sync.aligned.u32 104;" ::: "memory");
    const int ct = tid - 256;
    const int ny = jb.Nn - n0 < 128 ? jb.Nn - n0 : 128;   // dY columns of this row slice
    auto issue = [&](int c) {   // thread 0 of the warpgroup: chunk c -> staging slot c % NSTG (a chunk past s_end copies nothing)
      const int sl = c % NSTG;
      const size_t s0 = s_begin + (size_t)c * CH;
      if (s0 < s_end) {   // then rows s0 .. s0 + 31 < Mpad: in bounds of the stash
        mbar_expect_tx(SFULL(sl), (uint32_t)(CH * (jb.ldy + KN) * 4));
        bulk_g2s(smem_u32(smem + sl * W::STG), jb.dY + s0 * jb.ldy, (uint32_t)(CH * jb.ldy * 4), SFULL(sl));
        if constexpr (XMAP) tma_g2s_2d(smem_u32(smem + sl * W::STG + W::SY), xmap, jb.k0, (int)s0, SFULL(sl));
        else bulk_g2s(smem_u32(smem + sl * W::STG + W::SY), jb.X + s0 * KN, CH * KN * 4, SFULL(sl));
      } else {
        mbar_arrive(SFULL(sl));
      }
    };
    if (ct == 0)
      for (int c = 0; c < NSTG && c < nch; ++c) issue(c);
    float db0 = 0.f, db1 = 0.f;   // bias slots 0 and 1
    for (int c = 0; c < nch; ++c) {
      const int sl = c % NSTG, ob = c % NOP;
      const size_t s0 = s_begin + (size_t)c * CH;
      const int nvalid = s0 < s_end ? (s_end - s0 < (size_t)CH ? (int)(s_end - s0) : CH) : 0;
      const float* sy = reinterpret_cast<const float*>(smem + sl * W::STG);
      const float* sx = reinterpret_cast<const float*>(smem + sl * W::STG + W::SY);
      unsigned char* op = smem + W::SM_OP + ob * W::OPB;
      mbar_wait(SFULL(sl), (uint32_t)(c / NSTG) & 1u);
      mbar_wait(OPEMPTY(ob), ((uint32_t)(c / NOP) & 1u) ^ 1u);
      const bool half1 = (c * CH) & 32;   // the chunk lies in the second half of its 64-sample block: bias slot 1
      {   // A = dY^T: thread = row n, CH / 8 8-sample octets
        const bool nv = ct < ny;
        float db = half1 ? db1 : db0;
#pragma unroll
        for (int so = 0; so < CH / 8; ++so) {
          float v[8];
#pragma unroll
          for (int q = 0; q < 8; ++q) {
            v[q] = (nv && so * 8 + q < nvalid) ? sy[(so * 8 + q) * jb.ldy + n0 + ct] : 0.f;
            db += v[q];
          }
          split_store8_bf16(v, op + so * 2048 + ct * 16, op + A_BYTES + so * 2048 + ct * 16);
        }
        if (half1) db1 = db; else db0 = db;
      }
#pragma unroll 4
      for (int i = 0; i < KN * (CH / 8) / 128; ++i) {   // B = X^T: row k (KN), reduction index = sample
        const int item = ct + i * 128, k = item % KN, so = item / KN;
        float v[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) v[q] = (jb.k0 + k < jb.Kk && so * 8 + q < nvalid) ? sx[(so * 8 + q) * KN + k] : 0.f;
        split_store8_bf16(v, op + 2 * A_BYTES + so * KN * 16 + k * 16, op + 2 * A_BYTES + B_BYTES + so * KN * 16 + k * 16);
      }
      fence_async_smem();
      asm volatile("bar.sync 1, 128;" ::: "memory");   // the operands are written and the staging slot is read
      if (ct == 0) mbar_arrive(OPFULL(ob));
      if (ct == 0 && c + NSTG < nch) issue(c + NSTG);
    }
    if (ct < ny && jb.k0 == 0) {
      pp[(size_t)jb.Nn * jb.Kk + n0 + ct] = db0;
      pp[(size_t)jb.Nn * jb.Kk + jb.Nn + n0 + ct] = db1;
    }
    if (last_cta) pdl_wait();
    return;
  }
  // =============================== MMA warpgroups ===============================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 200;" ::: "memory");
  const int wg = warp >> 2;
  float acc[KN / 2];
#pragma unroll
  for (int i = 0; i < KN / 2; ++i) acc[i] = 0.f;
  for (int c = 0; c < nch; ++c) {
    const int ob = c % NOP;
    const uint32_t a = smem_u32(smem + W::SM_OP + ob * W::OPB) + wg * 1024, b = smem_u32(smem + W::SM_OP + ob * W::OPB + 2 * A_BYTES);
    mbar_wait(OPFULL(ob), (uint32_t)(c / NOP) & 1u);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < CH / 16; ++ks) {
      const uint64_t dah = gdesc(a + ks * 4096, 2048, 128), dal = gdesc(a + A_BYTES + ks * 4096, 2048, 128);
      const uint64_t dbh = gdesc(b + ks * 2 * KN * 16, KN * 16, 128), dbl = gdesc(b + B_BYTES + ks * 2 * KN * 16, KN * 16, 128);
      wgmma_bf16<KN>(acc, dal, dbh, (c > 0 || ks > 0) ? 1u : 0u);
      wgmma_bf16<KN>(acc, dah, dbl, 1u);
      wgmma_bf16<KN>(acc, dah, dbh, 1u);
    }
    wgmma_commit();
    if (c > 0) {   // the previous chunk's MMAs have completed: release its operand buffer
      wgmma_wait<1>();
      if ((tid & 127) == 0) mbar_arrive(OPEMPTY((c - 1) % NOP));
    }
  }
  wgmma_wait<0>();
  const int r0 = n0 + wg * 64 + (warp & 3) * 16 + (lane >> 2), c0 = (lane & 3) * 2;
#pragma unroll
  for (int j = 0; j < KN / 8; ++j)
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int n = r0 + 8 * r;
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int k = jb.k0 + j * 8 + c0 + e;
        if (n < jb.Nn && k < jb.Kk) pp[(size_t)n * jb.Kk + k] = acc[4 * j + 2 * r + e];
      }
    }
  if (last_cta) pdl_wait();
}

template <int KN>
__global__ void __launch_bounds__(384, 1) tc_wgrad(const __grid_constant__ WgJobsT J, size_t M, float* __restrict__ part) {
  wgrad_body<KN, false>(J, nullptr, M, part);
}
template <int KN>   // a separate name in profiles: the column pieces of one job, X through the tensor map
__global__ void __launch_bounds__(384, 1) tc_wgrad_piece(const __grid_constant__ WgJobsT J, const __grid_constant__ CUtensorMap xmap,
                                                         size_t M, float* __restrict__ part) {
  wgrad_body<KN, true>(J, &xmap, M, part);
}
// the same two kernels with the row count read on the device (wgrad_body's DEVM)
template <int KN>
__global__ void __launch_bounds__(384, 1) tc_wgrad_live(const __grid_constant__ WgJobsT J, size_t M, float* __restrict__ part,
                                                        const int* __restrict__ mcount) {
  wgrad_body<KN, false, true>(J, nullptr, M, part, mcount);
}
template <int KN>
__global__ void __launch_bounds__(384, 1) tc_wgrad_piece_live(const __grid_constant__ WgJobsT J, const __grid_constant__ CUtensorMap xmap,
                                                              size_t M, float* __restrict__ part, const int* __restrict__ mcount) {
  wgrad_body<KN, true, true>(J, &xmap, M, part, mcount);
}

// floats of the partial buffer that tc_wgrad uses for these jobs at msplit sample splits (two bias slots per row)
size_t wg_part_floats(const WgJobT* jobs, int njobs, int msplit) {
  size_t f = 0;
  for (int i = 0; i < njobs; ++i) f += (size_t)jobs[i].Nn * jobs[i].Kk + 2 * jobs[i].Nn;
  return f * msplit;
}

// map of the fp32 [rows][ldx] matrix X with a box of box_cols x box_rows floats (rows past `rows` read as zeros).  The library links
// cudart statically and not libcuda, so the driver's encoder is looked up through the runtime.
cudaError_t encode_x_map(CUtensorMap* map, const float* X, int ldx, size_t rows, int box_cols, int box_rows) {
  static PFN_cuTensorMapEncodeTiled_v12000 encode = nullptr;
  if (!encode) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    cudaError_t e = cudaGetDriverEntryPointByVersion("cuTensorMapEncodeTiled", &fn, 12000, cudaEnableDefault, &q);
    if (e != cudaSuccess) return e;
    if (q != cudaDriverEntryPointSuccess || !fn) return cudaErrorSymbolNotFound;
    encode = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(fn);
  }
  const cuuint64_t dims[2] = {(cuuint64_t)ldx, (cuuint64_t)rows}, strides[1] = {(cuuint64_t)ldx * 4};
  const cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows}, elem_strides[2] = {1, 1};
  const CUresult r = encode(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(X), dims, strides, box, elem_strides,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? cudaSuccess : cudaErrorInvalidValue;
}

// jobs -> tc_wgrad<KN> into part[off ..], or with PIECES one job as ceil(Kk / KN) column pieces of tc_wgrad_piece<KN>; R[i] receives
// job i's reduction (launch_wgrad_reduce).  chained: programmatic dependent launch behind the previous grid on the stream (see
// tc_wgrad_all).  mcount (not NULL): the _live kernels, whose rows are min(32 *mcount, M); the splits and the partial buffer stay M's.
template <int KN, bool PIECES = false>
cudaError_t launch_wgrad(const WgJobT* jobs, int njobs, size_t M, int D, int msplit, float* part, size_t off, RedJob* R, bool chained,
                         cudaStream_t st, const int* mcount = nullptr) {
  static bool attr = false;
  if (!attr) {
    cudaError_t e;
    if constexpr (PIECES) {
      e = cudaFuncSetAttribute(tc_wgrad_piece<KN>, cudaFuncAttributeMaxDynamicSharedMemorySize, Wg<KN>::SMEM);
      if (e == cudaSuccess) e = cudaFuncSetAttribute(tc_wgrad_piece_live<KN>, cudaFuncAttributeMaxDynamicSharedMemorySize, Wg<KN>::SMEM);
    } else {
      e = cudaFuncSetAttribute(tc_wgrad<KN>, cudaFuncAttributeMaxDynamicSharedMemorySize, Wg<KN>::SMEM);
      if (e == cudaSuccess) e = cudaFuncSetAttribute(tc_wgrad_live<KN>, cudaFuncAttributeMaxDynamicSharedMemorySize, Wg<KN>::SMEM);
    }
    if (e != cudaSuccess) return e;
    attr = true;
  }
  if (PIECES && njobs != 1) return cudaErrorInvalidValue;   // one tensor map per launch
  WgJobsT J{};
  int ctas = 0, nj = 0;
  for (int i = 0; i < njobs; ++i) {
    // dY chunks are staged as whole rows, X chunks as whole rows or (pieces) KN-column boxes: 16-byte multiples
    if ((PIECES ? jobs[i].ldx % 4 != 0 : jobs[i].ldx != KN) || jobs[i].ldy > WG_MAX_LDY || jobs[i].ldy % 4) return cudaErrorInvalidValue;
    const int pieces = PIECES ? (jobs[i].Kk + KN - 1) / KN : 1;
    if (nj + pieces > MAX_WG_JOBS) return cudaErrorInvalidValue;
    for (int p = 0; p < pieces; ++p, ++nj) {
      J.j[nj] = jobs[i]; J.j[nj].k0 = p * KN; J.j[nj].cta0 = ctas; J.j[nj].part_off = off;
      ctas += (jobs[i].Nn + 127) / 128 * msplit;
    }
    const size_t stride = (size_t)jobs[i].Nn * jobs[i].Kk + 2 * jobs[i].Nn;
    R[i] = RedJob{jobs[i].dW, jobs[i].db, jobs[i].Nn, jobs[i].Kk, jobs[i].ldw, msplit, 2, off, stride};
    off += stride * msplit;
  }
  if (off > wpart_floats(M, D)) return cudaErrorInvalidValue;
  J.njobs = nj; J.msplit = msplit;
  J.per_cta = (int)(((M + msplit - 1) / msplit + WG_BLOCK - 1) / WG_BLOCK * WG_BLOCK);
  cudaLaunchAttribute at{};
  at.id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at.val.programmaticStreamSerializationAllowed = 1;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(ctas); cfg.blockDim = dim3(384); cfg.dynamicSmemBytes = Wg<KN>::SMEM; cfg.stream = st;
  cfg.attrs = &at; cfg.numAttrs = chained ? 1 : 0;
  cudaError_t e;
  if constexpr (PIECES) {
    CUtensorMap xmap;
    e = encode_x_map(&xmap, jobs[0].X, jobs[0].ldx, M, KN, Wg<KN>::CH);
    if (e == cudaSuccess) e = mcount ? cudaLaunchKernelEx(&cfg, tc_wgrad_piece_live<KN>, J, xmap, M, part, mcount)
                                     : cudaLaunchKernelEx(&cfg, tc_wgrad_piece<KN>, J, xmap, M, part);
  } else {
    e = mcount ? cudaLaunchKernelEx(&cfg, tc_wgrad_live<KN>, J, M, part, mcount) : cudaLaunchKernelEx(&cfg, tc_wgrad<KN>, J, M, part);
  }
  return e != cudaSuccess ? e : cudaGetLastError();
}

// The weight-gradient stage of the TC engine's backward: the MLP GEMMs on tensor cores, the small heads on the fp32 SIMT kernel
// head_wgrad.  Four grids, each chained behind the one before with programmatic dependent launch:
//   1. the D-wide jobs (layers 1..7, fc_feature): (Nn / 128) x ms_big CTAs of one SM each, 128 at D = 256 and at D = 128, so one
//      wave on 132 SMs (256 at D = 64);
//   2. rgb_layers.0 (D / 2 rows, X = feat) as 64-column pieces, tc_wgrad_piece<64>: 4 pieces x 8 splits at D = 256.  The first ones
//      run on the SMs that grid 1 leaves free, the rest spread over all SMs when it ends.  Whole, this job made a second wave;
//   3. the encoding jobs (tc_wgrad<64>), which read only the dgrad stash;
//   4. the head jobs (head_wgrad).
// A chained grid starts once every CTA of the grid before it is resident.  The last CTA of each chained grid waits
// (griddepcontrol.wait) for the grid before it after storing its partials, so each grid completes only after every grid before it;
// one plain-launched wgrad_reduce then adds the splits of all 14 jobs.  Each job has its own region of the partial buffer, so the
// grids never write the same floats, and no two jobs write the same dW / db element (the encoding slice of layer 4 and the
// direction slice of rgb_layers.0 are at column offset D, enc[1] has no bias), so one reduce gives the same bits as one per grid.
// occ (nnb_field_grad with NNB_OCC_ONLY): the colour jobs (fc_feature, rgb_layers.0, fc_rgb) are left out, so grid 2 is not launched, the
// head grid runs the density head alone, and the colour parameters' gradients are not touched.  The kernels are those of the full stage.
// !bias (nnb_field_hvp_tc, whose tangent has no bias term): every job's db is NULL, so no bias slot of gw is touched.
// mcount (nnb_render_frame_train_bwd_tmin's reverse rounds): every grid runs on the first min(32 *mcount, L.M) rows, read on the device,
// with the split counts and partial regions of L.M (the _live kernels); at *mcount = L.M / 32 the results are those of mcount = NULL.
cudaError_t tc_wgrad_jobs(const nnb_render_args& a, const WsLayout& L, float* gw, bool occ, bool bias, cudaStream_t st,
                          const int* mcount = nullptr) {
  char* base = static_cast<char*>(a.workspace);
  auto F = [&](size_t off) { return reinterpret_cast<float*>(base + off); };
  const int D = L.D, DR = D / 2;
  WgJobT big[8], enc[2];
  int nb = 0;
  auto B = [&](size_t off) { return bias ? gw + off : nullptr; };
  for (int l = 1; l < 8; ++l) big[nb++] = WgJobT{F(L.dy[l]), F(L.h[l - 1]), gw + nnb::w_off(D, l), B(nnb::b_off(D, l)), D, D, D, D, nnb::w_ld(D, l), 0, 0};
  if (!occ) big[nb++] = WgJobT{F(L.dfeat), F(L.h[7]), gw + nnb::W_FEAT(D), gw + nnb::B_FEAT(D), D, D, D, D, D, 0, 0};
  const WgJobT rgb{F(L.dyr), F(L.feat), gw + nnb::W_RGBH(D), gw + nnb::B_RGBH(D), DR, DR, D, D, D + 27, 0, 0};
  enc[0] = WgJobT{F(L.dy[0]), F(L.enc), gw + nnb::w_off(D, 0), B(nnb::b_off(D, 0)), D, D, 64, 63, 63, 0, 0};
  enc[1] = WgJobT{F(L.dy[4]), F(L.enc), gw + nnb::w_off(D, 4) + D, nullptr, D, D, 64, 63, D + 63, 0, 0};
  const float* dyc = F(L.dyc);
  SmallJob sm[3] = {
      {dyc + 3, F(L.h[7]), gw + nnb::W_SIG(D), B(nnb::B_SIG(D)), 4, 1, D, D, D},
      {F(L.dyr), F(L.denc), gw + nnb::W_RGBH(D) + D, nullptr, DR, DR, 32, 27, D + 27},
      {dyc, F(L.hr), gw + nnb::W_RGB(D), gw + nnb::B_RGB(D), 4, 3, DR, DR, DR}};
  float* part = F(L.wpart);
  // sample splits: about one wave of 1-CTA-per-SM blocks per launch (16 | 4 row slices at D = 256)
  const int ms_big = L.M >= 8 * 128 ? tc_wgrad_msplit_big(D) : 1, ms_enc = L.M >= 32 * 64 ? 32 : 1;
  // Partial regions: D-wide jobs, rgb_layers.0, then heads, then encoding jobs.  In floats, np = num_params(D), at most 64 head
  // splits and 32 encoding splits: at D = 256 (D-wide + rgb) + heads = 4 491 264 + 270 592 <= 8 (np + 8192) = 4 832 288 <= wpart_floats,
  // and likewise at D = 128 (2 398 464 <= 2 669 632) and D = 64 (1 216 768 <= 1 686 656).  The encoding region (1 064 960 floats at
  // D = 256) fits as well only where wpart_floats is larger: at D = 256 when M > 36 864 (16 (np + 8192) at the C2 size), at D = 64
  // always, at D = 128 never.  Where it does not fit, the encoding jobs run after the chained reduce, with their own reduce, from
  // offset 0.
  const int nsm = occ ? 1 : 3;   // sm[0] is the density head
  const size_t trunk_f = wg_part_floats(big, nb, ms_big), big_f = trunk_f + (occ ? 0 : wg_part_floats(&rgb, 1, ms_big));
  const size_t head_f = small_jobs_part_floats(sm, nsm, L.M);
  const bool enc_chained = big_f + head_f + wg_part_floats(enc, 2, ms_enc) <= wpart_floats(L.M, D);
  RedJob R[9 + 2 + 3];
  cudaError_t e = D == 256 ? launch_wgrad<256>(big, nb, L.M, D, ms_big, part, 0, R, false, st, mcount)
                : D == 128 ? launch_wgrad<128>(big, nb, L.M, D, ms_big, part, 0, R, false, st, mcount)
                           : launch_wgrad<64>(big, nb, L.M, D, ms_big, part, 0, R, false, st, mcount);
  if (e != cudaSuccess) return e;
  int nr = nb;
  if (!occ) {
    e = launch_wgrad<64, true>(&rgb, 1, L.M, D, ms_big, part, trunk_f, R + nb, true, st, mcount);
    if (e != cudaSuccess) return e;
    nr += 1;
  }
  if (enc_chained) {   // encoding before heads: its CTAs need a whole SM each, and the small head CTAs would fragment the free SMs
    e = launch_wgrad<64>(enc, 2, L.M, D, ms_enc, part, big_f + head_f, R + nr, true, st, mcount);
    if (e != cudaSuccess) return e;
    nr += 2;
  }
  e = launch_head_wgrad(sm, nsm, L.M, D, part, big_f, R + nr, st, mcount);
  if (e != cudaSuccess) return e;
  nr += nsm;
  e = launch_wgrad_reduce(R, nr, part, st);
  if (e != cudaSuccess || enc_chained) return e;
  e = launch_wgrad<64>(enc, 2, L.M, D, ms_enc, part, 0, R, false, st, mcount);   // the chained reduce has read the whole buffer
  if (e != cudaSuccess) return e;
  return launch_wgrad_reduce(R, 2, part, st);
}
cudaError_t tc_wgrad_all(const nnb_render_args& a, const WsLayout& L, float* gw, cudaStream_t st) { return tc_wgrad_jobs(a, L, gw, false, true, st); }

// ---- data-gradient chain (the forward's skeleton run backwards) ---------------------------------------------------------------------
// Per 128-sample tile, two consumer warpgroups (64 rows each) and a producer warpgroup streaming TRANSPOSED weight stages: stage =
// `nrows` input features n x 16 output features k of one layer, element (n, k) = W[k * ldw + coloff + n], bf16 hi | lo (gradients
// span five decades).  A operand = the output gradient g_y of the current layer (bf16 hi | lo, K-major, rewritten in place by each
// epilogue); the epilogue applies the ReLU gate of the layer below (its gate bits from the forward, h > 0) and writes that layer's dY
// stash for the weight-gradient pass.  Order (matches the stage table): g_de = g_yr W_rgbh[:, 256:283] (N = 32),
// g_feat = g_yr W_rgbh[:, :256], g_h7 = g_feat W_feat + g_s w_sigma, then layers 7..1 (layer 4 first adds its encoding slice, N = 64)
// and layer 0 (encoding, N = 64).
template <int D>
__device__ __forceinline__ void prep_stage_t(const float* __restrict__ w, const StageDescT& sd, unsigned char* __restrict__ hi) {
  unsigned char* lo = hi + sd.nrows * 32;     // hi: [k-octet 0..1][nrows][8] bf16
  for (int idx = threadIdx.x; idx < sd.nrows * 2; idx += blockDim.x) {
    const int n = idx % sd.nrows, ko = idx / sd.nrows;
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int k = sd.k0 + ko * 8 + j;
      v[j] = (n < sd.nvalid && k < sd.kvalid) ? __ldg(w + sd.w_off + (size_t)k * sd.ldw + sd.coloff + n) : 0.f;
    }
    split_store8_bf16(v, hi + ko * sd.nrows * 16 + n * 16, lo + ko * sd.nrows * 16 + n * 16);
  }
}
template <int D>
__global__ void tc_prep_weights_t(const float* __restrict__ w, unsigned char* __restrict__ img) {
  const StageDescT sd = stage_t<D>(blockIdx.x);
  prep_stage_t<D>(w, sd, img + sd.img_off);
}
// the stages s0, s0 + 1, ... of the table into an image that starts at stage s0 (the trunk part of an occupancy-only chain)
template <int D>
__global__ void tc_prep_weights_t_from(const float* __restrict__ w, unsigned char* __restrict__ img, int s0) {
  const StageDescT sd = stage_t<D>(s0 + blockIdx.x);
  prep_stage_t<D>(w, sd, img + (sd.img_off - stage_t<D>(s0).img_off));
}

struct DgPtrs {
  const SampleRec* rec; const float4* gs; float4* gp; float4* gv; float4* dyc;
  const unsigned char* gates; float* dy[8]; float* dfeat; float* dyr;
};

// K-steps of one GEMM: D[64 x N] = A[64 x 16 ksteps] B^T, weight stages from the ring (released as their MMAs complete)
template <int D, int N>
__device__ __forceinline__ void dg_gemm(float* acc, uint32_t a_hi, uint32_t a_lo, int ksteps, uint32_t w_base, uint32_t bar0,
                                        uint32_t& slot, uint32_t& phase, int tl) {
  constexpr int STAGE_BYTES = Tc<D>::STAGE_BYTES;
  for (int s = 0; s < ksteps; ++s) {
    const uint32_t ko = (uint32_t)s * 4096u;
    const uint64_t dah = gdesc(a_hi + ko, 2048, 128), dal = gdesc(a_lo + ko, 2048, 128);
    const uint32_t wb = w_base + slot * STAGE_BYTES;
    const uint64_t dbh = gdesc(wb, N * 16, 128), dbl = gdesc(wb + N * 32, N * 16, 128);
    mbar_wait(bar0 + 8u * slot, phase);
    wgmma_fence();
    wgmma_bf16<N>(acc, dal, dbh, s > 0 ? 1u : 0u);
    wgmma_bf16<N>(acc, dah, dbl, 1u);
    wgmma_bf16<N>(acc, dah, dbh, 1u);
    wgmma_commit();
    if (s > 0) {
      wgmma_wait<1>();
      if (tl == 0) mbar_arrive(bar0 + 8u * (NST + (slot == 0 ? NST - 1 : slot - 1)));
    }
    if (++slot == NST) { slot = 0; phase ^= 1u; }
  }
  wgmma_wait<0>();
  if (tl == 0) mbar_arrive(bar0 + 8u * (NST + (slot == 0 ? NST - 1 : slot - 1)));
}

// MODE DG_RAYS (tc_dgrad, the render backward): rows are the samples of a.N rays, the records / cotangents / gradients are the
// workspace's [Mpad] arrays, and the dY stash is written when write_dy.  DG_POINTS / DG_POINTS_OCC (tc_points_vjp, nnb_field_vjp): rows
// are the explicit points a.pts [M]; P.gs is the caller's g_rgba [M] (rows >= M read as zero), P.gp / P.gv are g_pts / g_dirs [M] (P.gv
// may be NULL), only rows < M are stored and nothing is stashed.  DG_POINTS_OCC is the chain of an occupancy-only forward: it starts at
// g_h7 = g_s w_sigma (the colour prefix of the stage table is neither loaded nor issued) and reads only g_rgba[m].w.
// DEVN (points modes, nnb_geometry_frame): M = *count points, read when the kernel starts (see tc_fwd_body's DEVN).
// DG_POINTS_GRAD / DG_POINTS_GRAD_OCC (tc_points_grad, nnb_field_grad): DG_POINTS / DG_POINTS_OCC that also write the dY stash of every
// row of every tile, as DG_RAYS does with write_dy (rows >= M have a zero cotangent, so their dY are zeros); the occupancy-only chain
// writes dy0..dy7 and dyc = (0, 0, 0, d/d density logit).
// DG_POINTS_HVP_OCC (tc_points_hvp, nnb_field_hvp_tc): DG_POINTS_GRAD_OCC with the cotangent 1 on the logit of every row < M (P.gs is
// not read for it) and, in place of the first-order d p, the second-order point term of the tangent s' = u . d s / d p: from the
// encoding adjoint delta_enc and p, -u_c sum_l f^2 (delta_sin sin(f p_c) + delta_cos cos(f p_c)), f = 2^l, with u = P.gs[m].  P.gp may be
// NULL (no point term is stored).
// DG_FRAME (tc_dgrad_frame, nnb_render_frame_bwd): DG_RAYS on the rows of chunk `chunk` of every ray (M = 32 N, row m is sample
// chunk_sample(a, chunk, m)), the workspace arrays indexed by the row as tc_frame_stash wrote them.  With DEVN (tc_dgrad_frame_live): the
// rows of the live list `list` as tc_frame_stash_live wrote them, M = 32 *count (count clamped to 0..N) read when the kernel starts.
// DG_PACK (tc_dgrad_pack, nnb_render_bwd_tmin, DEVN): DG_RAYS on the packed stash of nnb_frame.cuh (M rows; its gate bits are laid out for
// M), on its first 32 count[C] rows (C = `chunk`, count = the rounds' counts, list = their lists), read when the kernel starts; row m is
// sample stash_row_sample(m).
enum : int { DG_RAYS = 0, DG_POINTS = 1, DG_POINTS_OCC = 2, DG_POINTS_GRAD = 3, DG_POINTS_GRAD_OCC = 4, DG_POINTS_HVP_OCC = 5, DG_FRAME = 6,
             DG_PACK = 7 };
template <int D, int MODE, bool DEVN = false>
__device__ __forceinline__ void tc_dgrad_body(const nnb_render_args& a, const unsigned char* __restrict__ wimg, const DgPtrs& P, size_t M,
                                              int n_tiles, int write_dy, const int* count = nullptr, int chunk = 0,
                                              const int* list = nullptr) {
  using T = Tc<D>;
  constexpr bool PACK = MODE == DG_PACK;
  constexpr bool HVP = MODE == DG_POINTS_HVP_OCC, CHUNK = MODE == DG_FRAME || PACK;
  static_assert(!PACK || DEVN, "the packed stash's row count is read on the device");
  const size_t m_cap = M;   // DG_PACK: rows of the packed stash
  constexpr bool PTS = MODE != DG_RAYS && !CHUNK, OCC = MODE == DG_POINTS_OCC || MODE == DG_POINTS_GRAD_OCC || HVP;
  constexpr bool GRAD = MODE == DG_POINTS_GRAD || MODE == DG_POINTS_GRAD_OCC || HVP;
  static_assert(!DEVN || (PTS && !GRAD) || CHUNK, "a device count of explicit points or of a frame round's rays");
  if constexpr (PTS) write_dy = GRAD ? 1 : 0;
  if constexpr (DEVN) {
    int c;   // rows
    if constexpr (PACK) c = 32 * min(max(count[chunk], 0), (int)(m_cap / 32));
    else if constexpr (CHUNK) c = 32 * frame_live_count(count, a.N);
    else c = *count;
    M = (size_t)c;
    n_tiles = (c + TILE - 1) / TILE;
    if ((int)blockIdx.x >= n_tiles) return;   // before any barrier exists
  }
  constexpr int DG_AHI = T::DG_AHI, DG_ALO = T::DG_ALO, DG_W = T::DG_W, DG_GENC = T::DG_GENC, DG_SMALL = T::DG_SMALL, DG_GYC = T::DG_GYC;
  constexpr int DG_BAR = T::DG_BAR, STAGE_BYTES = T::STAGE_BYTES, DR = D / 2;
  constexpr int S0 = T::dg_first_stage(OCC), S_END = S0 + T::dg_tile_stages(OCC);   // the stages of one tile
  constexpr int IMG0 = OCC ? (int)T::IMG_T_PREFIX_BYTES : 0;   // wimg holds the stages from S0 on
  // K-steps of the chain's GEMMs (constant expressions: Tc::dg_steps; every trunk layer has ST_TRUNK, static_assert in Tc)
  constexpr int ST_DE = T::dg_steps(0, OCC), ST_FEAT = T::dg_steps(1, OCC), ST_H7 = T::dg_steps(2, OCC), ST_TRUNK = T::dg_steps(3, OCC);
  constexpr int ST_ENC4 = T::dg_steps(10, OCC), ST_ENC0 = T::dg_steps(11, OCC);
  extern __shared__ __align__(1024) unsigned char smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* s_small = reinterpret_cast<float*>(smem + DG_SMALL);
  const uint32_t bar0 = smem_u32(smem + DG_BAR);
  if (threadIdx.x == 0) {
    for (int i = 0; i < NST; ++i) { mbar_init(bar0 + 8u * i, 1); mbar_init(bar0 + 8u * (NST + i), 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (int i = threadIdx.x; i < 5 * DR; i += blockDim.x)
    s_small[i] = (i < 3 * DR) ? __ldg(a.weights + nnb::W_RGB(D) + i) : __ldg(a.weights + nnb::W_SIG(D) + (i - 3 * DR));
  __syncthreads();
  const int my_tiles = (n_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
  // GRAD: each warpgroup forms the tile count again after its setmaxnreg instead of holding it across (which spilled it at D = 256)
  auto cta_tiles = [&]() {
    if constexpr (GRAD) return ((int)computed_here((uint32_t)n_tiles) - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
    else return my_tiles;
  };
  if (warp >= 8) {   // weight producer (see tc_field_fwd)
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
    if (warp == 8 && lane == 0) {
      uint32_t slot = 0, phase = 0;
      const int n_my = cta_tiles();
      for (int t = 0; t < n_my; ++t)
        for (int s = S0; s < S_END; ++s) {
          const uint32_t bytes = (uint32_t)stage_t<D>(s).nrows * 64u;
          mbar_wait(bar0 + 8u * (NST + slot), phase ^ 1u);
          mbar_expect_tx(bar0 + 8u * slot, bytes);
          bulk_g2s(smem_u32(smem + DG_W + slot * STAGE_BYTES), wimg + (stage_t<D>(s).img_off - IMG0), bytes, bar0 + 8u * slot);
          if (++slot == NST) { slot = 0; phase ^= 1u; }
        }
    }
    return;
  }
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
  const int wg = warp >> 2, tl = threadIdx.x & 127;
  const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2), c0 = (lane & 3) * 2;
  float* genc = reinterpret_cast<float*>(smem + DG_GENC) + wg * 64 * 64;   // [64 rows][64] encoding gradient; [64][32] g_de before
  float* gyc = reinterpret_cast<float*>(smem + DG_GYC) + wg * 64 * 4;
  const uint32_t a_hi = smem_u32(smem + DG_AHI) + wg * 1024, a_lo = smem_u32(smem + DG_ALO) + wg * 1024;
  const uint32_t w_base = smem_u32(smem + DG_W);
  const uint32_t bar_id = 1u + (uint32_t)wg;
  auto wg_sync = [&]() { asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory"); };
  uint32_t slot = 0, phase = 0;
  float acc[D / 2];   // the 32- / 64-wide GEMMs use its first registers (every result is consumed before the next GEMM)
  // ReLU gate bits of the layer below the next epilogue (the rgb hidden layer's for the head prologue), loaded before the GEMM that
  // precedes that epilogue so the load completes behind its MMAs
  uint32_t gm[D / 64];
  const size_t Mpad = PACK ? m_cap : (size_t)n_tiles * TILE;
  // epilogue of a D-wide layer: x (+ g_s w_sigma) -> ReLU gate gm (when `gated`) -> dY stash -> next A operand (in place)
  auto epiD = [&](size_t mt, bool gated, float* dst, bool add_sigma) {
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int row = r0 + 8 * r;
      const size_t rowoff = (mt + row) * D + c0;
      const float g_s = add_sigma ? gyc[(row - wg * 64) * 4 + 3] : 0.f;
      unsigned char* ahi = smem + DG_AHI + row * 16 + c0 * 2;
#pragma unroll
      for (int j = 0; j < D / 8; ++j) {
        float v0 = acc[4 * j + 2 * r], v1 = acc[4 * j + 2 * r + 1];
        if (add_sigma) { v0 += g_s * s_small[3 * DR + j * 8 + c0]; v1 += g_s * s_small[3 * DR + j * 8 + c0 + 1]; }
        if (gated) {
          const uint32_t b = gm[j / 8] << (4 * (j & 7) + 2 * r);   // gate bits of columns c0 and c0 + 1 at bits 31 and 30
          v0 = (b & 0x80000000u) ? v0 : 0.f; v1 = (b & 0x40000000u) ? v1 : 0.f;
        }
        if (dst) __stcs(reinterpret_cast<float2*>(dst + rowoff + j * 8), make_float2(v0, v1));
        uint32_t hw, lw;
        split2_bf16(v0, v1, hw, lw);
        *reinterpret_cast<uint32_t*>(ahi + j * 2048) = hw;
        *reinterpret_cast<uint32_t*>(ahi + DG_ALO + j * 2048) = lw;
      }
    }
    fence_async_smem();
    wg_sync();
  };
  auto epi_enc = [&](bool add) {   // 64-wide encoding gradient -> genc
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        float* g = genc + (r0 + 8 * r - wg * 64) * 64 + j * 8 + c0;
        if (add) { g[0] += acc[4 * j + 2 * r]; g[1] += acc[4 * j + 2 * r + 1]; }
        else { g[0] = acc[4 * j + 2 * r]; g[1] = acc[4 * j + 2 * r + 1]; }
      }
  };

  const int n_my = cta_tiles();
  for (int t = 0; t < n_my; ++t) {
    const int tile = blockIdx.x + t * gridDim.x;
    const size_t mt = (size_t)tile * TILE;
    load_gates<OCC ? D / 2 : D / 4>(P.gates + gate_bits_off(OCC ? 7 : 8, tile, threadIdx.x, Mpad, D), gm);
    wg_sync();   // the previous tile's encoding adjoint is done with genc
    if (tl < 64) {   // head adjoints (one thread per row)
      const size_t m = mt + wg * 64 + tl;
      if constexpr (OCC) {
        float gw;
        if constexpr (HVP) gw = (m < M) ? 1.f : 0.f;
        else gw = (m < M) ? reinterpret_cast<const float*>(P.gs + m)[3] : 0.f;
        gyc[tl * 4 + 3] = gw * density_act_grad(P.rec[m].s, a.flags);
        if constexpr (GRAD) __stcs(P.dyc + m, make_float4(0.f, 0.f, 0.f, gyc[tl * 4 + 3]));
      } else {
        const float4 g = (m < M) ? P.gs[m] : make_float4(0.f, 0.f, 0.f, 0.f);
        const SampleRec rec = P.rec[m];
        const float g0 = g.x * rec.r * (1.f - rec.r), g1 = g.y * rec.g * (1.f - rec.g), g2 = g.z * rec.b * (1.f - rec.b);
        const float g3 = g.w * density_act_grad(rec.s, a.flags);
        if (write_dy) __stcs(P.dyc + m, make_float4(g0, g1, g2, g3));
        gyc[tl * 4] = g0; gyc[tl * 4 + 1] = g1; gyc[tl * 4 + 2] = g2; gyc[tl * 4 + 3] = g3;
      }
    }
    wg_sync();
    if constexpr (OCC) {   // g_h7 = (g_s w_sigma) * (h7 > 0)
#pragma unroll
      for (int i = 0; i < D / 2; ++i) acc[i] = 0.f;
      epiD(mt, true, GRAD ? P.dy[7] : nullptr, true);
    } else {
      {   // g_yr = (g_yc W_rgb) * (hr > 0), in the accumulator-fragment mapping of the gate bits -> A operand (K = D/2) + dY stash
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const int row = r0 + 8 * r;
          const float* g4 = gyc + (row - wg * 64) * 4;
          unsigned char* ahi = smem + DG_AHI + row * 16 + c0 * 2;
#pragma unroll
          for (int j = 0; j < DR / 8; ++j) {
            const int col = j * 8 + c0;
            const float x0 = g4[0] * s_small[col] + g4[1] * s_small[DR + col] + g4[2] * s_small[2 * DR + col];
            const float x1 = g4[0] * s_small[col + 1] + g4[1] * s_small[DR + col + 1] + g4[2] * s_small[2 * DR + col + 1];
            const uint32_t b = gm[j / 8] << (4 * (j & 7) + 2 * r);
            const float v0 = (b & 0x80000000u) ? x0 : 0.f, v1 = (b & 0x40000000u) ? x1 : 0.f;
            if (write_dy) __stcs(reinterpret_cast<float2*>(P.dyr + (mt + row) * DR + col), make_float2(v0, v1));
            uint32_t hw, lw;
            split2_bf16(v0, v1, hw, lw);
            *reinterpret_cast<uint32_t*>(ahi + j * 2048) = hw;
            *reinterpret_cast<uint32_t*>(ahi + DG_ALO + j * 2048) = lw;
          }
        }
      }
      fence_async_smem();
      wg_sync();
      // g_de (direction-encoding slice of rgb_layers.0) -> view-direction adjoint
      dg_gemm<D, 32>(acc, a_hi, a_lo, ST_DE, w_base, bar0, slot, phase, tl);
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          float* g = genc + (r0 + 8 * r - wg * 64) * 32 + j * 8 + c0;
          g[0] = acc[4 * j + 2 * r]; g[1] = acc[4 * j + 2 * r + 1];
        }
      wg_sync();
      if (tl < 64) {
        const size_t m = mt + wg * 64 + tl, mm = m < M ? m : M - 1;
        Ray ray; float z, p[3], v[3], gvd[3];
        if constexpr (PTS) {
#pragma unroll
          for (int c = 0; c < 3; ++c) v[c] = a.dirs ? __ldg(a.dirs + 3 * mm + c) : 1.f;
        } else {
          if constexpr (PACK) sample_geometry(a, stash_row_sample(a, list, count, chunk, m), ray, z, p);
          else if constexpr (CHUNK && DEVN) sample_geometry(a, live_sample(a, chunk, list, (int)(M >> 5), m), ray, z, p);
          else if constexpr (CHUNK) chunk_geometry(a, chunk, m, ray, z, p);
          else row_geometry_tc(a, m, M, ray, z, p);
          if (a.pts) {
#pragma unroll
            for (int c = 0; c < 3; ++c) v[c] = a.dirs ? __ldg(a.dirs + 3 * mm + c) : 1.f;
          } else {
            view_dir(a, ray, v);
          }
        }
        const float* ge = genc + tl * 32;
        encode_bwd<4>(v, [&](int k) { return ge[k]; }, gvd);
        if (!PTS || (P.gv && m < M)) P.gv[m] = make_float4(gvd[0], gvd[1], gvd[2], 0.f);
      }
      dg_gemm<D, D>(acc, a_hi, a_lo, ST_FEAT, w_base, bar0, slot, phase, tl);   // g_feat
      epiD(mt, false, write_dy ? P.dfeat : nullptr, false);
      load_gates<D / 2>(P.gates + gate_bits_off(7, tile, threadIdx.x, Mpad, D), gm);
      dg_gemm<D, D>(acc, a_hi, a_lo, ST_H7, w_base, bar0, slot, phase, tl);   // g_h7 = g_feat W_feat + g_s w_sigma
      epiD(mt, true, write_dy ? P.dy[7] : nullptr, true);
    }
    for (int l = 7; l >= 1; --l) {
      load_gates<D / 2>(P.gates + gate_bits_off(l - 1, tile, threadIdx.x, Mpad, D), gm);
      if (l == 4) { dg_gemm<D, 64>(acc, a_hi, a_lo, ST_ENC4, w_base, bar0, slot, phase, tl); epi_enc(false); }
      dg_gemm<D, D>(acc, a_hi, a_lo, ST_TRUNK, w_base, bar0, slot, phase, tl);   // g_h(l-1) = dY_l W_l
      epiD(mt, true, write_dy ? P.dy[l - 1] : nullptr, false);
    }
    dg_gemm<D, 64>(acc, a_hi, a_lo, ST_ENC0, w_base, bar0, slot, phase, tl);   // encoding gradient of layer 0
    epi_enc(true);
    wg_sync();
    if (tl < 64) {   // encoding adjoint -> d p
      const size_t m = mt + wg * 64 + tl;
      Ray ray; float z, p[3], gp[3];
      if constexpr (PTS) {
        const size_t mm = m < M ? m : M - 1;
#pragma unroll
        for (int c = 0; c < 3; ++c) p[c] = __ldg(a.pts + 3 * mm + c);
      } else if constexpr (PACK) {
        sample_geometry(a, stash_row_sample(a, list, count, chunk, m), ray, z, p);
      } else if constexpr (CHUNK && DEVN) {
        sample_geometry(a, live_sample(a, chunk, list, (int)(M >> 5), m), ray, z, p);
      } else if constexpr (CHUNK) {
        chunk_geometry(a, chunk, m, ray, z, p);
      } else {
        row_geometry_tc(a, m, M, ray, z, p);
      }
      const float* ge = genc + tl * 64;
      if constexpr (HVP) {   // the point term of simt_field_tangent, in its order and rounding
        if (P.gp && m < M) {
          const float4 uv = P.gs[m];
          const float u[3] = {uv.x, uv.y, uv.z};
#pragma unroll
          for (int c = 0; c < 3; ++c) {
            float s2 = 0.f;
#pragma unroll
            for (int l = 0; l < 10; ++l) {
              const float f = (float)(1 << l);
              float sn, cs; sincosf(__fmul_rn(f, p[c]), &sn, &cs);
              s2 = fmaf(__fmul_rn(f, f), fmaf(ge[3 + 6 * l + c], sn, __fmul_rn(ge[6 + 6 * l + c], cs)), s2);
            }
            gp[c] = -__fmul_rn(s2, u[c]);
          }
          P.gp[m] = make_float4(gp[0], gp[1], gp[2], 0.f);
        }
      } else {
        encode_bwd<10>(p, [&](int k) { return ge[k]; }, gp);
        if (!PTS || m < M) P.gp[m] = make_float4(gp[0], gp[1], gp[2], 0.f);
      }
    }
  }
}

template <int D>
__global__ void __launch_bounds__(N_THREADS, 1) tc_dgrad(nnb_render_args a, const unsigned char* __restrict__ wimg,
                                                         const __grid_constant__ DgPtrs P, size_t M,
                                                         int n_tiles, int write_dy) {
  tc_dgrad_body<D, DG_RAYS>(a, wimg, P, M, n_tiles, write_dy);
}
// the chain of one reverse round of nnb_render_frame_bwd on chunk k's stash (M = 32 N)
template <int D>
__global__ void __launch_bounds__(N_THREADS, 1) tc_dgrad_frame(nnb_render_args a, const unsigned char* __restrict__ wimg,
                                                               const __grid_constant__ DgPtrs P, size_t M, int n_tiles, int write_dy, int k) {
  tc_dgrad_body<D, DG_FRAME>(a, wimg, P, M, n_tiles, write_dy, nullptr, k);
}
// tc_dgrad_frame on the rays of round k's live list (*count of them; the launch is sized for N)
template <int D>
__global__ void __launch_bounds__(N_THREADS, 1) tc_dgrad_frame_live(nnb_render_args a, const unsigned char* __restrict__ wimg,
                                                                    const __grid_constant__ DgPtrs P, int write_dy, int k,
                                                                    const int* __restrict__ count, const int* __restrict__ list) {
  tc_dgrad_body<D, DG_FRAME, true>(a, wimg, P, 0, 0, write_dy, count, k, list);
}
// the chain of nnb_render_bwd_tmin on the packed stash of M rows, over its first 32 counts[C] rows (DG_PACK; the launch is sized for M)
template <int D>
__global__ void __launch_bounds__(N_THREADS, 1) tc_dgrad_pack(nnb_render_args a, const unsigned char* __restrict__ wimg,
                                                              const __grid_constant__ DgPtrs P, size_t M, int write_dy, int C,
                                                              const int* __restrict__ counts, const int* __restrict__ lists) {
  tc_dgrad_body<D, DG_PACK, true>(a, wimg, P, M, 0, write_dy, counts, C, lists);
}

// nnb_field_vjp: the forward of explicit points with records and gate bits (FWD_VJP), then the chain on them (DG_POINTS[_OCC])
template <int D>
__global__ void __launch_bounds__(N_THREADS, 1) tc_points_vjp_fwd(nnb_render_args a, const unsigned char* __restrict__ wimg,
                                                                  SampleRec* __restrict__ recs, float4* __restrict__ out,
                                                                  unsigned char* __restrict__ gates, size_t M, int n_tiles) {
  TcStash st{};
  st.gates = gates;
  tc_fwd_body<D, FWD_VJP>(a, wimg, recs, out, st, MarchPtrs{}, M, n_tiles, 0);
}
template <int D, int MODE>
__global__ void __launch_bounds__(N_THREADS, 1) tc_points_vjp(nnb_render_args a, const unsigned char* __restrict__ wimg,
                                                              const __grid_constant__ DgPtrs P, size_t M, int n_tiles) {
  tc_dgrad_body<D, MODE>(a, wimg, P, M, n_tiles, 0);
}
// the two kernels of nnb_field_vjp on the *count points of nnb_geometry_frame
template <int D>
__global__ void __launch_bounds__(N_THREADS, 1) tc_points_vjp_fwd_n(nnb_render_args a, const unsigned char* __restrict__ wimg,
                                                                    SampleRec* __restrict__ recs, float4* __restrict__ out,
                                                                    unsigned char* __restrict__ gates, const int* __restrict__ count) {
  TcStash st{};
  st.gates = gates;
  MarchPtrs q{};
  q.count = count;
  tc_fwd_body<D, FWD_VJP, true>(a, wimg, recs, out, st, q, 0, 0, 0);
}
template <int D, int MODE>
__global__ void __launch_bounds__(N_THREADS, 1) tc_points_vjp_n(nnb_render_args a, const unsigned char* __restrict__ wimg,
                                                                const __grid_constant__ DgPtrs P, const int* __restrict__ count) {
  tc_dgrad_body<D, MODE, true>(a, wimg, P, 0, 0, 0, count);
}
// nnb_field_grad: the forward of explicit points with records, gate bits and the fp32 training stash (FWD_GRAD), then the chain with
// the dY stash (DG_POINTS_GRAD[_OCC]); tc_wgrad_jobs follows on that stash
template <int D>
__global__ void __launch_bounds__(N_THREADS, 1) tc_points_grad_fwd(nnb_render_args a, const unsigned char* __restrict__ wimg,
                                                                   SampleRec* __restrict__ recs, float4* __restrict__ out,
                                                                   const __grid_constant__ TcStash st, size_t M, int n_tiles) {
  tc_fwd_body<D, FWD_GRAD>(a, wimg, recs, out, st, MarchPtrs{}, M, n_tiles, 1);
}
template <int D, int MODE>
__global__ void __launch_bounds__(N_THREADS, 1) tc_points_grad(nnb_render_args a, const unsigned char* __restrict__ wimg,
                                                               const __grid_constant__ DgPtrs P, size_t M, int n_tiles) {
  tc_dgrad_body<D, MODE>(a, wimg, P, M, n_tiles, 1);
}
// nnb_field_hvp_tc, after the occupancy-only tc_points_vjp_fwd: the chain for a cotangent 1 on the logit with the dY stash and the point
// term (DG_POINTS_HVP_OCC), and the tangent chain (FWD_TANGENT, u read through the output pointer) into the tangent stash st
template <int D>
__global__ void __launch_bounds__(N_THREADS, 1) tc_points_hvp(nnb_render_args a, const unsigned char* __restrict__ wimg,
                                                              const __grid_constant__ DgPtrs P, size_t M, int n_tiles) {
  tc_dgrad_body<D, DG_POINTS_HVP_OCC>(a, wimg, P, M, n_tiles, 1);
}
template <int D>
__global__ void __launch_bounds__(N_THREADS, 1) tc_points_tangent(nnb_render_args a, const unsigned char* __restrict__ wimg,
                                                                  const float4* __restrict__ u, const __grid_constant__ TcStash st, size_t M,
                                                                  int n_tiles) {
  tc_fwd_body<D, FWD_TANGENT>(a, wimg, nullptr, const_cast<float4*>(u), st, MarchPtrs{}, M, n_tiles, 1);
}

template <int D>
cudaError_t upload_stage_table_t() {
  using T = Tc<D>;
  static bool ready = false;
  if (ready) return cudaSuccess;
  StageDescT h[T::N_STAGES_T];
  int s = 0, off = 0;
  auto add = [&](int w_off, int ldw, int coloff, int nvalid, int k0, int kvalid, int nrows) {
    h[s] = StageDescT{w_off, ldw, coloff, nvalid, k0, kvalid, nrows, off};
    off += nrows * 64; ++s;
  };
  constexpr int DR = D / 2, KS = T::KS;
  for (int i = 0; i < DR / 16; ++i) add(nnb::W_RGBH(D), D + 27, D, 27, 16 * i, DR, 32);
  for (int i = 0; i < DR / 16; ++i) add(nnb::W_RGBH(D), D + 27, 0, D, 16 * i, DR, D);
  for (int i = 0; i < KS; ++i) add(nnb::W_FEAT(D), D, 0, D, 16 * i, D, D);
  // A producer that waits for a stage no consumer takes never returns: the chain's bounds (Tc::dg_steps) must be the table's, for the
  // whole chain and for the occupancy-only chain, which starts here
  if (s != T::dg_first_stage(true) || (size_t)off != T::IMG_T_PREFIX_BYTES) return cudaErrorInvalidValue;
  for (int l = 7; l >= 1; --l) {
    if (l == 4) for (int i = 0; i < KS; ++i) add(nnb::w_off(D, 4), D + 63, D, 63, 16 * i, D, 64);
    for (int i = 0; i < KS; ++i) add(nnb::w_off(D, l), nnb::w_ld(D, l), 0, D, 16 * i, D, D);
  }
  for (int i = 0; i < KS; ++i) add(nnb::w_off(D, 0), 63, 0, 63, 16 * i, D, 64);
  if (s != T::dg_tile_stages(false) || s - T::dg_first_stage(true) != T::dg_tile_stages(true) || (size_t)off != T::IMG_T_BYTES)
    return cudaErrorInvalidValue;
  cudaError_t e;
  if constexpr (D == 256) e = cudaMemcpyToSymbol(c_stages_t_256, h, sizeof(h));
  else if constexpr (D == 128) e = cudaMemcpyToSymbol(c_stages_t_128, h, sizeof(h));
  else e = cudaMemcpyToSymbol(c_stages_t_64, h, sizeof(h));
  if (e == cudaSuccess) ready = true;
  return e;
}

// the data-gradient stage of the TC engine's backward (stash layout of nnb_simt.cu)
template <int D>
cudaError_t tc_dgrad_launch_dim(const nnb_render_bwd_args& b, const WsLayout& L, int write_dy, cudaStream_t st) {
  using T = Tc<D>;
  const nnb_render_args& a = b.fwd;
  cudaError_t e = upload_stage_table_t<D>();
  if (e != cudaSuccess) return e;
  static bool attr = false;
  static int n_sm = 0;
  if (!attr) {
    e = cudaFuncSetAttribute(tc_dgrad<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, T::DG_TOTAL);
    if (e != cudaSuccess) return e;
    int dev = 0; cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
    attr = true;
  }
  char* base = static_cast<char*>(a.workspace);
  auto F = [&](size_t off) { return reinterpret_cast<float*>(base + off); };
  unsigned char* img = reinterpret_cast<unsigned char*>(base + L.total + align_up(T::IMG_BYTES, 256));
  DgPtrs P{};
  P.rec = reinterpret_cast<const SampleRec*>(base + L.rec);
  P.gs = reinterpret_cast<const float4*>(base + L.gs); P.gp = reinterpret_cast<float4*>(base + L.gp); P.gv = reinterpret_cast<float4*>(base + L.gv);
  P.dyc = reinterpret_cast<float4*>(base + L.dyc);
  for (int l = 0; l < 8; ++l) P.dy[l] = F(L.dy[l]);
  P.gates = reinterpret_cast<const unsigned char*>(base + L.gates); P.dfeat = F(L.dfeat); P.dyr = F(L.dyr);
  tc_prep_weights_t<D><<<T::N_STAGES_T, 256, 0, st>>>(a.weights, img);
  const int n_tiles = (int)((L.M + TILE - 1) / TILE);
  const int grid = n_tiles < n_sm ? n_tiles : n_sm;
  tc_dgrad<D><<<grid, N_THREADS, T::DG_TOTAL, st>>>(a, (const unsigned char*)img, P, L.M, n_tiles, write_dy);
  return cudaGetLastError();
}

cudaError_t tc_dgrad_launch(const nnb_render_bwd_args& b, const WsLayout& L, int write_dy, cudaStream_t st) {
  return L.D == 128 ? tc_dgrad_launch_dim<128>(b, L, write_dy, st)
       : L.D == 64  ? tc_dgrad_launch_dim<64>(b, L, write_dy, st) : tc_dgrad_launch_dim<256>(b, L, write_dy, st);
}

template <int D>
cudaError_t upload_stage_table() {
  using T = Tc<D>;
  static bool ready = false;
  if (ready) return cudaSuccess;
  StageDesc h[T::N_STAGES_PTS];
  int s = 0, off = 0;
  auto add = [&](int w_off, int ldw, int kcol0, int kvalid, int nrows) {
    h[s].w_off = w_off; h[s].ldw = ldw; h[s].kcol0 = kcol0; h[s].kvalid = kvalid; h[s].nrows = nrows; h[s].img_off = off;
    off += nrows * 64; ++s;
  };
  // per layer, one stage per K-step of 16; the encoding K-steps (layers 0 and 4) come first
  constexpr int KS = Tc<D>::KS;
  for (int i = 0; i < 4; ++i) add(nnb::w_off(D, 0), 63, 16 * i, 63, D);
  for (int l = 1; l < 8; ++l) {
    if (l == 4) for (int i = 0; i < 4; ++i) add(nnb::w_off(D, 4), D + 63, D + 16 * i, D + 63, D);
    for (int i = 0; i < KS; ++i) add(nnb::w_off(D, l), nnb::w_ld(D, l), 16 * i, D, D);
  }
  // A producer that waits for a stage no consumer takes never returns: the counts the kernels loop over (Tc::tile_stages) must be
  // the table's, for rays, for points and for the occupancy-only prefix.
  if (s != T::N_STAGES_OCC) return cudaErrorInvalidValue;
  for (int i = 0; i < KS; ++i) add(nnb::W_FEAT(D), D, 16 * i, D, D);
  for (int i = 0; i < KS; ++i) add(nnb::W_RGBH(D), D + 27, 16 * i, D, D / 2);
  if (s != T::N_STAGES || (size_t)off != T::IMG_BYTES) return cudaErrorInvalidValue;
  for (int i = 0; i < 2; ++i) add(nnb::W_RGBH(D), D + 27, D + 16 * i, D + 27, D / 2);   // points mode: the direction columns
  if (s != T::N_STAGES_PTS || (size_t)off != T::IMG_PTS_BYTES) return cudaErrorInvalidValue;
  cudaError_t e;
  if constexpr (D == 256) e = cudaMemcpyToSymbol(c_stages_256, h, sizeof(h));
  else if constexpr (D == 128) e = cudaMemcpyToSymbol(c_stages_128, h, sizeof(h));
  else e = cudaMemcpyToSymbol(c_stages_64, h, sizeof(h));
  if (e == cudaSuccess) ready = true;
  return e;
}

template <int D>
cudaError_t tc_render_fwd_dim(const nnb_render_args& a, const WsLayout& L, cudaStream_t st) {
  using T = Tc<D>;
  cudaError_t e = upload_stage_table<D>();
  if (e != cudaSuccess) return e;
  static bool attr = false;
  static int n_sm = 0;
  if (!attr) {
    e = cudaFuncSetAttribute(tc_field_fwd<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, T::SM_TOTAL);
    if (e != cudaSuccess) return e;
    int dev = 0; cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
    attr = true;
  }
  char* base = static_cast<char*>(a.workspace);
  unsigned char* img = reinterpret_cast<unsigned char*>(base + L.total);
  SampleRec* recs = reinterpret_cast<SampleRec*>(base + L.rec);
  TcStash ts{};
  const int stash = (a.flags & NNB_STASH) ? 1 : 0;
  if (stash) {
    for (int l = 0; l < 8; ++l) ts.h[l] = reinterpret_cast<float*>(base + L.h[l]);
    ts.feat = reinterpret_cast<float*>(base + L.feat); ts.hr = reinterpret_cast<float*>(base + L.hr);
    ts.enc = reinterpret_cast<float*>(base + L.enc); ts.denc = reinterpret_cast<float*>(base + L.denc);
    ts.gates = reinterpret_cast<unsigned char*>(base + L.gates);
  }
  nnb_prof_mark(st);
  tc_prep_weights<D><<<T::N_STAGES, 256, 0, st>>>(a.weights, img);   // 152 stage images (fp16 hi | lo) at D = 256
  nnb_prof_mark(st);
  const int n_tiles = (int)((L.M + TILE - 1) / TILE);
  const int grid = n_tiles < n_sm ? n_tiles : n_sm;
  tc_field_fwd<D><<<grid, N_THREADS, T::SM_TOTAL, st>>>(a, (const unsigned char*)img, recs, ts, L.M, n_tiles, stash);
  nnb_prof_mark(st);
  e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  e = launch_composite_fwd(a, recs, st);
  nnb_prof_mark(st);
  return e;
}

// the points forward: weight image into img, then a.pts / a.dirs [M][3] -> out [M][4].  count (nnb_geometry_frame): M = *count <= a.N,
// read on the device; the launch is sized for a.N.
template <int D>
cudaError_t tc_points_fwd_launch(const nnb_render_args& a, unsigned char* img, float* out_rgba, size_t M, const int* count, cudaStream_t st) {
  using T = Tc<D>;
  cudaError_t e = upload_stage_table<D>();
  if (e != cudaSuccess) return e;
  static bool attr = false;
  static int n_sm = 0;
  if (!attr) {
    e = cudaFuncSetAttribute(tc_points_fwd<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, T::SM_TOTAL);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(tc_points_fwd_n<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, T::SM_TOTAL);
    if (e != cudaSuccess) return e;
    int dev = 0; cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
    attr = true;
  }
  const int n_st = (a.flags & NNB_OCC_ONLY) ? T::N_STAGES_OCC : T::N_STAGES_PTS;   // the stages the kernel walks
  tc_prep_weights<D><<<n_st, 256, 0, st>>>(a.weights, img);
  const int n_tiles = (int)((M + TILE - 1) / TILE);
  const int grid = n_tiles < n_sm ? n_tiles : n_sm;
  if (count) tc_points_fwd_n<D><<<grid, N_THREADS, T::SM_TOTAL, st>>>(a, (const unsigned char*)img, reinterpret_cast<float4*>(out_rgba), count);
  else tc_points_fwd<D><<<grid, N_THREADS, T::SM_TOTAL, st>>>(a, (const unsigned char*)img, reinterpret_cast<float4*>(out_rgba), M, n_tiles);
  return cudaGetLastError();
}

// nnb_field_fwd on this engine: a.pts / a.dirs [L.M][3] -> out_rgba [L.M][4]
template <int D>
cudaError_t tc_points_fwd_dim(const nnb_render_args& a, const WsLayout& L, float* out_rgba, cudaStream_t st) {
  return tc_points_fwd_launch<D>(a, reinterpret_cast<unsigned char*>(static_cast<char*>(a.workspace) + L.total), out_rgba, L.M, nullptr, st);
}

// Workspace of nnb_ray_march: march_layout_bytes (nnb_march.cuh) with the weight image of the occupancy-only stages as its own part
template <int D> MarchWs march_layout(int N, int n_steps) {
  return march_layout_bytes(N, n_steps, (size_t)Tc<D>::N_STAGES_OCC * Tc<D>::STAGE_BYTES);
}

// nnb_ray_march: weight image once, then run_ray_march with one tc_march launch per 128-step block and tc_secant over the hit rays
template <int D>
cudaError_t tc_ray_march_dim(const nnb_ray_march_args& r, cudaStream_t st) {
  using T = Tc<D>;
  cudaError_t e = upload_stage_table<D>();
  if (e != cudaSuccess) return e;
  static bool attr = false;
  static int n_sm = 0;
  if (!attr) {
    e = cudaFuncSetAttribute(tc_march<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, T::SM_TOTAL);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(tc_secant<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, T::SM_TOTAL);
    if (e != cudaSuccess) return e;
    int dev = 0; cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
    attr = true;
  }
  const MarchWs w = march_layout<D>(r.N, r.n_steps);
  unsigned char* img = static_cast<unsigned char*>(r.workspace) + w.img;
  tc_prep_weights<D><<<T::N_STAGES_OCC, 256, 0, st>>>(r.weights, img);
  const int grid = r.N < n_sm ? r.N : n_sm, tiles = (r.N + TILE - 1) / TILE;
  return run_ray_march(
      r, w, D, st, [&](const nnb_render_args& a, const MarchPtrs& q) { tc_march<D><<<grid, N_THREADS, T::SM_TOTAL, st>>>(a, img, q, r.N); },
      [&](const nnb_render_args& a, const MarchPtrs& q) { tc_secant<D><<<tiles < n_sm ? tiles : n_sm, N_THREADS, T::SM_TOTAL, st>>>(a, img, q); });
}

// Workspace of nnb_field_vjp, every section 256-byte aligned: records [Npad] | gate bits (gate_bits_off; h0..h7 only when occ) | forward
// weight image (the occupancy-only prefix when occ) | transposed weight image (its trunk part, from dg_first_stage(true) on, when occ)
struct VjpWs { size_t rec, gates, img, img_t, total; };
template <int D> VjpWs vjp_layout(int N, bool occ) {
  using T = Tc<D>;
  const size_t Npad = align_up((size_t)N, TILE);
  VjpWs w{};
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t o = off; off += align_up(bytes, 256); return o; };
  w.rec = take(Npad * sizeof(SampleRec));
  w.gates = take(occ ? Npad * D : gate_bits_bytes(Npad, D));
  w.img = take(occ ? (size_t)T::N_STAGES_OCC * T::STAGE_BYTES : T::IMG_PTS_BYTES);
  w.img_t = take(occ ? T::IMG_T_BYTES - T::IMG_T_PREFIX_BYTES : T::IMG_T_BYTES);
  w.total = off;
  return w;
}

// nnb_field_vjp: both weight images, the forward with records and gate bits, the chain.  count (nnb_geometry_frame, occupancy-only):
// the points are the first *count <= a.N rows, read on the device; the workspace and the launches are sized for a.N.
template <int D>
cudaError_t tc_field_vjp_dim(const nnb_render_args& a, const float* g_rgba, float* out_rgba, float* g_pts, float* g_dirs, cudaStream_t st,
                             const int* count = nullptr) {
  using T = Tc<D>;
  const bool occ = (a.flags & NNB_OCC_ONLY) != 0;
  if (count && !occ) return cudaErrorInvalidValue;   // only the occupancy-only chain has a device-count instantiation
  cudaError_t e = upload_stage_table<D>();
  if (e == cudaSuccess) e = upload_stage_table_t<D>();
  if (e != cudaSuccess) return e;
  static bool attr = false;
  static int n_sm = 0;
  if (!attr) {
    e = cudaFuncSetAttribute(tc_points_vjp_fwd<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, T::SM_TOTAL);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(tc_points_vjp<D, DG_POINTS>, cudaFuncAttributeMaxDynamicSharedMemorySize, T::DG_TOTAL);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(tc_points_vjp<D, DG_POINTS_OCC>, cudaFuncAttributeMaxDynamicSharedMemorySize, T::DG_TOTAL);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(tc_points_vjp_fwd_n<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, T::SM_TOTAL);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(tc_points_vjp_n<D, DG_POINTS_OCC>, cudaFuncAttributeMaxDynamicSharedMemorySize, T::DG_TOTAL);
    if (e != cudaSuccess) return e;
    int dev = 0; cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
    attr = true;
  }
  const VjpWs w = vjp_layout<D>(a.N, occ);
  char* base = static_cast<char*>(a.workspace);
  SampleRec* recs = reinterpret_cast<SampleRec*>(base + w.rec);
  unsigned char* gates = reinterpret_cast<unsigned char*>(base + w.gates);
  unsigned char *img = reinterpret_cast<unsigned char*>(base + w.img), *img_t = reinterpret_cast<unsigned char*>(base + w.img_t);
  tc_prep_weights<D><<<occ ? T::N_STAGES_OCC : T::N_STAGES_PTS, 256, 0, st>>>(a.weights, img);
  tc_prep_weights_t_from<D><<<T::dg_tile_stages(occ), 256, 0, st>>>(a.weights, img_t, T::dg_first_stage(occ));
  const int n_tiles = (a.N + TILE - 1) / TILE;
  const int grid = n_tiles < n_sm ? n_tiles : n_sm;
  float4* out4 = reinterpret_cast<float4*>(out_rgba);
  if (count) tc_points_vjp_fwd_n<D><<<grid, N_THREADS, T::SM_TOTAL, st>>>(a, img, recs, out4, gates, count);
  else tc_points_vjp_fwd<D><<<grid, N_THREADS, T::SM_TOTAL, st>>>(a, img, recs, out4, gates, (size_t)a.N, n_tiles);
  DgPtrs P{};
  P.rec = recs; P.gates = gates;
  P.gs = reinterpret_cast<const float4*>(g_rgba); P.gp = reinterpret_cast<float4*>(g_pts); P.gv = reinterpret_cast<float4*>(g_dirs);
  if (count) tc_points_vjp_n<D, DG_POINTS_OCC><<<grid, N_THREADS, T::DG_TOTAL, st>>>(a, img_t, P, count);
  else if (occ) tc_points_vjp<D, DG_POINTS_OCC><<<grid, N_THREADS, T::DG_TOTAL, st>>>(a, img_t, P, (size_t)a.N, n_tiles);
  else tc_points_vjp<D, DG_POINTS><<<grid, N_THREADS, T::DG_TOTAL, st>>>(a, img_t, P, (size_t)a.N, n_tiles);
  return cudaGetLastError();
}

// Workspace of nnb_field_grad, every section 256-byte aligned: make_layout(N, 1, NNB_STASH, NNB_ENGINE_TC, D) (records, the fp32 stash
// and its dY half, the weight-gradient partials, the gate bits) | the forward weight image (the occupancy-only prefix when occ) | the
// transposed weight image (its trunk part when occ), as in vjp_layout
struct GradWs { WsLayout L; size_t img, img_t, total; };
template <int D> GradWs grad_layout(int N, bool occ) {
  using T = Tc<D>;
  GradWs w{};
  w.L = make_layout(N, 1, NNB_STASH, NNB_ENGINE_TC, D);
  size_t off = w.L.total;
  auto take = [&](size_t bytes) { const size_t o = off; off += align_up(bytes, 256); return o; };
  w.img = take(occ ? (size_t)T::N_STAGES_OCC * T::STAGE_BYTES : T::IMG_PTS_BYTES);
  w.img_t = take(occ ? T::IMG_T_BYTES - T::IMG_T_PREFIX_BYTES : T::IMG_T_BYTES);
  w.total = off;
  return w;
}

// nnb_field_grad: both weight images, the forward with the training stash, the chain with the dY stash, then (g_weights) the weight-
// gradient stage on Mpad rows; the rows past N have dY = 0, so they add exactly 0 to every dW / db
template <int D>
cudaError_t tc_field_grad_dim(const nnb_render_args& a, const float* g_rgba, float* out_rgba, float* g_pts, float* g_dirs, float* g_weights,
                              cudaStream_t st) {
  using T = Tc<D>;
  const bool occ = (a.flags & NNB_OCC_ONLY) != 0;
  cudaError_t e = upload_stage_table<D>();
  if (e == cudaSuccess) e = upload_stage_table_t<D>();
  if (e != cudaSuccess) return e;
  static bool attr = false;
  static int n_sm = 0;
  if (!attr) {
    e = cudaFuncSetAttribute(tc_points_grad_fwd<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, T::SM_TOTAL);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(tc_points_grad<D, DG_POINTS_GRAD>, cudaFuncAttributeMaxDynamicSharedMemorySize, T::DG_TOTAL);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(tc_points_grad<D, DG_POINTS_GRAD_OCC>, cudaFuncAttributeMaxDynamicSharedMemorySize, T::DG_TOTAL);
    if (e != cudaSuccess) return e;
    int dev = 0; cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
    attr = true;
  }
  const GradWs w = grad_layout<D>(a.N, occ);
  const WsLayout& L = w.L;
  char* base = static_cast<char*>(a.workspace);
  auto F = [&](size_t off) { return reinterpret_cast<float*>(base + off); };
  SampleRec* recs = reinterpret_cast<SampleRec*>(base + L.rec);
  unsigned char* gates = reinterpret_cast<unsigned char*>(base + L.gates);
  unsigned char *img = reinterpret_cast<unsigned char*>(base + w.img), *img_t = reinterpret_cast<unsigned char*>(base + w.img_t);
  TcStash ts{};
  for (int l = 0; l < 8; ++l) ts.h[l] = F(L.h[l]);
  ts.feat = F(L.feat); ts.hr = F(L.hr); ts.enc = F(L.enc); ts.denc = F(L.denc); ts.gates = gates;
  tc_prep_weights<D><<<occ ? T::N_STAGES_OCC : T::N_STAGES_PTS, 256, 0, st>>>(a.weights, img);
  tc_prep_weights_t_from<D><<<T::dg_tile_stages(occ), 256, 0, st>>>(a.weights, img_t, T::dg_first_stage(occ));
  const int n_tiles = (a.N + TILE - 1) / TILE;
  const int grid = n_tiles < n_sm ? n_tiles : n_sm;
  tc_points_grad_fwd<D><<<grid, N_THREADS, T::SM_TOTAL, st>>>(a, img, recs, reinterpret_cast<float4*>(out_rgba), ts, (size_t)a.N, n_tiles);
  DgPtrs P{};
  P.rec = recs; P.gates = gates;
  P.gs = reinterpret_cast<const float4*>(g_rgba); P.gp = reinterpret_cast<float4*>(g_pts); P.gv = reinterpret_cast<float4*>(g_dirs);
  P.dyc = reinterpret_cast<float4*>(base + L.dyc);
  for (int l = 0; l < 8; ++l) P.dy[l] = F(L.dy[l]);
  P.dfeat = F(L.dfeat); P.dyr = F(L.dyr);
  if (occ) tc_points_grad<D, DG_POINTS_GRAD_OCC><<<grid, N_THREADS, T::DG_TOTAL, st>>>(a, img_t, P, (size_t)a.N, n_tiles);
  else tc_points_grad<D, DG_POINTS_GRAD><<<grid, N_THREADS, T::DG_TOTAL, st>>>(a, img_t, P, (size_t)a.N, n_tiles);
  e = cudaGetLastError();
  if (e != cudaSuccess || !g_weights) return e;
  WsLayout Lw = L;
  Lw.M = L.Mpad;   // whole tiles: the stash rows past N are written, with zero dY
  return tc_wgrad_jobs(a, Lw, g_weights, occ, true, st);
}

// Workspace of nnb_field_hvp_tc, every section 256-byte aligned: grad_layout(N, occ = true) | the bf16 image of the occupancy-only
// forward stages.  The tangent stash (e', h'0..h'7, Npad rows) takes the place of the fp32 activation stash (enc, h0..h7), which this
// call does not write: the tangent chain gates with the forward's bits.
struct HvpWs { GradWs g; size_t img16, total; };
template <int D> HvpWs hvp_layout(int N) {
  HvpWs w{};
  w.g = grad_layout<D>(N, true);
  w.img16 = w.g.total;
  w.total = w.img16 + align_up((size_t)Tc<D>::N_STAGES_OCC * Tc<D>::STAGE_BYTES, 256);
  return w;
}

// nnb_field_hvp_tc: the three weight images, the occupancy-only forward with records and gate bits (tc_points_vjp_fwd), the chain for a
// cotangent 1 on the logit with the dY stash and the point term, then (g_weights) the tangent chain and the weight-gradient stage on
// (dY, tangent) without bias jobs, on Mpad rows: the rows past N have dY = 0 and u = 0, so they add exactly 0
template <int D>
cudaError_t tc_field_hvp_dim(const nnb_render_args& a, const float* u, float* g_pts, float* g_weights, cudaStream_t st) {
  using T = Tc<D>;
  cudaError_t e = upload_stage_table<D>();
  if (e == cudaSuccess) e = upload_stage_table_t<D>();
  if (e != cudaSuccess) return e;
  static bool attr = false;
  static int n_sm = 0;
  if (!attr) {
    e = cudaFuncSetAttribute(tc_points_vjp_fwd<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, T::SM_TOTAL);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(tc_points_hvp<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, T::DG_TOTAL);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(tc_points_tangent<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, T::SM_TOTAL);
    if (e != cudaSuccess) return e;
    int dev = 0; cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
    attr = true;
  }
  const HvpWs w = hvp_layout<D>(a.N);
  const WsLayout& L = w.g.L;
  char* base = static_cast<char*>(a.workspace);
  auto F = [&](size_t off) { return reinterpret_cast<float*>(base + off); };
  SampleRec* recs = reinterpret_cast<SampleRec*>(base + L.rec);
  unsigned char* gates = reinterpret_cast<unsigned char*>(base + L.gates);
  unsigned char *img = reinterpret_cast<unsigned char*>(base + w.g.img), *img_t = reinterpret_cast<unsigned char*>(base + w.g.img_t);
  unsigned char* img16 = reinterpret_cast<unsigned char*>(base + w.img16);
  tc_prep_weights<D><<<T::N_STAGES_OCC, 256, 0, st>>>(a.weights, img);
  tc_prep_weights_t_from<D><<<T::dg_tile_stages(true), 256, 0, st>>>(a.weights, img_t, T::dg_first_stage(true));
  const int n_tiles = (a.N + TILE - 1) / TILE;
  const int grid = n_tiles < n_sm ? n_tiles : n_sm;
  tc_points_vjp_fwd<D><<<grid, N_THREADS, T::SM_TOTAL, st>>>(a, img, recs, nullptr, gates, (size_t)a.N, n_tiles);
  DgPtrs P{};
  P.rec = recs; P.gates = gates;
  P.gs = reinterpret_cast<const float4*>(u); P.gp = reinterpret_cast<float4*>(g_pts);
  P.dyc = reinterpret_cast<float4*>(base + L.dyc);
  for (int l = 0; l < 8; ++l) P.dy[l] = F(L.dy[l]);
  tc_points_hvp<D><<<grid, N_THREADS, T::DG_TOTAL, st>>>(a, img_t, P, (size_t)a.N, n_tiles);
  e = cudaGetLastError();
  if (e != cudaSuccess || !g_weights) return e;
  TcStash ts{};
  for (int l = 0; l < 8; ++l) ts.h[l] = F(L.h[l]);
  ts.enc = F(L.enc); ts.gates = gates;
  tc_prep_weights_bf16<D><<<T::N_STAGES_OCC, 256, 0, st>>>(a.weights, img16);
  tc_points_tangent<D><<<grid, N_THREADS, T::SM_TOTAL, st>>>(a, img16, reinterpret_cast<const float4*>(u), ts, (size_t)a.N, n_tiles);
  e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  WsLayout Lw = L;
  Lw.M = L.Mpad;   // whole tiles: the stash rows past N are written, with zero dY and zero tangents
  return tc_wgrad_jobs(a, Lw, g_weights, true, false, st);
}

// Workspace of nnb_geometry_frame, every section 256-byte aligned: hit count | ray0, dir [N][3], far, depth [N] | compacted rows: surface
// points, view directions [N][3], pixel indices [N], normal cotangents, d logit / d p, colour query outputs [N] float4 | nnb_ray_march's
// workspace (N rays) | nnb_field_vjp's occupancy-only workspace (N points) | the points forward's weight image (the only part of
// nnb_field_fwd's tensor-core workspace that the points forward uses)
struct GeoWs { size_t count, ray0, dir, far, depth, pts, vdir, pix, gs, gp, rgba, march, vjp, img, total; };
template <int D> GeoWs geo_layout(int N, int n_steps) {
  GeoWs w{};
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t o = off; off += align_up(bytes, 256); return o; };
  const size_t n = (size_t)N;
  w.count = take(4);
  w.ray0 = take(n * 12); w.dir = take(n * 12); w.far = take(n * 4); w.depth = take(n * 4);
  w.pts = take(n * 12); w.vdir = take(n * 12); w.pix = take(n * 4); w.gs = take(n * 16); w.gp = take(n * 16); w.rgba = take(n * 16);
  w.march = take(march_layout<D>(N, n_steps).total);
  w.vjp = take(vjp_layout<D>(N, true).total);
  w.img = take(Tc<D>::IMG_PTS_BYTES);
  w.total = off;
  return w;
}

// nnb_geometry_frame: rays, the fused march (tc_ray_march_dim), compaction, normals (tc_field_vjp_dim) and colour (tc_points_fwd_launch)
// of the compacted rows with their device count, shading.  Nothing is read back.
template <int D>
cudaError_t tc_geometry_frame_dim(const nnb_geometry_args& g, cudaStream_t st) {
  const GeoWs w = geo_layout<D>(g.N, g.n_steps);
  char* base = static_cast<char*>(g.workspace);
  auto F = [&](size_t off) { return reinterpret_cast<float*>(base + off); };
  auto F4 = [&](size_t off) { return reinterpret_cast<float4*>(base + off); };
  int* count = reinterpret_cast<int*>(base + w.count);
  cudaError_t e = cudaMemsetAsync(count, 0, 4, st);
  if (e != cudaSuccess) return e;
  const int blocks = (g.N + 255) / 256;
  geo_rays<<<blocks, 256, 0, st>>>(g.T, g.pixels, g.N, g.radius, F(w.ray0), F(w.dir), F(w.far), g.ray0, g.ray_dir, g.far_);
  nnb_ray_march_args r{};
  r.weights = g.weights; r.ray0 = F(w.ray0); r.ray_dir = F(w.dir); r.far_ = F(w.far); r.frac = g.frac;
  r.N = g.N; r.n_steps = g.n_steps; r.n_secant = g.n_secant; r.hidden_dim = D; r.near_ = g.near_; r.tau = g.tau;
  r.flags = g.flags; r.engine = NNB_ENGINE_TC; r.depth = F(w.depth);
  r.workspace = base + w.march; r.workspace_bytes = w.vjp - w.march;
  e = tc_ray_march_dim<D>(r, st);
  if (e != cudaSuccess) return e;
  int* pix = reinterpret_cast<int*>(base + w.pix);
  geo_compact<<<blocks, 256, 0, st>>>(g.N, F(w.ray0), F(w.dir), F(w.depth), count, F(w.pts), F(w.vdir), pix, F4(w.gs), g.rgb, g.rgb_surf,
                                      g.depth, reinterpret_cast<float4*>(g.grad));
  nnb_render_args a{};
  a.weights = g.weights; a.pts = F(w.pts); a.dirs = nullptr; a.N = g.N; a.S = 1; a.hidden_dim = D; a.engine = NNB_ENGINE_TC;
  a.flags = NNB_RAW_DENSITY | NNB_OCC_ONLY; a.workspace = base + w.vjp; a.workspace_bytes = w.img - w.vjp;
  e = tc_field_vjp_dim<D>(a, F(w.gs), nullptr, F(w.gp), nullptr, st, count);   // d logit / d p
  if (e != cudaSuccess) return e;
  a.dirs = F(w.vdir); a.flags = g.flags & (NNB_DIST_ALPHA | NNB_SOFTPLUS); a.workspace = base + w.img; a.workspace_bytes = w.total - w.img;
  e = tc_points_fwd_launch<D>(a, reinterpret_cast<unsigned char*>(base + w.img), F(w.rgba), (size_t)g.N, count, st);   // surface colour
  if (e != cudaSuccess) return e;
  geo_shade<<<blocks, 256, 0, st>>>(g.T, count, pix, F4(w.gp), F4(w.rgba), g.rgb, g.rgb_surf, reinterpret_cast<float4*>(g.grad));
  return cudaGetLastError();
}

// nnb_render_frame: weight image once, then run_render_frame (nnb_frame.cuh) with one tc_frame launch per 32-sample chunk
template <int D>
cudaError_t tc_render_frame_dim(const nnb_render_args& a, float t_min, int* n_eval, float* t_final, cudaStream_t st) {
  using T = Tc<D>;
  cudaError_t e = upload_stage_table<D>();
  if (e != cudaSuccess) return e;
  static bool attr = false;
  static int n_sm = 0;
  if (!attr) {
    e = cudaFuncSetAttribute(tc_frame<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, T::SM_TOTAL);
    if (e != cudaSuccess) return e;
    int dev = 0; cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
    attr = true;
  }
  const FrameWs w = frame_layout_bytes(a.N, T::IMG_BYTES);
  unsigned char* img = static_cast<unsigned char*>(a.workspace) + w.img;
  tc_prep_weights<D><<<T::N_STAGES, 256, 0, st>>>(a.weights, img);
  const int tiles = (a.N + 3) / 4, grid = tiles < n_sm ? tiles : n_sm;
  return run_render_frame(a, w, t_min, n_eval, t_final, st,
                          [&](const FramePtrs& f) { tc_frame<D><<<grid, N_THREADS, T::SM_TOTAL, st>>>(a, img, f); });
}

// Workspace of nnb_render_frame_bwd: frame_bwd_layout_bytes (nnb_frame.cuh) with this engine's forward weight image, the chunk stash
// make_layout(N, 32, NNB_STASH, NNB_ENGINE_TC, D) (32 N rows) and the transposed weight image
template <int D> FrameBwdWs frame_bwd_layout(int N, int S) {
  return frame_bwd_layout_bytes(N, S, Tc<D>::IMG_BYTES, make_layout(N, 32, NNB_STASH, NNB_ENGINE_TC, D).total, Tc<D>::IMG_T_BYTES);
}

// the lazy set-up of nnb_render_frame_bwd and of its two halves (both stage tables, the kernels' shared-memory limits); returns the
// SM count, 0 on an error (in *e)
template <int D>
int frame_bwd_setup(cudaError_t* e) {
  using T = Tc<D>;
  *e = upload_stage_table<D>();
  if (*e == cudaSuccess) *e = upload_stage_table_t<D>();
  if (*e != cudaSuccess) return 0;
  static bool attr = false;
  static int n_sm = 0;
  if (!attr) {
    *e = cudaFuncSetAttribute(tc_frame<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, T::SM_TOTAL);
    if (*e == cudaSuccess) *e = cudaFuncSetAttribute(tc_frame_stash<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, T::SM_TOTAL);
    if (*e == cudaSuccess) *e = cudaFuncSetAttribute(tc_dgrad_frame<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, T::DG_TOTAL);
    if (*e == cudaSuccess) *e = cudaFuncSetAttribute(tc_frame_stash_live<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, T::SM_TOTAL);
    if (*e == cudaSuccess) *e = cudaFuncSetAttribute(tc_dgrad_frame_live<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, T::DG_TOTAL);
    if (*e != cudaSuccess) return 0;
    int dev = 0; cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
    attr = true;
  }
  return n_sm;
}

// The forward half of nnb_render_frame_bwd (nnb_render_frame_train_fwd): the forward weight image, then the forward (run_render_frame at
// t_min = 0, so every ray runs every round) with the carry after each chunk copied to the checkpoints.  It leaves the weight image and
// the checkpoints in the workspace for the reverse half.  nnb_render_frame_train_fwd_tmin: the same at t_min, which also leaves the
// per-ray chunk counts (FramePtrs::chunks) for the reverse rounds; a ray that stopped keeps its carry, so every checkpoint from its last
// chunk on holds its final transmittance.
template <int D>
cudaError_t tc_frame_train_fwd_dim(const nnb_render_args& a, cudaStream_t st, float t_min = 0.f, int* n_eval = nullptr,
                                   float* t_final = nullptr) {
  using T = Tc<D>;
  cudaError_t e;
  const int n_sm = frame_bwd_setup<D>(&e);
  if (e != cudaSuccess) return e;
  const int N = a.N, C = (a.S + 31) / 32;
  const FrameBwdWs w = frame_bwd_layout<D>(N, a.S);
  char* base = static_cast<char*>(a.workspace);
  unsigned char* img = reinterpret_cast<unsigned char*>(base + w.f.img);
  tc_prep_weights<D><<<T::N_STAGES, 256, 0, st>>>(a.weights, img);
  const int tiles = (N + 3) / 4, grid = tiles < n_sm ? tiles : n_sm;   // 4 ray-chunks of 32 rows per tile
  float* ckpt = reinterpret_cast<float*>(base + w.ckpt);
  cudaError_t ec = cudaSuccess;
  e = run_render_frame(a, w.f, t_min, n_eval, t_final, st, [&](const FramePtrs& f) {
    tc_frame<D><<<grid, N_THREADS, T::SM_TOTAL, st>>>(a, img, f);
    if (f.k + 1 < C && ec == cudaSuccess) ec = cudaMemcpyAsync(ckpt + (size_t)f.k * N, f.carry, (size_t)N * 4, cudaMemcpyDeviceToDevice, st);
  });
  return e == cudaSuccess ? ec : e;
}

// The reverse half of nnb_render_frame_bwd (nnb_render_frame_train_bwd): the transposed weight image, then the reverse rounds
// k = C - 1 .. 0, each on the chunk stash: tc_frame_stash, frame_chunk_adjoint, tc_dgrad_frame, (g_weights) the weight-gradient stage,
// whose reduce adds the round's dW into g_weights, and frame_ray_acc; then frame_ray_finish and ray_reduce.  The rounds run one after
// another on the stream.  Of what the forward half wrote it reads the forward weight image and the checkpoints only (data, no index or
// counter), so a workspace the forward half did not fill gives wrong numbers, never an access outside the workspace.
// live (nnb_render_frame_train_bwd_tmin): round k runs on the rays that evaluated chunk k (frame_live_list from the forward's chunk counts,
// into the forward's first ray list and round counter, which are free once the forward has ended): the _live kernels, and the
// weight-gradient stage on the list's rows.  Every count and counter read is clamped (1..C, 0..N), so a backward without its forward still
// stays inside the workspace.
template <int D>
cudaError_t tc_frame_train_bwd_dim(const nnb_render_bwd_args& b, cudaStream_t st, bool live = false) {
  using T = Tc<D>;
  const nnb_render_args& a = b.fwd;
  cudaError_t e;
  const int n_sm = frame_bwd_setup<D>(&e);
  if (e != cudaSuccess) return e;
  const int N = a.N, C = (a.S + 31) / 32;
  const FrameBwdWs w = frame_bwd_layout<D>(N, a.S);
  char* base = static_cast<char*>(a.workspace);
  auto F = [&](size_t off) { return reinterpret_cast<float*>(base + off); };
  unsigned char *img = reinterpret_cast<unsigned char*>(base + w.f.img), *img_t = reinterpret_cast<unsigned char*>(base + w.img_t);
  tc_prep_weights_t<D><<<T::N_STAGES_T, 256, 0, st>>>(a.weights, img_t);
  const int tiles = (N + 3) / 4, grid = tiles < n_sm ? tiles : n_sm;   // 4 ray-chunks of 32 rows per tile
  // the chunk stash: make_layout's offsets from its own base
  nnb_render_args ac = a;
  ac.workspace = base + w.chunk; ac.workspace_bytes = w.img_t - w.chunk;
  const WsLayout L = make_layout(N, 32, NNB_STASH, NNB_ENGINE_TC, D);
  char* cb = base + w.chunk;
  auto CF = [&](size_t off) { return reinterpret_cast<float*>(cb + off); };
  SampleRec* recs = reinterpret_cast<SampleRec*>(cb + L.rec);
  TcStash ts{};
  for (int l = 0; l < 8; ++l) ts.h[l] = CF(L.h[l]);
  ts.feat = CF(L.feat); ts.hr = CF(L.hr); ts.enc = CF(L.enc); ts.denc = CF(L.denc); ts.gates = reinterpret_cast<unsigned char*>(cb + L.gates);
  DgPtrs P{};
  P.rec = recs; P.gates = ts.gates;
  P.gs = reinterpret_cast<const float4*>(cb + L.gs); P.gp = reinterpret_cast<float4*>(cb + L.gp); P.gv = reinterpret_cast<float4*>(cb + L.gv);
  P.dyc = reinterpret_cast<float4*>(cb + L.dyc);
  for (int l = 0; l < 8; ++l) P.dy[l] = CF(L.dy[l]);
  P.dfeat = CF(L.dfeat); P.dyr = CF(L.dyr);
  FrameBwdPtrs fb{};
  fb.rounds = C; fb.ckpt = F(w.ckpt); fb.suffix = F(w.suffix); fb.rec = recs;
  fb.gs = reinterpret_cast<float4*>(cb + L.gs); fb.gp = P.gp; fb.gv = P.gv; fb.raypart = F(w.raypart);
  const int write_dy = b.g_weights ? 1 : 0, warps = (N + 7) / 8;
  int* list = reinterpret_cast<int*>(base + w.f.list[0]);
  int* count = reinterpret_cast<int*>(base);   // round counter 0 of the forward
  const FrameLive fl{reinterpret_cast<const int*>(base + w.f.chunks), list, count};
  for (int k = C - 1; k >= 0; --k) {
    FramePtrs f{};
    f.k = k;
    fb.k = k;
    if (live) {
      f.list = list; f.count = count;
      frame_live_list<<<1, 1024, 0, st>>>(fl.chunks, N, k, C, list, count);
      tc_frame_stash_live<D><<<grid, N_THREADS, T::SM_TOTAL, st>>>(a, img, recs, ts, f);
      frame_chunk_adjoint_live<<<warps, 256, 0, st>>>(b, fb, fl);
      tc_dgrad_frame_live<D><<<grid, N_THREADS, T::DG_TOTAL, st>>>(a, img_t, P, write_dy, k, count, list);
    } else {
      tc_frame_stash<D><<<grid, N_THREADS, T::SM_TOTAL, st>>>(a, img, recs, ts, f, tiles);
      frame_chunk_adjoint<false><<<warps, 256, 0, st>>>(b, fb);
      tc_dgrad_frame<D><<<grid, N_THREADS, T::DG_TOTAL, st>>>(a, img_t, P, (size_t)N * 32, tiles, write_dy, k);
    }
    e = cudaGetLastError();
    if (e == cudaSuccess && b.g_weights) e = tc_wgrad_jobs(ac, L, b.g_weights, false, true, st, live ? count : nullptr);
    if (e != cudaSuccess) return e;
    if (live) frame_ray_acc_live<<<warps, 256, 0, st>>>(a, fb, fl);
    else frame_ray_acc<false><<<warps, 256, 0, st>>>(a, fb);
  }
  float* rayred = CF(L.rayred);
  frame_ray_finish<<<warps, 256, 0, st>>>(b, F(w.raypart), rayred);
  e = cudaGetLastError();
  return e != cudaSuccess ? e : launch_ray_reduce(b, rayred, st);
}

// Workspace of nnb_render_fwd_tmin / nnb_render_bwd_tmin, every section 256-byte aligned: the packed stash make_layout(4 ceil(N / 4), 32 C,
// NNB_STASH, NNB_ENGINE_TC, D) at offset 0 (C 128 ceil(N / 4) rows: every ray in every round, each round padded to the tile) | carry,
// chunk counts [N] | lane partials [N][5][32] | checkpoints [C - 1][N] | lists [C][N] | counts [C + 1] | ray lane partials [N][9][32] |
// the forward and the transposed weight images.
struct StashTminWs { WsLayout L; size_t carry, chunks, part, ckpt, lists, counts, raypart, img, img_t, total; };
template <int D> StashTminWs stash_tmin_layout(int N, int S) {
  StashTminWs w{};
  const int C = (S + 31) / 32;
  const size_t n = (size_t)N;
  w.L = make_layout((N + 3) / 4 * 4, 32 * C, NNB_STASH, NNB_ENGINE_TC, D);
  size_t off = w.L.total;
  auto take = [&](size_t bytes) { const size_t o = off; off += align_up(bytes, 256); return o; };
  w.carry = take(n * 4); w.chunks = take(n * 4); w.part = take(n * 640); w.ckpt = take((size_t)(C - 1) * n * 4);
  w.lists = take((size_t)C * n * 4); w.counts = take((size_t)(C + 1) * 4); w.raypart = take(n * 288 * 4);
  w.img = take(Tc<D>::IMG_BYTES); w.img_t = take(Tc<D>::IMG_T_BYTES);
  w.total = off;
  return w;
}
template <int D>
int stash_tmin_setup(cudaError_t* e) {
  using T = Tc<D>;
  *e = upload_stage_table<D>();
  if (*e == cudaSuccess) *e = upload_stage_table_t<D>();
  if (*e != cudaSuccess) return 0;
  static bool attr = false;
  static int n_sm = 0;
  if (!attr) {
    *e = cudaFuncSetAttribute(tc_stash_pack<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, T::SM_TOTAL);
    if (*e == cudaSuccess) *e = cudaFuncSetAttribute(tc_dgrad_pack<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, T::DG_TOTAL);
    if (*e != cudaSuccess) return 0;
    int dev = 0; cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
    attr = true;
  }
  return n_sm;
}
// the training stash pointers of a layout at `base`
inline TcStash stash_ptrs(char* base, const WsLayout& L) {
  TcStash ts{};
  for (int l = 0; l < 8; ++l) ts.h[l] = reinterpret_cast<float*>(base + L.h[l]);
  ts.feat = reinterpret_cast<float*>(base + L.feat); ts.hr = reinterpret_cast<float*>(base + L.hr);
  ts.enc = reinterpret_cast<float*>(base + L.enc); ts.denc = reinterpret_cast<float*>(base + L.denc);
  ts.gates = reinterpret_cast<unsigned char*>(base + L.gates);
  return ts;
}

// nnb_render_fwd_tmin: the forward weight image, then rounds k = 0 .. C - 1: frame_live_list (round k's list from the chunk counts),
// tc_stash_pack (chunk k of the listed rays with the training stash, into the packed stash) and stash_frame_step (frame_step's compositing
// and stop rule on the round's records); then frame_finish.  Every launch sizes itself from device counts; nothing is read back.
template <int D>
cudaError_t tc_render_tmin_fwd_dim(const nnb_frame_args& fa, cudaStream_t st) {
  using T = Tc<D>;
  const nnb_render_args& a = fa.fwd;
  cudaError_t e;
  const int n_sm = stash_tmin_setup<D>(&e);
  if (e != cudaSuccess) return e;
  const int N = a.N, C = (a.S + 31) / 32;
  const StashTminWs w = stash_tmin_layout<D>(N, a.S);
  char* base = static_cast<char*>(a.workspace);
  auto I = [&](size_t off) { return reinterpret_cast<int*>(base + off); };
  unsigned char* img = reinterpret_cast<unsigned char*>(base + w.img);
  tc_prep_weights<D><<<T::N_STAGES, 256, 0, st>>>(a.weights, img);
  SampleRec* recs = reinterpret_cast<SampleRec*>(base + w.L.rec);
  const TcStash ts = stash_ptrs(base, w.L);
  const int tiles = (N + 3) / 4, grid = tiles < n_sm ? tiles : n_sm, warps = (N + 7) / 8;
  int *lists = I(w.lists), *counts = I(w.counts);
  FramePtrs f{};
  f.t_min = fa.t_min;
  f.carry = reinterpret_cast<float*>(base + w.carry); f.chunks = I(w.chunks); f.part = reinterpret_cast<float*>(base + w.part);
  float* ckpt = reinterpret_cast<float*>(base + w.ckpt);
  for (int k = 0; k < C; ++k) {
    f.k = k; f.list = lists + (size_t)k * N; f.count = counts + k;
    frame_live_list<<<1, 1024, 0, st>>>(f.chunks, N, k, C, lists + (size_t)k * N, counts + k);
    tc_stash_pack<D><<<grid, N_THREADS, T::SM_TOTAL, st>>>(a, img, recs, ts, f, w.L.M);
    stash_frame_step<<<warps, 256, 0, st>>>(a, f, recs, ckpt, C);
  }
  frame_finish<<<warps, 256, 0, st>>>(a, f, fa.n_eval, fa.t_final);
  return cudaGetLastError();
}

// nnb_render_bwd_tmin: the transposed weight image; the C lists again from the chunk counts (frame_live_list); stash_chunk_adjoint (every
// ray's compositing adjoint, padding cotangents, the row count); the data-gradient chain on the packed rows (tc_dgrad_pack); with
// g_weights, one weight-gradient stage on those rows; stash_ray_acc, frame_ray_finish and ray_reduce.  Of what the forward wrote it reads
// the chunk counts (clamped to 1..C), the checkpoints and the stash, so a backward without its forward gives wrong numbers, never an
// access outside the workspace.
template <int D>
cudaError_t tc_render_tmin_bwd_dim(const nnb_render_bwd_args& b, cudaStream_t st) {
  using T = Tc<D>;
  const nnb_render_args& a = b.fwd;
  cudaError_t e;
  const int n_sm = stash_tmin_setup<D>(&e);
  if (e != cudaSuccess) return e;
  const int N = a.N, C = (a.S + 31) / 32;
  const StashTminWs w = stash_tmin_layout<D>(N, a.S);
  const WsLayout& L = w.L;
  char* base = static_cast<char*>(a.workspace);
  auto F = [&](size_t off) { return reinterpret_cast<float*>(base + off); };
  auto I = [&](size_t off) { return reinterpret_cast<int*>(base + off); };
  unsigned char* img_t = reinterpret_cast<unsigned char*>(base + w.img_t);
  tc_prep_weights_t<D><<<T::N_STAGES_T, 256, 0, st>>>(a.weights, img_t);
  const int *chunks = I(w.chunks);
  int *lists = I(w.lists), *counts = I(w.counts);
  for (int k = 0; k < C; ++k) frame_live_list<<<1, 1024, 0, st>>>(chunks, N, k, C, lists + (size_t)k * N, counts + k);
  DgPtrs P{};
  P.rec = reinterpret_cast<const SampleRec*>(base + L.rec); P.gates = reinterpret_cast<const unsigned char*>(base + L.gates);
  P.gs = reinterpret_cast<const float4*>(base + L.gs); P.gp = reinterpret_cast<float4*>(base + L.gp); P.gv = reinterpret_cast<float4*>(base + L.gv);
  P.dyc = reinterpret_cast<float4*>(base + L.dyc);
  for (int l = 0; l < 8; ++l) P.dy[l] = F(L.dy[l]);
  P.dfeat = F(L.dfeat); P.dyr = F(L.dyr);
  FrameBwdPtrs fb{};
  fb.rounds = C; fb.ckpt = F(w.ckpt); fb.rec = P.rec;
  fb.gs = reinterpret_cast<float4*>(base + L.gs); fb.gp = P.gp; fb.gv = P.gv; fb.raypart = F(w.raypart);
  const int warps = (N + 7) / 8, tiles = (int)(L.M / TILE), grid = tiles < n_sm ? tiles : n_sm;
  stash_chunk_adjoint<<<(N + 3 * C + 7) / 8, 256, 0, st>>>(b, fb, chunks, lists, counts);
  tc_dgrad_pack<D><<<grid, N_THREADS, T::DG_TOTAL, st>>>(a, img_t, P, L.M, b.g_weights ? 1 : 0, C, counts, lists);
  e = cudaGetLastError();
  if (e == cudaSuccess && b.g_weights) e = tc_wgrad_jobs(a, L, b.g_weights, false, true, st, counts + C);
  if (e != cudaSuccess) return e;
  stash_ray_acc<<<warps, 256, 0, st>>>(a, fb, chunks, lists, counts);
  float* rayred = F(L.rayred);
  frame_ray_finish<<<warps, 256, 0, st>>>(b, F(w.raypart), rayred);
  e = cudaGetLastError();
  return e != cudaSuccess ? e : launch_ray_reduce(b, rayred, st);
}

template <int D> size_t tc_extra_dim() { return align_up(Tc<D>::IMG_BYTES, 256) + align_up(Tc<D>::IMG_T_BYTES, 256); }

}  // namespace

size_t tc_workspace_extra(int N, int S, uint32_t flags, int D) {
  return D == 128 ? tc_extra_dim<128>() : (D == 64 ? tc_extra_dim<64>() : tc_extra_dim<256>());
}

// S >= 16 bounds the rays one 64-row block overlaps (Tc<D>::RAYB_RAYS); S <= 1024 is the compositing adjoint's limit
bool tc_supports(int S) { return S >= 16 && S <= 1024; }

cudaError_t tc_render_fwd(const nnb_render_args& a, const WsLayout& L, cudaStream_t st) {
  if (!tc_supports(a.S)) return cudaErrorNotSupported;
  return L.D == 128 ? tc_render_fwd_dim<128>(a, L, st) : (L.D == 64 ? tc_render_fwd_dim<64>(a, L, st) : tc_render_fwd_dim<256>(a, L, st));
}

size_t tc_ray_march_workspace(int N, int n_steps, int D) {
  return D == 128 ? march_layout<128>(N, n_steps).total : (D == 64 ? march_layout<64>(N, n_steps).total : march_layout<256>(N, n_steps).total);
}
cudaError_t tc_ray_march(const nnb_ray_march_args& r, int D, cudaStream_t st) {
  return D == 128 ? tc_ray_march_dim<128>(r, st) : (D == 64 ? tc_ray_march_dim<64>(r, st) : tc_ray_march_dim<256>(r, st));
}

cudaError_t tc_field_fwd_points(const nnb_render_args& a, const WsLayout& L, float* out_rgba, cudaStream_t st) {
  return L.D == 128 ? tc_points_fwd_dim<128>(a, L, out_rgba, st)
       : L.D == 64  ? tc_points_fwd_dim<64>(a, L, out_rgba, st) : tc_points_fwd_dim<256>(a, L, out_rgba, st);
}

size_t tc_field_vjp_workspace(int N, uint32_t flags, int D) {
  const bool occ = (flags & NNB_OCC_ONLY) != 0;
  return D == 128 ? vjp_layout<128>(N, occ).total : (D == 64 ? vjp_layout<64>(N, occ).total : vjp_layout<256>(N, occ).total);
}
cudaError_t tc_field_vjp(const nnb_render_args& a, const float* g_rgba, float* out_rgba, float* g_pts, float* g_dirs, int D, cudaStream_t st) {
  return D == 128 ? tc_field_vjp_dim<128>(a, g_rgba, out_rgba, g_pts, g_dirs, st)
       : D == 64  ? tc_field_vjp_dim<64>(a, g_rgba, out_rgba, g_pts, g_dirs, st) : tc_field_vjp_dim<256>(a, g_rgba, out_rgba, g_pts, g_dirs, st);
}

size_t tc_field_grad_workspace(int N, uint32_t flags, int D) {
  const bool occ = (flags & NNB_OCC_ONLY) != 0;
  return D == 128 ? grad_layout<128>(N, occ).total : (D == 64 ? grad_layout<64>(N, occ).total : grad_layout<256>(N, occ).total);
}
cudaError_t tc_field_grad(const nnb_render_args& a, const float* g_rgba, float* out_rgba, float* g_pts, float* g_dirs, float* g_weights, int D,
                          cudaStream_t st) {
  return D == 128 ? tc_field_grad_dim<128>(a, g_rgba, out_rgba, g_pts, g_dirs, g_weights, st)
       : D == 64  ? tc_field_grad_dim<64>(a, g_rgba, out_rgba, g_pts, g_dirs, g_weights, st)
                  : tc_field_grad_dim<256>(a, g_rgba, out_rgba, g_pts, g_dirs, g_weights, st);
}

size_t tc_field_hvp_workspace(int N, int D) {
  return D == 128 ? hvp_layout<128>(N).total : (D == 64 ? hvp_layout<64>(N).total : hvp_layout<256>(N).total);
}
cudaError_t tc_field_hvp(const nnb_render_args& a, const float* u, float* g_pts, float* g_weights, int D, cudaStream_t st) {
  return D == 128 ? tc_field_hvp_dim<128>(a, u, g_pts, g_weights, st)
       : D == 64  ? tc_field_hvp_dim<64>(a, u, g_pts, g_weights, st) : tc_field_hvp_dim<256>(a, u, g_pts, g_weights, st);
}

size_t tc_render_frame_workspace(int N, int D) {
  return frame_layout_bytes(N, D == 128 ? Tc<128>::IMG_BYTES : (D == 64 ? Tc<64>::IMG_BYTES : Tc<256>::IMG_BYTES)).total;
}
cudaError_t tc_render_frame(const nnb_render_args& a, float t_min, int* n_eval, float* t_final, int D, cudaStream_t st) {
  return D == 128 ? tc_render_frame_dim<128>(a, t_min, n_eval, t_final, st)
       : D == 64  ? tc_render_frame_dim<64>(a, t_min, n_eval, t_final, st) : tc_render_frame_dim<256>(a, t_min, n_eval, t_final, st);
}

size_t tc_render_frame_bwd_workspace(int N, int S, int D) {
  return D == 128 ? frame_bwd_layout<128>(N, S).total : (D == 64 ? frame_bwd_layout<64>(N, S).total : frame_bwd_layout<256>(N, S).total);
}
cudaError_t tc_render_frame_train_fwd(const nnb_render_args& a, int D, cudaStream_t st) {
  return D == 128 ? tc_frame_train_fwd_dim<128>(a, st) : (D == 64 ? tc_frame_train_fwd_dim<64>(a, st) : tc_frame_train_fwd_dim<256>(a, st));
}
cudaError_t tc_render_frame_train_bwd(const nnb_render_bwd_args& b, int D, cudaStream_t st) {
  return D == 128 ? tc_frame_train_bwd_dim<128>(b, st) : (D == 64 ? tc_frame_train_bwd_dim<64>(b, st) : tc_frame_train_bwd_dim<256>(b, st));
}
cudaError_t tc_render_frame_train_fwd_tmin(const nnb_frame_args& f, int D, cudaStream_t st) {
  const nnb_render_args& a = f.fwd;
  return D == 128 ? tc_frame_train_fwd_dim<128>(a, st, f.t_min, f.n_eval, f.t_final)
       : D == 64  ? tc_frame_train_fwd_dim<64>(a, st, f.t_min, f.n_eval, f.t_final)
                  : tc_frame_train_fwd_dim<256>(a, st, f.t_min, f.n_eval, f.t_final);
}
cudaError_t tc_render_frame_train_bwd_tmin(const nnb_render_bwd_args& b, int D, cudaStream_t st) {
  return D == 128 ? tc_frame_train_bwd_dim<128>(b, st, true)
       : (D == 64 ? tc_frame_train_bwd_dim<64>(b, st, true) : tc_frame_train_bwd_dim<256>(b, st, true));
}
size_t tc_render_tmin_workspace(int N, int S, int D) {
  return D == 128 ? stash_tmin_layout<128>(N, S).total : (D == 64 ? stash_tmin_layout<64>(N, S).total : stash_tmin_layout<256>(N, S).total);
}
cudaError_t tc_render_fwd_tmin(const nnb_frame_args& f, int D, cudaStream_t st) {
  return D == 128 ? tc_render_tmin_fwd_dim<128>(f, st) : (D == 64 ? tc_render_tmin_fwd_dim<64>(f, st) : tc_render_tmin_fwd_dim<256>(f, st));
}
cudaError_t tc_render_bwd_tmin(const nnb_render_bwd_args& b, int D, cudaStream_t st) {
  return D == 128 ? tc_render_tmin_bwd_dim<128>(b, st) : (D == 64 ? tc_render_tmin_bwd_dim<64>(b, st) : tc_render_tmin_bwd_dim<256>(b, st));
}
// nnb_render_frame_bwd: the two halves in sequence
cudaError_t tc_render_frame_bwd(const nnb_render_bwd_args& b, int D, cudaStream_t st) {
  const cudaError_t e = tc_render_frame_train_fwd(b.fwd, D, st);
  return e != cudaSuccess ? e : tc_render_frame_train_bwd(b, D, st);
}

size_t tc_geometry_frame_workspace(int N, int n_steps, int D) {
  return D == 128 ? geo_layout<128>(N, n_steps).total : (D == 64 ? geo_layout<64>(N, n_steps).total : geo_layout<256>(N, n_steps).total);
}
cudaError_t tc_geometry_frame(const nnb_geometry_args& g, int D, cudaStream_t st) {
  return D == 128 ? tc_geometry_frame_dim<128>(g, st) : (D == 64 ? tc_geometry_frame_dim<64>(g, st) : tc_geometry_frame_dim<256>(g, st));
}

// Backward of the TC engine: compositing / ray adjoints of nnb_simt.cu around tc_dgrad and tc_wgrad, which read and write the SIMT
// engine's fp32 stash layout.
cudaError_t tc_render_bwd(const nnb_render_bwd_args& b, const WsLayout& L, cudaStream_t st) {
  return simt_render_bwd_with(b, L, st, tc_dgrad_launch, tc_wgrad_all);
}

// the weight-gradient stage of tc_render_bwd alone, on whatever the stash holds (nnb_debug_wgrad)
cudaError_t tc_wgrad_stage(const nnb_render_args& a, const WsLayout& L, float* gw, cudaStream_t st) { return tc_wgrad_all(a, L, gw, st); }
