// nnb_render_frame (the volumetric view of a frame with compositing fused into the field's forward), the parts both engines share: the
// per-ray state of the rounds (FramePtrs), the back end of a ray-chunk (frame_step), the end of the call (frame_finish), the workspace
// layout without the engine's own part (frame_layout_bytes) and the rounds themselves (run_render_frame).  nnb_tc.cu (tc_frame) and
// nnb_simt.cu (simt_frame) supply the field evaluations.
//
// Round k evaluates samples 32 k .. 32 k + 31 of every ray still live and composites them into per-ray lane partials in the workspace; a
// ray whose transmittance fell below t_min, or that has no chunk left, leaves; frame_finish writes the outputs.
#pragma once
#include "nnb_workspace.cuh"

namespace {

struct FramePtrs {
  int k;               // this round evaluates samples 32 k .. 32 k + 31 of its rays
  float t_min;
  const int* list;     // the rays of this round (NULL in round 0: every ray, ray-chunk = ray)
  const int* count;    // device count of `list` (NULL: a.N)
  int *next_list, *next_count;   // rays still live after this round
  float* carry;        // [N] transmittance after the ray's last evaluated chunk
  int* chunks;         // [N] chunks the ray evaluated (written when it leaves)
  float* part;         // [N][5][32] lane partials C0, C1, C2, Dist, acc of composite_chunk
};
constexpr int FRAME_MAX_ROUNDS = 32;   // S <= 1024

// Back end of a frame tile, one warp per ray-chunk: composite_fwd's chunk step on the chunk's (r, g, b, a) rows (s_rows, one float4 per
// row; lane i reads row i, lanes past the ray's last sample are invalid), continued from the ray's carry and lane partials of the rounds
// before.  The ray leaves when its carry is below t_min or it has no chunk left; otherwise it is appended to the next round's list.
__device__ __forceinline__ void frame_step(const nnb_render_args& a, const FramePtrs& f, int slot, int n_live, const unsigned char* s_rows,
                                           int lane) {
  if (slot >= n_live) return;
  const int n = f.list ? f.list[slot] : slot;
  const int i = 32 * f.k + lane;
  const bool valid = i < a.S;
  float4 me = make_float4(0.f, 0.f, 0.f, 0.f);
  float z = 0.f, alpha = 0.f;
  if (valid) {
    me = *reinterpret_cast<const float4*>(s_rows + lane * 16);
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
    if (carry < f.t_min || 32 * (f.k + 1) >= a.S) f.chunks[n] = f.k + 1;
    else f.next_list[atomicAdd(f.next_count, 1)] = n;
  }
}

// one warp per ray after the last round: composite_fwd's tail on the ray's lane partials, n_eval and t_final
__global__ void frame_finish(nnb_render_args a, const __grid_constant__ FramePtrs f, int* __restrict__ n_eval, float* __restrict__ t_final) {
  const int lane = threadIdx.x & 31, n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (n >= a.N) return;
  Ray ray; setup_ray(a, n, ray);
  const float* part = f.part + (size_t)n * 160 + lane;
  composite_tail(a, n, ray, part[0], part[32], part[64], part[96], part[128], lane);
  if (lane == 0) {
    if (n_eval) n_eval[n] = min(32 * f.chunks[n], a.S);
    if (t_final) t_final[n] = f.carry[n];
  }
}

// Workspace of nnb_render_frame, every section 256-byte aligned: counters [FRAME_MAX_ROUNDS + 1] (k >= 1: rays of round k) | carry,
// chunks [N] | lane partials [N][5][32] | the two ray lists that alternate between rounds [N] | the engine's own part (img_bytes: the
// tensor-core engine's forward weight image; none on the exact engine).  S does not enter.
struct FrameWs { size_t carry, chunks, part, list[2], img, total; };
inline FrameWs frame_layout_bytes(int N, size_t img_bytes) {
  FrameWs w{};
  size_t off = align_up((size_t)(FRAME_MAX_ROUNDS + 1) * 4, 256);
  auto take = [&](size_t bytes) { const size_t o = off; off += align_up(bytes, 256); return o; };
  const size_t n = (size_t)N;
  w.carry = take(n * 4); w.chunks = take(n * 4); w.part = take(n * 640); w.list[0] = take(n * 4); w.list[1] = take(n * 4);
  w.img = img_bytes ? take(img_bytes) : off;
  w.total = off;
  return w;
}

// The rounds of nnb_render_frame on either engine: round(f) launches one round (chunk f.k of the rays of f.list, of every ray when it is
// NULL; round k takes its rays from the list round k - 1 appended to), then frame_finish.  Every launch after the first sizes itself from
// a device counter; nothing is read back.
template <class Round>
cudaError_t run_render_frame(const nnb_render_args& a, const FrameWs& w, float t_min, int* n_eval, float* t_final, cudaStream_t st,
                             Round round) {
  char* base = static_cast<char*>(a.workspace);
  auto I = [&](size_t off) { return reinterpret_cast<int*>(base + off); };
  int* counters = I(0);
  cudaError_t e = cudaMemsetAsync(counters, 0, (FRAME_MAX_ROUNDS + 1) * 4, st);
  if (e != cudaSuccess) return e;
  FramePtrs f{};
  f.t_min = t_min;
  f.carry = reinterpret_cast<float*>(base + w.carry); f.chunks = I(w.chunks); f.part = reinterpret_cast<float*>(base + w.part);
  const int rounds = (a.S + 31) / 32;
  for (int k = 0; k < rounds; ++k) {
    f.k = k;
    f.list = k > 0 ? I(w.list[k & 1]) : nullptr; f.count = k > 0 ? counters + k : nullptr;
    f.next_list = I(w.list[(k + 1) & 1]); f.next_count = counters + k + 1;   // not written by the last round
    round(f);
  }
  frame_finish<<<(a.N + 7) / 8, 256, 0, st>>>(a, f, n_eval, t_final);
  return cudaGetLastError();
}


// ---- nnb_render_frame_bwd (the differentiable frame, t_min = 0, either engine): the forward above with checkpoints, then reverse
// rounds k = C - 1 .. 0 (C = ceil(S / 32)).  Round k evaluates chunk k of every ray again with a chunk-sized training stash, runs
// frame_chunk_adjoint, the data-gradient chain and the weight-gradient stage on it, and adds the chunk's point and direction adjoints to
// the ray's lane partials (frame_ray_acc).  frame_ray_finish then forms each ray's pose adjoint from them as ray_bwd does.  Every sum runs
// in a fixed order: chunk by chunk from the last, in the lanes of composite_bwd / ray_bwd.
// Rows of the chunk stash: ray n owns R consecutive rows, row R n + j is sample 32 k + j.  The tensor-core engine pads every ray to R = 32
// rows (PACKED = false); the exact engine packs them, R = min(S, 32) (PACKED = true), so that at S < 32 a round evaluates N S rows.
struct FrameBwdPtrs {
  int k, rounds;          // this round's chunk; C
  const float* ckpt;      // [C - 1][N]: transmittance into chunk k + 1 (after chunk k) of every ray, written by the forward
  float* suffix;          // [N] carry_s of composite_chunk_bwd between rounds
  const SampleRec* rec;   // [R N] records of the chunk (the chunk stash)
  float4* gs;             // [R N] d / d (rgb, a) of the chunk's samples
  const float4 *gp, *gv;  // [R N] d / d p and d / d viewdir of the chunk's samples
  float* raypart;         // [N][9][32] lane partials of ray_bwd's so, sd, sv
};

// rows per ray of the chunk stash (see above)
template <bool PACKED> __device__ __forceinline__ int chunk_rows(const nnb_render_args& a) { return PACKED ? min(a.S, 32) : 32; }

// one warp per ray, lane = sample 32 k + lane: composite_bwd's adjoint of chunk k, the suffix of the later chunks carried in f.suffix.
// A packed ray has no row for a lane past its last sample (lane >= R only when S < 32): that lane writes nothing.  The exact engine's
// instantiation (PACKED) takes composite_bwd's fused form of d L / d alpha (composite_chunk_bwd<true>).
template <bool PACKED>
__global__ void frame_chunk_adjoint(nnb_render_bwd_args b, const __grid_constant__ FrameBwdPtrs f) {
  const nnb_render_args& a = b.fwd;
  const int lane = threadIdx.x & 31, n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (n >= a.N) return;
  Ray ray; setup_ray(a, n, ray);
  float gD = b.g_depth_pred ? __ldg(b.g_depth_pred + n) : 0.f;
  if ((a.flags & NNB_EVAL) && (a.flags & NNB_NORMALISE)) gD = gD / ray.nrm;
  const float gC0 = __ldg(b.g_rgb + 3 * n), gC1 = __ldg(b.g_rgb + 3 * n + 1), gC2 = __ldg(b.g_rgb + 3 * n + 2);
  const float gsum = (a.flags & NNB_WHITE_BG) ? (gC0 + gC1 + gC2) : 0.f;
  const int i = 32 * f.k + lane;
  const bool valid = i < a.S;
  const int R = chunk_rows<PACKED>(a);
  const size_t m = (size_t)n * R + lane;
  const SampleRec me = valid ? f.rec[m] : SampleRec{0, 0, 0, 0, 0, 0, 0, 0};
  float alpha = 0.f, df = 1.f;   // df = d alpha / d a
  if (valid) {
    alpha = composite_alpha(a, i, me.a, me.z, [&] { return sample_z(a, n, i + 1); });
    if (a.flags & NNB_DIST_ALPHA) {
      if (i >= a.S - 1) df = 0.f;
      else { const float delta = __fsub_rn(sample_z(a, n, i + 1), me.z); df = delta * expf(-me.a * delta); }
    }
  }
  const float carry = f.k > 0 ? f.ckpt[(size_t)(f.k - 1) * a.N + n] : 1.f;
  float carry_s = f.k == f.rounds - 1 ? 0.f : f.suffix[n];
  const float4 g = composite_chunk_bwd<PACKED>(alpha, valid, me.r, me.g, me.b, me.z, df, lane, carry, gC0, gC1, gC2, gD, gsum, carry_s);
  if (!PACKED || lane < R) f.gs[m] = g;
  if (lane == 0) f.suffix[n] = carry_s;
}

// one warp per ray: the chunk's terms of ray_bwd's lane sums (lane = sample 32 k + lane), added to the ray's lane partials (written by the
// first round, k = C - 1)
template <bool PACKED>
__global__ void frame_ray_acc(nnb_render_args a, const __grid_constant__ FrameBwdPtrs f) {
  const int lane = threadIdx.x & 31, n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (n >= a.N) return;
  float* part = f.raypart + (size_t)n * 288 + lane;
  float v[9];
#pragma unroll
  for (int c = 0; c < 9; ++c) v[c] = f.k == f.rounds - 1 ? 0.f : part[32 * c];
  if (32 * f.k + lane < a.S) {   // a packed ray's rows: lane < R
    const size_t m = (size_t)n * chunk_rows<PACKED>(a) + lane;
    const float4 g = f.gp[m], dv = f.gv[m];
    const float z = f.rec[m].z;
    v[0] += g.x; v[1] += g.y; v[2] += g.z;
    v[3] += z * g.x; v[4] += z * g.y; v[5] += z * g.z;
    v[6] += dv.x; v[7] += dv.y; v[8] += dv.z;
  }
#pragma unroll
  for (int c = 0; c < 9; ++c) part[32 * c] = v[c];
}

// Early ray termination in the reverse rounds (nnb_render_frame_train_bwd_tmin): ray n evaluated chunks 0 .. c_n - 1 in the forward
// (c_n = FramePtrs::chunks[n], clamped to 1..C), so reverse round k visits only the rays with c_n > k.  frame_live_list writes them to
// `list` in increasing n, with their count in *count; the round's stash row 32 slot + j is sample 32 k + j of ray list[slot], and the
// per-ray kernels run one warp per slot.  A ray starts its suffix carry and lane partials in its own last round, k = c_n - 1.
struct FrameLive { const int* chunks; const int* list; const int* count; };
__device__ __forceinline__ int frame_ray_chunks(const int* chunks, int n, int C) { return min(max(chunks[n], 1), C); }
__device__ __forceinline__ int frame_live_count(const int* count, int N) { return min(max(*count, 0), N); }

// one CTA of 1024 threads: list = {n : c_n > k} in increasing n, *count = its size.  1024 rays at a time, each placed by a block scan of
// the live flags (no atomics: the order of the list is the order of the weight-gradient sums, so it must not depend on scheduling).
__global__ void __launch_bounds__(1024) frame_live_list(const int* __restrict__ chunks, int N, int k, int C, int* __restrict__ list,
                                                        int* __restrict__ count) {
  __shared__ int s_warp[32];
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  int base = 0;
  for (int n0 = 0; n0 < N; n0 += 1024) {
    const int n = n0 + t;
    const int live = n < N && frame_ray_chunks(chunks, n, C) > k ? 1 : 0;
    int x = live;   // inclusive scan over the warp, then over the warps' totals
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
    if (lane == 31) s_warp[warp] = x;
    __syncthreads();
    if (warp == 0) {
      int v = s_warp[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, v, o); if (lane >= o) v += y; }
      s_warp[lane] = v;
    }
    __syncthreads();
    const int before = base + (warp > 0 ? s_warp[warp - 1] : 0) + x - live;
    if (live) list[before] = n;
    base += s_warp[31];
    __syncthreads();   // s_warp is rewritten by the next 1024 rays
  }
  if (t == 0) *count = base;
}

// frame_chunk_adjoint<false> on round k's live list: one warp per slot, ray n = list[slot], rows 32 slot .. 32 slot + 31; the ray's suffix
// starts at 0 in its own last round, k = c_n - 1.  A copy of that kernel's body: shared, nvcc 12.9 changed the existing kernels' SASS.
__global__ void frame_chunk_adjoint_live(nnb_render_bwd_args b, const __grid_constant__ FrameBwdPtrs f, const __grid_constant__ FrameLive l) {
  const nnb_render_args& a = b.fwd;
  const int lane = threadIdx.x & 31, slot = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (slot >= frame_live_count(l.count, a.N)) return;
  const int n = l.list[slot];
  Ray ray; setup_ray(a, n, ray);
  float gD = b.g_depth_pred ? __ldg(b.g_depth_pred + n) : 0.f;
  if ((a.flags & NNB_EVAL) && (a.flags & NNB_NORMALISE)) gD = gD / ray.nrm;
  const float gC0 = __ldg(b.g_rgb + 3 * n), gC1 = __ldg(b.g_rgb + 3 * n + 1), gC2 = __ldg(b.g_rgb + 3 * n + 2);
  const float gsum = (a.flags & NNB_WHITE_BG) ? (gC0 + gC1 + gC2) : 0.f;
  const int i = 32 * f.k + lane;
  const bool valid = i < a.S;
  const size_t m = (size_t)slot * 32 + lane;
  const SampleRec me = valid ? f.rec[m] : SampleRec{0, 0, 0, 0, 0, 0, 0, 0};
  float alpha = 0.f, df = 1.f;   // df = d alpha / d a
  if (valid) {
    alpha = composite_alpha(a, i, me.a, me.z, [&] { return sample_z(a, n, i + 1); });
    if (a.flags & NNB_DIST_ALPHA) {
      if (i >= a.S - 1) df = 0.f;
      else { const float delta = __fsub_rn(sample_z(a, n, i + 1), me.z); df = delta * expf(-me.a * delta); }
    }
  }
  const float carry = f.k > 0 ? f.ckpt[(size_t)(f.k - 1) * a.N + n] : 1.f;
  float carry_s = f.k == frame_ray_chunks(l.chunks, n, f.rounds) - 1 ? 0.f : f.suffix[n];
  f.gs[m] = composite_chunk_bwd<false>(alpha, valid, me.r, me.g, me.b, me.z, df, lane, carry, gC0, gC1, gC2, gD, gsum, carry_s);
  if (lane == 0) f.suffix[n] = carry_s;
}

// frame_ray_acc<false> on round k's live list (a copy, as above): the ray's lane partials are written by its own last round, k = c_n - 1
__global__ void frame_ray_acc_live(nnb_render_args a, const __grid_constant__ FrameBwdPtrs f, const __grid_constant__ FrameLive l) {
  const int lane = threadIdx.x & 31, slot = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (slot >= frame_live_count(l.count, a.N)) return;
  const int n = l.list[slot];
  const bool first = f.k == frame_ray_chunks(l.chunks, n, f.rounds) - 1;
  float* part = f.raypart + (size_t)n * 288 + lane;
  float v[9];
#pragma unroll
  for (int c = 0; c < 9; ++c) v[c] = first ? 0.f : part[32 * c];
  if (32 * f.k + lane < a.S) {
    const size_t m = (size_t)slot * 32 + lane;
    const float4 g = f.gp[m], dv = f.gv[m];
    const float z = f.rec[m].z;
    v[0] += g.x; v[1] += g.y; v[2] += g.z;
    v[3] += z * g.x; v[4] += z * g.y; v[5] += z * g.z;
    v[6] += dv.x; v[7] += dv.y; v[8] += dv.z;
  }
#pragma unroll
  for (int c = 0; c < 9; ++c) part[32 * c] = v[c];
}

// one warp per ray after the last round: ray_bwd's warp sums of the lane partials and its per-ray adjoint -> rayred [N][16] (ray_reduce
// follows)
__global__ void frame_ray_finish(nnb_render_bwd_args b, const float* __restrict__ raypart, float* __restrict__ rayred) {
  const nnb_render_args& a = b.fwd;
  const int lane = threadIdx.x & 31, n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (n >= a.N) return;
  Ray r; setup_ray(a, n, r);
  const float* part = raypart + (size_t)n * 288 + lane;
  float so[3], sd[3], sv[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) { so[c] = warp_sum(part[32 * c]); sd[c] = warp_sum(part[32 * (3 + c)]); sv[c] = warp_sum(part[32 * (6 + c)]); }
  if (lane == 0) ray_adjoint(b, n, r, so, sd, sv, rayred);
}

// Workspace of nnb_render_frame_bwd, every section 256-byte aligned: frame_layout_bytes(N, img_bytes) (the forward, with the engine's forward
// weight image) | checkpoints [C - 1][N] | suffix carries [N] | ray lane partials [N][9][32] | the chunk stash (chunk_bytes: the records,
// training stash, gate bits, per-ray reduction and weight-gradient partials of R N samples) | the engine's transposed weight image.  Only
// the checkpoints grow with S: 4 bytes per ray and chunk.
struct FrameBwdWs { FrameWs f; size_t ckpt, suffix, raypart, chunk, img_t, total; };
inline FrameBwdWs frame_bwd_layout_bytes(int N, int S, size_t img_bytes, size_t chunk_bytes, size_t img_t_bytes) {
  FrameBwdWs w{};
  w.f = frame_layout_bytes(N, img_bytes);
  size_t off = w.f.total;
  auto take = [&](size_t bytes) { const size_t o = off; off += align_up(bytes, 256); return o; };
  const size_t n = (size_t)N;
  w.ckpt = take((size_t)((S + 31) / 32 - 1) * n * 4); w.suffix = take(n * 4); w.raypart = take(n * 288 * 4);
  w.chunk = take(chunk_bytes); w.img_t = take(img_t_bytes);
  w.total = off;
  return w;
}

}  // namespace
