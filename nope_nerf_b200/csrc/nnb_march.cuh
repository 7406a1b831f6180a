// The geometry view's fused ray march and one-call frame, the parts both engines share: the march arithmetic and its per-ray state
// (MarchPtrs), the back end of a 128-step block (march_scan), the rounds of the march (run_ray_march) and its end (march_finish), and the
// per-pixel stages of nnb_geometry_frame (geo_rays, geo_compact, geo_shade).  nnb_tc.cu (tc_march / tc_secant) and nnb_simt.cu
// (simt_march / simt_secant) supply the field evaluations.
//
// Every product and sum below is rounded on its own (no FMA contraction), in the order of Renderer.ray_marching / Renderer.secant and of
// Renderer.phong_renderer, so that depths, points, secant iterates and shading carry the bits the torch code computes.
#pragma once
#include "nnb_workspace.cuh"

namespace {

constexpr int MARCH_BLOCK = 128;   // steps of a ray that one round of the march evaluates

__device__ __forceinline__ float march_depth(float near, float far, float frac) {   // near (1 - frac) + far frac
  return __fadd_rn(__fmul_rn(near, __fsub_rn(1.f, frac)), __fmul_rn(far, frac));
}
__device__ __forceinline__ float secant_depth(const float4& b) {   // b = (d_low, d_high, f_low, f_high)
  return __fadd_rn(__fdiv_rn(__fmul_rn(-b.z, __fsub_rn(b.y, b.x)), __fsub_rn(b.w, b.z)), b.x);
}
enum : int { RAY_SEARCHING = 0, RAY_HIT = 1, RAY_OCCUPIED = 2, RAY_NO_HIT = 3 };   // MarchPtrs::status
struct MarchPtrs {
  const float *ray0, *dir, *far, *frac;   // [N][3], [N][3], [N], [n_steps]
  float near, tau;
  int n_steps, n_secant;
  int block;           // march round: this launch evaluates steps 128 block .. 128 block + 127 of its rays
  const int* list;     // march round: the rays of this round (NULL: every ray, tile = ray); secant passes: the hit rays
  const int* count;    // device count of `list` (NULL: the launch's n_tiles)
  int *next_list, *next_count;   // rays still searching after this block
  int *hit_list, *hit_count;
  float* carry;        // [N] val of the ray's last evaluated step
  int *status, *first; // [N]
  float4 *brk0, *brk1; // [N] bracket found by the march | bracket after the secant passes so far
};

// p = ray0 + dir depth of one ray, a product then a sum per component
__device__ __forceinline__ void march_point(const MarchPtrs& q, int ray, float depth, float p[3]) {
#pragma unroll
  for (int c = 0; c < 3; ++c) p[c] = __fadd_rn(__ldg(q.ray0 + (size_t)ray * 3 + c), __fmul_rn(__ldg(q.dir + (size_t)ray * 3 + c), depth));
}
// one secant step of a hit ray: f_mid = f() = occupancy - tau at the iterate of its bracket (brk0 on the first pass, brk1 after) moves
// the low or the high end of the bracket to the iterate; the result goes to brk1
template <class F>
__device__ __forceinline__ void secant_update(const MarchPtrs& q, int ray, bool first_pass, F f) {
  float4 b = (first_pass ? q.brk0 : q.brk1)[ray];
  const float d_mid = secant_depth(b), f_mid = f();
  if (f_mid < 0.f) { b.x = d_mid; b.z = f_mid; } else { b.y = d_mid; b.w = f_mid; }
  q.brk1[ray] = b;
}

// Back end of a march tile, one warp: the first pair (i, i + 1) of the tile's steps, including the pair formed with the previous
// block's last value, whose rounded product val[i] val[i + 1] is negative.  A ray with that pair, or whose very first value is not
// negative, is finished; any other ray with steps left is appended to the next round's list.  s_val: the block's MARCH_BLOCK values.
__device__ __forceinline__ void march_scan(const MarchPtrs& q, int ray, const float* s_val, int lane) {
  const int base = q.block * MARCH_BLOCK;
  const int nv = min(MARCH_BLOCK, q.n_steps - base);   // steps of the ray in this tile; the rows past them were evaluated on a clamped index
  const float prev = lane > 0 ? s_val[4 * lane - 1] : (q.block > 0 ? q.carry[ray] : 0.f);   // 0: step 0 has no predecessor
  const float4 v = *reinterpret_cast<const float4*>(s_val + 4 * lane);
  uint32_t m = 0;
  if (4 * lane + 0 < nv && __fmul_rn(prev, v.x) < 0.f) m |= 1u;
  if (4 * lane + 1 < nv && __fmul_rn(v.x, v.y) < 0.f) m |= 2u;
  if (4 * lane + 2 < nv && __fmul_rn(v.y, v.z) < 0.f) m |= 4u;
  if (4 * lane + 3 < nv && __fmul_rn(v.z, v.w) < 0.f) m |= 8u;
  const uint32_t lanes = __ballot_sync(0xffffffffu, m != 0);
  const int src = lanes ? __ffs(lanes) - 1 : 0;
  const int r = __shfl_sync(0xffffffffu, 4 * lane + __ffs(m) - 1, src);   // tile row of the pair's second step
  if (lane != 0) return;
  if (q.block == 0 && !(s_val[0] < 0.f)) { q.status[ray] = RAY_OCCUPIED; return; }
  if (lanes) {
    const float f_low = r > 0 ? s_val[r - 1] : prev, f_high = s_val[r];
    const int i = base + r - 1;
    q.first[ray] = i;
    q.status[ray] = f_low < 0.f ? RAY_HIT : RAY_NO_HIT;
    if (f_low < 0.f) {
      const float far = __ldg(q.far + ray);
      q.brk0[ray] = make_float4(march_depth(q.near, far, __ldg(q.frac + i)), march_depth(q.near, far, __ldg(q.frac + i + 1)), f_low, f_high);
      q.hit_list[atomicAdd(q.hit_count, 1)] = ray;
    }
  } else if (base + MARCH_BLOCK < q.n_steps) {
    q.carry[ray] = s_val[MARCH_BLOCK - 1];
    q.next_list[atomicAdd(q.next_count, 1)] = ray;
  }
}

// depth (and the optional first / bracket) of every ray from the state the march and the secant passes left
__global__ void march_finish(const __grid_constant__ MarchPtrs q, int N, float* __restrict__ depth, int* __restrict__ first,
                             float4* __restrict__ bracket) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const int s = q.status[i];
  depth[i] = s == RAY_HIT ? secant_depth((q.n_secant > 0 ? q.brk1 : q.brk0)[i]) : (s == RAY_OCCUPIED ? 0.f : __int_as_float(0x7f800000));
  if (first) first[i] = (s == RAY_HIT || s == RAY_NO_HIT) ? q.first[i] : -1;
  if (bracket) bracket[i] = s == RAY_HIT ? q.brk0[i] : make_float4(0.f, 0.f, 0.f, 0.f);
}

// Workspace of nnb_ray_march, every section 256-byte aligned: counters [rounds + 1] (0: hit rays; k >= 1: rays of round k) | status,
// first, carry [N] | the two ray lists that alternate between rounds, the hit list [N] | brk0, brk1 [N] float4 | the engine's own part
// (img_bytes: the tensor-core engine's weight image; none on the exact engine)
struct MarchWs { size_t status, first, carry, list[2], hits, brk0, brk1, img, total; int rounds; };
inline MarchWs march_layout_bytes(int N, int n_steps, size_t img_bytes) {
  MarchWs w{};
  w.rounds = (n_steps + MARCH_BLOCK - 1) / MARCH_BLOCK;
  size_t off = align_up((size_t)(w.rounds + 1) * 4, 256);
  auto take = [&](size_t bytes) { const size_t o = off; off += align_up(bytes, 256); return o; };
  w.status = take((size_t)N * 4); w.first = take((size_t)N * 4); w.carry = take((size_t)N * 4);
  w.list[0] = take((size_t)N * 4); w.list[1] = take((size_t)N * 4); w.hits = take((size_t)N * 4);
  w.brk0 = take((size_t)N * 16); w.brk1 = take((size_t)N * 16);
  w.img = img_bytes ? take(img_bytes) : off;
  w.total = off;
  return w;
}

// The rounds of nnb_ray_march on either engine: round(a, q) launches one round (q.block; the rays of q.list, every ray when it is
// NULL), secant(a, q) the q.n_secant secant passes over the *q.count hit rays of q.list, then march_finish.  Every launch after the first
// sizes itself from a device counter; nothing is read back.
template <class Round, class Secant>
cudaError_t run_ray_march(const nnb_ray_march_args& r, const MarchWs& w, int D, cudaStream_t st, Round round, Secant secant) {
  char* base = static_cast<char*>(r.workspace);
  auto I = [&](size_t off) { return reinterpret_cast<int*>(base + off); };
  int* counters = I(0);
  cudaError_t e = cudaMemsetAsync(base, 0, w.status + (size_t)r.N * 4, st);   // counters and status (RAY_SEARCHING)
  if (e != cudaSuccess) return e;
  nnb_render_args a{};
  a.weights = r.weights; a.flags = (r.flags & (NNB_DIST_ALPHA | NNB_SOFTPLUS)) | NNB_OCC_ONLY; a.hidden_dim = D;
  MarchPtrs q{};
  q.ray0 = r.ray0; q.dir = r.ray_dir; q.far = r.far_; q.frac = r.frac; q.near = r.near_; q.tau = r.tau;
  q.n_steps = r.n_steps; q.n_secant = r.n_secant;
  q.hit_list = I(w.hits); q.hit_count = counters;
  q.carry = reinterpret_cast<float*>(base + w.carry); q.status = I(w.status); q.first = I(w.first);
  q.brk0 = reinterpret_cast<float4*>(base + w.brk0); q.brk1 = reinterpret_cast<float4*>(base + w.brk1);
  for (int k = 0; k < w.rounds; ++k) {
    q.block = k;
    q.list = k > 0 ? I(w.list[k & 1]) : nullptr; q.count = k > 0 ? counters + k : nullptr;
    q.next_list = I(w.list[(k + 1) & 1]); q.next_count = counters + k + 1;   // not written by the last round
    round(a, q);
  }
  if (r.n_secant > 0) {
    q.list = q.hit_list; q.count = counters;
    secant(a, q);
  }
  march_finish<<<(r.N + 255) / 256, 256, 0, st>>>(q, r.N, r.depth, r.first, reinterpret_cast<float4*>(r.bracket));
  return cudaGetLastError();
}

// ---- nnb_geometry_frame: the geometry view (Renderer.phong_renderer) of N pixels on the device ----------------------------------
// Every product, sum, quotient and square root below is rounded on its own (no FMA contraction), in the order the header states.
__device__ __forceinline__ float dot3_rn(const float* u, const float* v) {   // (u0 v0 + u1 v1) + u2 v2
  return __fadd_rn(__fadd_rn(__fmul_rn(u[0], v[0]), __fmul_rn(u[1], v[1])), __fmul_rn(u[2], v[2]));
}
// one thread per pixel: ray origin cw = T[:3, 3], unit direction of pw - cw with pw = T (x, y, 1, 1), far sphere intersection
// (Renderer._rays_world, Renderer._sphere_far)
__global__ void geo_rays(const float* __restrict__ T, const float* __restrict__ pix, int N, float radius, float* __restrict__ ray0,
                         float* __restrict__ dir, float* __restrict__ far, float* __restrict__ o_ray0, float* __restrict__ o_dir,
                         float* __restrict__ o_far) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  float t[12];
#pragma unroll
  for (int k = 0; k < 12; ++k) t[k] = __ldg(T + k);
  const float x = __ldg(pix + 2 * (size_t)i), y = __ldg(pix + 2 * (size_t)i + 1);
  const float c[3] = {t[3], t[7], t[11]};
  float d[3], v[3];
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const float pw = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(t[4 * r], x), __fmul_rn(t[4 * r + 1], y)), t[4 * r + 2]), t[4 * r + 3]);
    d[r] = __fsub_rn(pw, c[r]);
  }
  const float nd = __fsqrt_rn(dot3_rn(d, d));
#pragma unroll
  for (int r = 0; r < 3; ++r) v[r] = __fdiv_rn(d[r], nd);
  const float dt = dot3_rn(v, c), nc = __fsqrt_rn(dot3_rn(c, c));
  const float under = __fsub_rn(__fmul_rn(dt, dt), __fsub_rn(__fmul_rn(nc, nc), __fmul_rn(radius, radius)));
  float f = under > 0.f ? __fsub_rn(__fsqrt_rn(under), dt) : 0.f;
  f = f < 0.f ? 0.f : f;
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    ray0[3 * (size_t)i + r] = c[r]; dir[3 * (size_t)i + r] = v[r];
    if (o_ray0) o_ray0[3 * (size_t)i + r] = c[r];
    if (o_dir) o_dir[3 * (size_t)i + r] = v[r];
  }
  far[i] = f;
  if (o_far) o_far[i] = f;
}
// one thread per pixel, after the march: an object ray (finite depth, not 0) appends its surface point p = ray0 + dir depth, view
// direction -dir, pixel index and the cotangent (0, 0, 0, 1) of the normal to the compacted rows; any other pixel gets its final colours
__global__ void geo_compact(int N, const float* __restrict__ ray0, const float* __restrict__ dir, const float* __restrict__ depth,
                            int* __restrict__ count, float* __restrict__ pts, float* __restrict__ vdir, int* __restrict__ pix,
                            float4* __restrict__ gs, float* __restrict__ rgb, float* __restrict__ rgb_surf, float* __restrict__ o_depth,
                            float4* __restrict__ o_grad) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const float dep = depth[i];
  if (o_depth) o_depth[i] = dep;
  if (isfinite(dep) && dep != 0.f) {
    const int k = atomicAdd(count, 1);   // the row order does not matter: a point's outputs depend on that point alone
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float v = dir[3 * (size_t)i + c];
      pts[3 * (size_t)k + c] = __fadd_rn(ray0[3 * (size_t)i + c], __fmul_rn(v, dep));
      vdir[3 * (size_t)k + c] = -v;
    }
    pix[k] = i;
    gs[k] = make_float4(0.f, 0.f, 0.f, 1.f);
  } else {
#pragma unroll
    for (int c = 0; c < 3; ++c) { rgb[3 * (size_t)i + c] = 1.f; rgb_surf[3 * (size_t)i + c] = 0.f; }
    if (o_grad) o_grad[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
}
// one thread per compacted row k < *count: grad = -d logit / d p, n = grad / |grad|, rgb = min(0.3 + 0.7 max(n . light, 0), 1) with
// light = cw / |cw|, rgb_surf = the colour query's rgb, scattered to the row's pixel.  The clamps are comparisons, so a NaN (a zero
// gradient) passes through them as it does through torch's clamp_min / clamp_max.
__global__ void geo_shade(const float* __restrict__ T, const int* __restrict__ count, const int* __restrict__ pix, const float4* __restrict__ gp,
                          const float4* __restrict__ rgba, float* __restrict__ rgb, float* __restrict__ rgb_surf, float4* __restrict__ o_grad) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= *count) return;
  const int i = pix[k];
  const float4 g4 = gp[k], s4 = rgba[k];
  const float g[3] = {-g4.x, -g4.y, -g4.z}, c[3] = {__ldg(T + 3), __ldg(T + 7), __ldg(T + 11)};
  const float ng = __fsqrt_rn(dot3_rn(g, g)), nc = __fsqrt_rn(dot3_rn(c, c));
  float n[3], l[3];
#pragma unroll
  for (int r = 0; r < 3; ++r) { n[r] = __fdiv_rn(g[r], ng); l[r] = __fdiv_rn(c[r], nc); }
  const float dt = dot3_rn(n, l);
  float s = __fadd_rn(0.3f, __fmul_rn(dt < 0.f ? 0.f : dt, 0.7f));
  s = s > 1.f ? 1.f : s;
  const float surf[3] = {s4.x, s4.y, s4.z};
#pragma unroll
  for (int r = 0; r < 3; ++r) { rgb[3 * (size_t)i + r] = s; rgb_surf[3 * (size_t)i + r] = surf[r]; }
  if (o_grad) o_grad[i] = make_float4(g[0], g[1], g[2], 0.f);
}

}  // namespace
