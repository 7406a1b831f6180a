// Small kernels around the render path: SE(3) exp-map pose (forward + adjoint), fused
// photometric/depth loss + cotangent seeds, dense chamfer point-cloud loss, Adam.
#include "nnb_common.cuh"

namespace {

// ---- LearnPose.forward (model/poses.py:23-31, model/common.py:277-330) ----------------
__device__ void exp_so3(const float r[3], float R[9], float* n_out, float* A_out, float* B_out) {
  float n0 = sqrtf(r[0] * r[0] + r[1] * r[1] + r[2] * r[2]);
  float n = n0 + 1e-15f;                                   // common.py:296
  float A = sinf(n) / n, B = (1.f - cosf(n)) / (n * n);
  float K[9] = {0.f, -r[2], r[1], r[2], 0.f, -r[0], -r[1], r[0], 0.f};
  float K2[9];
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) {
    float s = 0.f; for (int k = 0; k < 3; ++k) s += K[3 * i + k] * K[3 * k + j];
    K2[3 * i + j] = s;
  }
  for (int i = 0; i < 9; ++i) R[i] = ((i % 4 == 0) ? 1.f : 0.f) + A * K[i] + B * K2[i];
  *n_out = n0; *A_out = A; *B_out = B;
}

__global__ void pose_fwd_k(const float* r, const float* t, const float* init, int cam, const int* cam_dev, float* c2w) {
  if (threadIdx.x != 0) return;
  if (cam_dev) cam = *cam_dev;
  float rv[3] = {r[3 * cam], r[3 * cam + 1], r[3 * cam + 2]}, R[9], n0, A, B;
  exp_so3(rv, R, &n0, &A, &B);
  float c[16] = {R[0], R[1], R[2], t[3 * cam], R[3], R[4], R[5], t[3 * cam + 1], R[6], R[7], R[8], t[3 * cam + 2], 0, 0, 0, 1};
  if (init) {
    const float* I = init + 16 * cam;
    for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) {
      float s = 0.f; for (int k = 0; k < 4; ++k) s += c[4 * i + k] * I[4 * k + j];
      c2w[4 * i + j] = s;
    }
  } else for (int i = 0; i < 16; ++i) c2w[i] = c[i];
}

__global__ void pose_bwd_k(const float* r, const float* t, const float* init, int cam, const int* cam_dev, const float* g_c2w, float* g_r, float* g_t) {
  if (threadIdx.x != 0) return;
  if (cam_dev) cam = *cam_dev;
  float g[16];
  if (init) {  // c2w = C @ I  ->  gC = g @ I^T
    const float* I = init + 16 * cam;
    for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) {
      float s = 0.f; for (int k = 0; k < 4; ++k) s += g_c2w[4 * i + k] * I[4 * j + k];
      g[4 * i + j] = s;
    }
  } else for (int i = 0; i < 16; ++i) g[i] = g_c2w[i];
  if (g_t) for (int i = 0; i < 3; ++i) g_t[3 * cam + i] += g[4 * i + 3];
  if (!g_r) return;
  float rv[3] = {r[3 * cam], r[3 * cam + 1], r[3 * cam + 2]}, R[9], n0, A, B;
  exp_so3(rv, R, &n0, &A, &B);
  float gR[9]; for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) gR[3 * i + j] = g[4 * i + j];
  float K[9] = {0.f, -rv[2], rv[1], rv[2], 0.f, -rv[0], -rv[1], rv[0], 0.f};
  float K2[9];
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) { float s = 0.f; for (int k = 0; k < 3; ++k) s += K[3 * i + k] * K[3 * k + j]; K2[3 * i + j] = s; }
  float gA = 0.f, gB = 0.f;
  for (int i = 0; i < 9; ++i) { gA += gR[i] * K[i]; gB += gR[i] * K2[i]; }
  // gK = A gR + B (gR K^T + K^T gR)
  float gK[9];
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) {
    float s1 = 0.f, s2 = 0.f;
    for (int k = 0; k < 3; ++k) { s1 += gR[3 * i + k] * K[3 * j + k]; s2 += K[3 * k + i] * gR[3 * k + j]; }
    gK[3 * i + j] = A * gR[3 * i + j] + B * (s1 + s2);
  }
  float gr[3] = {gK[7] - gK[5], gK[2] - gK[6], gK[3] - gK[1]};
  if (n0 > 0.f) {  // autograd's norm sub-gradient at r = 0 is 0
    float n = n0 + 1e-15f;
    float dA = (cosf(n) * n - sinf(n)) / (n * n);
    float dB = (sinf(n) * n * n - (1.f - cosf(n)) * 2.f * n) / (n * n * n * n);
    float gn = gA * dA + gB * dB;
    for (int i = 0; i < 3; ++i) gr[i] += gn * rv[i] / n0;
  }
  for (int i = 0; i < 3; ++i) g_r[3 * cam + i] += gr[i];
}

// ---- Loss.forward rgb + depth terms (model/losses.py:27-32,59-61,192-202) --------------
__device__ float block_sum(float v, float* sh) {
  v = warp_sum(v);
  int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();
  if (l == 0) sh[w] = v;
  __syncthreads();
  float t = (threadIdx.x < (blockDim.x >> 5)) ? sh[threadIdx.x] : 0.f;
  if (w == 0) t = warp_sum(t);
  if (threadIdx.x == 0) sh[32] = t;
  __syncthreads();
  return sh[32];
}

__global__ void loss_rgb_depth_k(const float* rgb, const float* rgb_gt, const float* img, const float* const* img_pp, const int64_t* ray_idx, int HW,
                                 const float* dp, const float* dg, const uint8_t* mask, int N, float w_rgb, float w_depth,
                                 int rgb_l2, float grad_scale, float* out, float* g_rgb, float* g_dp, float* g_dg, const float* w_dev) {
  __shared__ float sh[33];
  if (img_pp) img = *img_pp;      // frame pointer fetched from device memory (lets a captured CUDA graph follow a new frame)
  if (w_dev) { w_rgb = w_dev[0]; w_depth = w_dev[1]; }   // annealed weights (training.py:208-217) without re-capturing the graph
  float l1 = 0.f, l2 = 0.f, ld = 0.f, cnt = 0.f;
  for (int n = threadIdx.x; n < N; n += blockDim.x) {
    for (int c = 0; c < 3; ++c) {
      float gt = rgb_gt ? rgb_gt[3 * n + c] : img[(size_t)c * HW + ray_idx[n]];
      float d = rgb[3 * n + c] - gt;
      l1 += fabsf(d); l2 += d * d;
    }
    if (mask[n]) { cnt += 1.f; ld += fabsf(dp[n] - dg[n]); }
  }
  l1 = block_sum(l1, sh); l2 = block_sum(l2, sh); ld = block_sum(ld, sh); cnt = block_sum(cnt, sh);
  float cden = fmaxf(cnt, 1.f);
  if (threadIdx.x == 0) {
    float lrgb = (rgb_l2 ? l2 : l1) / (float)N, ldep = ld / cden;
    out[0] = w_rgb * lrgb + w_depth * ldep; out[1] = lrgb; out[2] = ldep; out[3] = l2 / (3.f * (float)N);
  }
  for (int n = threadIdx.x; n < N; n += blockDim.x) {
    for (int c = 0; c < 3; ++c) {
      float gt = rgb_gt ? rgb_gt[3 * n + c] : img[(size_t)c * HW + ray_idx[n]];
      float d = rgb[3 * n + c] - gt;
      float g = rgb_l2 ? 2.f * d : (d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f));
      g_rgb[3 * n + c] = grad_scale * w_rgb * g / (float)N;
    }
    float gd = 0.f;
    if (mask[n]) { float d = dp[n] - dg[n]; gd = grad_scale * w_depth * (d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f)) / cden; }
    g_dp[n] = gd; g_dg[n] = -gd;
  }
}

// ---- dense chamfer (model/losses.py:114-148) ---------------------------------------------
// Brute-force nearest neighbour of every a in A among B (the reference materialises the (P,Q) distance matrix and takes
// torch.argmin: ties -> first index), both directions in ONE launch, then mean |a - b_nn| and its adjoints.
//   * SIMT fp32, 2 * P * Q pairs (P = Q = 16 128 at the 384x672 DPT map / pc_ratio 4: 520 M pairs, ~6 instructions each).
//   * squared distances in the difference form (a-b)^2 (no cancellation, no sqrt per pair: the MUFU pipe is 1/4 rate); ordering
//     by d^2 equals ordering by |a-b| and exact duplicates keep the first index.
//   * one thread owns 4 queries, the target comes from shared memory already duplicated (bx,bx | by,by | bz,bz) so every
//     LDS feeds two queries.
constexpr int NS_THREADS = 128, NS_QPT = 4, NS_CHUNK = 256;

// two fp32 lanes, each rounded like a scalar sub / mul / fma (the (a-b)^2 ordering and tie-breaking stay those of scalar code)
__device__ __forceinline__ float2 pk2(float a, float b) { return make_float2(a, b); }
__device__ __forceinline__ void upk2(float2 v, float& a, float& b) { a = v.x; b = v.y; }
__device__ __forceinline__ float2 sub2(float2 a, float2 b) { return make_float2(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y)); }
__device__ __forceinline__ float2 mul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 fma2(float2 a, float2 b, float2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }

__global__ void __launch_bounds__(NS_THREADS) nn_search_k(const float* __restrict__ X, int P, const float* __restrict__ Y, int Q,
                                                          unsigned long long* kxy, unsigned long long* kyx, int per_split) {
  const bool rev = blockIdx.z != 0;
  const float* __restrict__ A = rev ? Y : X; const float* __restrict__ B = rev ? X : Y;
  const int na = rev ? Q : P, nb = rev ? P : Q;
  unsigned long long* keys = rev ? kyx : kxy;
  if (blockIdx.x * (NS_THREADS * NS_QPT) >= na) return;
  const int t0 = blockIdx.y * per_split, t1 = min(nb, t0 + per_split);
  if (t0 >= t1) return;
  __shared__ float4 sxy[NS_CHUNK];                // {(bx,bx), (by,by)}
  __shared__ float2 sz[NS_CHUNK];                 // (bz,bz)
  const int q0 = (blockIdx.x * NS_THREADS + threadIdx.x) * NS_QPT;
  float a[NS_QPT][3];
#pragma unroll
  for (int j = 0; j < NS_QPT; ++j)
#pragma unroll
    for (int c = 0; c < 3; ++c) a[j][c] = (q0 + j < na) ? A[3 * (size_t)(q0 + j) + c] : 0.f;
  const float2 ax0 = pk2(a[0][0], a[1][0]), ay0 = pk2(a[0][1], a[1][1]), az0 = pk2(a[0][2], a[1][2]);
  const float2 ax1 = pk2(a[2][0], a[3][0]), ay1 = pk2(a[2][1], a[3][1]), az1 = pk2(a[2][2], a[3][2]);
  float best[NS_QPT]; int bi[NS_QPT];
#pragma unroll
  for (int j = 0; j < NS_QPT; ++j) { best[j] = INFINITY; bi[j] = 0; }
  for (int c0 = t0; c0 < t1; c0 += NS_CHUNK) {
    const int n = min(NS_CHUNK, t1 - c0);
    __syncthreads();
    for (int k = threadIdx.x; k < n; k += NS_THREADS) {
      const float bx = B[3 * (size_t)(c0 + k)], by = B[3 * (size_t)(c0 + k) + 1], bz = B[3 * (size_t)(c0 + k) + 2];
      sxy[k] = make_float4(bx, bx, by, by); sz[k] = pk2(bz, bz);
    }
    __syncthreads();
#pragma unroll 4
    for (int k = 0; k < n; ++k) {
      const float4 u4 = sxy[k]; const float2 ux = make_float2(u4.x, u4.y), uy = make_float2(u4.z, u4.w), w = sz[k];
      float2 dx = sub2(ax0, ux), dy = sub2(ay0, uy), dz = sub2(az0, w);
      const float2 e0 = fma2(dz, dz, fma2(dy, dy, mul2(dx, dx)));
      dx = sub2(ax1, ux); dy = sub2(ay1, uy); dz = sub2(az1, w);
      const float2 e1 = fma2(dz, dz, fma2(dy, dy, mul2(dx, dx)));
      float d[NS_QPT];
      upk2(e0, d[0], d[1]); upk2(e1, d[2], d[3]);
#pragma unroll
      for (int j = 0; j < NS_QPT; ++j) if (d[j] < best[j]) { best[j] = d[j]; bi[j] = c0 + k; }
    }
  }
#pragma unroll
  for (int j = 0; j < NS_QPT; ++j)
    if (q0 + j < na) atomicMin(keys + q0 + j, ((unsigned long long)__float_as_uint(best[j]) << 32) | (unsigned)bi[j]);
}
// Reduction after the search, with results fixed by the inputs alone (no float atomics).  Points are numbered in one space u in
// [0, P + Q): X[u] for u < P, Y[u - P] after.  Every point is the source of one pair (itself -> its nearest neighbour, term
// weight * v / (|v| * n) with v = a - b_nn) and the target of the pairs whose nearest neighbour it is; its adjoint is its own term
// minus the sum of its group's terms.
//   * chamfer_pairs_k: per point its own term (+= into its adjoint, one writer per element), the term in 64-bit fixed point added
//     into its target's accumulator (integer atomics: the sum is exact, so the order of the adds cannot change a bit), and one loss
//     partial per block (stored in the block's first key slot, which no other block reads);
//   * chamfer_finish_k: per point, minus its accumulator rounded once to float; block 0's first warp adds up the loss partials.
// A target that is everyone's nearest neighbour gets P same-address integer adds, as many as the float scatter had.
constexpr int CH_THREADS = 256;

// the pair term weight * v / (|v| * na) of a -> b (zero for a zero-length pair)
__device__ __forceinline__ void pair_term(const float* A, const float* B, int i, int j, int na, float weight, float& dist, float t[3]) {
  const float vx = __fsub_rn(A[3 * i], B[3 * j]), vy = __fsub_rn(A[3 * i + 1], B[3 * j + 1]), vz = __fsub_rn(A[3 * i + 2], B[3 * j + 2]);
  dist = __fsqrt_rn(__fmaf_rn(vz, vz, __fmaf_rn(vy, vy, __fmul_rn(vx, vx))));
  const float s = dist > 0.f ? __fdiv_rn(weight, __fmul_rn(dist, (float)na)) : 0.f;
  t[0] = __fmul_rn(s, vx); t[1] = __fmul_rn(s, vy); t[2] = __fmul_rn(s, vz);
}

// Fixed point of the group sums: a finite term of a source in a cloud of na points has components of magnitude <= |weight| / na
// (|v_c| <= |v|), and a group has at most na of them, so the terms scaled by 2^F na / |weight| with F = 62 - bits(na) and rounded to
// integers add up in 64 bits without overflow.  Each term is rounded to a quantum of 2^-F |weight| / na (2^-48 |weight| / na at
// na = 16 128) before the exact sum; the sum is rounded to float once.
__device__ __forceinline__ double group_scale(int na, float weight) {
  return weight != 0.f ? ldexp((double)na / fabs((double)weight), 62 - (32 - __clz(na))) : 0.0;
}

// keys [P + Q]: kxy then kyx.  With adjoints: acc [P + Q][3] fixed-point group sums and bad [P + Q] (bit c: a non-finite term in
// component c), zeroed by the caller
__global__ void __launch_bounds__(CH_THREADS) chamfer_pairs_k(const float* X, int P, const float* Y, int Q, unsigned long long* keys,
                                                               float weight, const float* weight_dev, float* gX, float* gY, int* ixy, int* iyx,
                                                               unsigned long long* acc, unsigned* bad) {
  __shared__ float sh[33];
  const int u = blockIdx.x * blockDim.x + threadIdx.x;
  const bool rev = u >= P; const int i = rev ? u - P : u;
  const float* A = rev ? Y : X; const float* B = rev ? X : Y; const int na = rev ? Q : P;
  float* gA = rev ? gY : gX;
  if (weight_dev) weight = *weight_dev;
  float dist = 0.f;
  if (u < P + Q) {
    const int j = (int)(unsigned)(keys[u] & 0xffffffffull);
    if (ixy) (rev ? iyx : ixy)[i] = j;
    float t[3];
    pair_term(A, B, i, j, na, weight, dist, t);
    if (gA) {
      const int tu = rev ? j : P + j;
      const double sc = group_scale(na, weight);
      unsigned nf = 0;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        gA[3 * i + c] += t[c];
        if (!isfinite(t[c])) { nf |= 1u << c; continue; }
        const long long q = __double2ll_rn((double)t[c] * sc);
        if (q != 0) atomicAdd(acc + 3 * (size_t)tu + c, (unsigned long long)q);
      }
      if (nf) atomicOr(bad + tu, nf);
    }
    dist /= (float)na;
  }
  // blocks never straddle the two directions' normalisation because dist is already divided by its own count
  const float tot = block_sum(dist, sh);        // its barriers order every read of this block's keys before the store below
  if (threadIdx.x == 0) reinterpret_cast<float*>(keys + (size_t)blockIdx.x * CH_THREADS)[0] = tot;
}

// loss += the nb block partials, summed by one warp in a fixed order
__device__ __forceinline__ void add_loss_partials(const unsigned long long* keys, int nb, float* loss) {
  float s = 0.f;
  for (int b = threadIdx.x; b < nb; b += 32) s += reinterpret_cast<const float*>(keys + (size_t)b * CH_THREADS)[0];
  s = warp_sum(s);
  if (threadIdx.x == 0) loss[0] += s;
}
__global__ void chamfer_loss_k(const unsigned long long* keys, int nb, float* loss) { add_loss_partials(keys, nb, loss); }

// a component that received a non-finite term becomes NaN (the float scatter would have carried the NaN / Inf as well)
__global__ void __launch_bounds__(CH_THREADS) chamfer_finish_k(int P, int Q, const unsigned long long* __restrict__ acc,
                                                                const unsigned* __restrict__ bad, float weight, const float* weight_dev,
                                                                float* gX, float* gY, const unsigned long long* keys, int nb, float* loss) {
  if (blockIdx.x == 0 && threadIdx.x < 32) add_loss_partials(keys, nb, loss);
  const int u = blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= P + Q) return;
  if (weight_dev) weight = *weight_dev;
  const bool tx = u < P;                       // an X point's group are Y points (na = Q), and the other way round
  const double sc = group_scale(tx ? Q : P, weight);
  if (sc == 0.0) return;
  float* g = tx ? gX + 3 * (size_t)u : gY + 3 * (size_t)(u - P);
  const unsigned b = bad[u];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const long long v = (long long)acc[3 * (size_t)u + c];
    if ((b >> c) & 1u) g[c] = __int_as_float(0x7fffffff);
    else if (v != 0) g[c] -= (float)((double)v / sc);
  }
}

// Learn_Distortion.forward (model/distortions.py:19-27) for a device-resident camera index:
//   scale_eff = fixed-last-view ? 1 : max(scale, 0.01) ; shift = shifts[cam]   -> out[2]
__global__ void distortion_fwd_k(const float* scales, const float* shifts, int V, const int* cam_dev, int fix_last, float* out) {
  if (threadIdx.x != 0) return;
  int cam = *cam_dev;
  float s = scales[cam];
  if (s < 0.01f) s = 0.01f;
  if (fix_last && cam == V - 1) s = 1.f;
  out[0] = s; out[1] = shifts[cam];
}
// its adjoint: the constant replacements carry no gradient
__global__ void distortion_bwd_k(const float* scales, int V, const int* cam_dev, int fix_last, const float* g_ss, float* g_scales, float* g_shifts) {
  if (threadIdx.x != 0) return;
  int cam = *cam_dev;
  bool live = scales[cam] >= 0.01f && !(fix_last && cam == V - 1);
  if (g_scales && live) g_scales[cam] += g_ss[0];
  if (g_shifts) g_shifts[cam] += g_ss[1];
}
// Adam with device-resident step counter and learning rate (CUDA-graph friendly): state = {step (int32), lr (float)}
__global__ void adam_dev_k(float* p, const float* g, float* m, float* v, int64_t n, const int* step_dev, const float* lr_dev, float b1, float b2, float eps) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int step = *step_dev;
  const float bc1 = 1.f - powf(b1, (float)step), bc2 = 1.f - powf(b2, (float)step);
  const float lr_bc1 = *lr_dev / bc1, rsqrt_bc2 = rsqrtf(bc2);
  float gi = g[i];
  float mi = b1 * m[i] + (1.f - b1) * gi;
  float vi = b2 * v[i] + (1.f - b2) * gi * gi;
  m[i] = mi; v[i] = vi;
  p[i] -= lr_bc1 * mi / (sqrtf(vi) * rsqrt_bc2 + eps);
}
__global__ void incr_k(int* a, int n) { if (threadIdx.x < n) a[threadIdx.x] += 1; }

// N distinct pixel ids uniformly from [0, HW): rejection sampling against a shared-memory hash set.
// u holds 2N uniforms in [0,1) (torch.rand); same distribution as torch.randperm(HW)[:N] (training.py:257) at a
// fraction of its cost (randperm sorts all HW keys).  Deterministic for a given u: a duplicated candidate is kept by
// the lowest ray index, first draws beat redraws, and the (very rare) leftovers are resolved serially.
__device__ __forceinline__ int hs_claim(int* key, int* owner, int tsize, int cand, int who) {
  unsigned h = ((unsigned)cand * 2654435761u) & (unsigned)(tsize - 1);
  while (true) {
    int prev = atomicCAS(&key[h], -1, cand);
    if (prev == -1 || prev == cand) { atomicMin(&owner[h], who); return (int)h; }
    h = (h + 1) & (unsigned)(tsize - 1);
  }
}
__global__ void sample_pixels_k(const float* __restrict__ u, int HW, int N, int tsize, long long* __restrict__ out) {
  extern __shared__ int hs[];   // key[tsize] | owner[tsize] | pending list
  int* key = hs; int* owner = hs + tsize; int* pend = owner + tsize; __shared__ int npend;
  for (int i = threadIdx.x; i < tsize; i += blockDim.x) { key[i] = -1; owner[i] = 0x7fffffff; }
  if (threadIdx.x == 0) npend = 0;
  __syncthreads();
  // round 1: first draw, ties -> lowest ray index
  for (int i = threadIdx.x; i < N; i += blockDim.x) {
    int cand = min(HW - 1, (int)(u[i] * (float)HW));
    out[i] = ((long long)hs_claim(key, owner, tsize, cand, i) << 32) | (unsigned)cand;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < N; i += blockDim.x) {
    int slot = (int)(out[i] >> 32), cand = (int)(out[i] & 0xffffffffll);
    out[i] = (owner[slot] == i) ? (long long)cand : -1ll;
  }
  __syncthreads();
  // round 2: losers redraw; first-round winners always outrank them (who = N + i)
  for (int i = threadIdx.x; i < N; i += blockDim.x) {
    if (out[i] >= 0) continue;
    int cand = min(HW - 1, (int)(u[i + N] * (float)HW));
    out[i] = -2ll - (((long long)hs_claim(key, owner, tsize, cand, N + i) << 32) | (unsigned)cand);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < N; i += blockDim.x) {
    if (out[i] >= 0) continue;
    long long enc = -2ll - out[i];
    int slot = (int)(enc >> 32), cand = (int)(enc & 0xffffffffll);
    if (owner[slot] == N + i) out[i] = cand;
    else { int k = atomicAdd(&npend, 1); pend[k] = i; out[i] = -(long long)cand - 2; }
  }
  __syncthreads();
  if (threadIdx.x == 0 && npend > 0) {   // leftovers (probability ~ (N/HW)^2 each): next free id, in ray order
    for (int a = 1; a < npend; ++a) { int v = pend[a], b = a - 1; while (b >= 0 && pend[b] > v) { pend[b + 1] = pend[b]; --b; } pend[b + 1] = v; }
    for (int k = 0; k < npend; ++k) {
      int i = pend[k]; int cand = (int)(-(out[i] + 2));
      while (true) {
        cand = (cand + 1) % HW;
        unsigned h = ((unsigned)cand * 2654435761u) & (unsigned)(tsize - 1);
        bool found = false;
        while (key[h] != -1) { if (key[h] == cand) { found = true; break; } h = (h + 1) & (unsigned)(tsize - 1); }
        if (!found) { key[h] = cand; break; }
      }
      out[i] = cand;
    }
  }
}

__global__ void adam_k(float* p, const float* g, float* m, float* v, int64_t n, float lr_bc1, float rsqrt_bc2, float b1, float b2, float eps) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float gi = g[i];
  float mi = b1 * m[i] + (1.f - b1) * gi;
  float vi = b2 * v[i] + (1.f - b2) * gi * gi;
  m[i] = mi; v[i] = vi;
  p[i] -= lr_bc1 * mi / (sqrtf(vi) * rsqrt_bc2 + eps);
}

}  // namespace

cudaError_t launch_pose_fwd(const float* r, const float* t, const float* init, int cam, const int* cam_dev, float* c2w, cudaStream_t st) {
  pose_fwd_k<<<1, 32, 0, st>>>(r, t, init, cam, cam_dev, c2w); return cudaGetLastError();
}
cudaError_t launch_pose_bwd(const float* r, const float* t, const float* init, int cam, const int* cam_dev, const float* g, float* gr, float* gt,
                            cudaStream_t st) {
  pose_bwd_k<<<1, 32, 0, st>>>(r, t, init, cam, cam_dev, g, gr, gt); return cudaGetLastError();
}
cudaError_t launch_distortion_fwd(const float* sc, const float* sh, int V, const int* cam_dev, int fix_last, float* out, cudaStream_t st) {
  distortion_fwd_k<<<1, 32, 0, st>>>(sc, sh, V, cam_dev, fix_last, out); return cudaGetLastError();
}
cudaError_t launch_distortion_bwd(const float* sc, int V, const int* cam_dev, int fix_last, const float* g_ss, float* g_sc, float* g_sh, cudaStream_t st) {
  distortion_bwd_k<<<1, 32, 0, st>>>(sc, V, cam_dev, fix_last, g_ss, g_sc, g_sh); return cudaGetLastError();
}
cudaError_t launch_adam_dev(float* p, const float* g, float* m, float* v, int64_t n, const int* step_dev, const float* lr_dev, float b1, float b2,
                            float eps, cudaStream_t st) {
  adam_dev_k<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(p, g, m, v, n, step_dev, lr_dev, b1, b2, eps); return cudaGetLastError();
}
cudaError_t launch_sample_pixels(const float* u, int HW, int N, long long* out, cudaStream_t st) {
  int tsize = 1024; while (tsize < 4 * N) tsize <<= 1;
  if (((size_t)2 * tsize + N) * 4 > 200 * 1024) tsize >>= 1;     // N in (4096, 8192]: load factor 1/2 still fits 200 KB
  size_t smem = ((size_t)2 * tsize + N) * 4;
  if (smem > 200 * 1024) return cudaErrorInvalidValue;
  static bool attr = false;
  if (!attr) { cudaFuncSetAttribute(sample_pixels_k, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024); attr = true; }
  sample_pixels_k<<<1, 1024, smem, st>>>(u, HW, N, tsize, out);
  return cudaGetLastError();
}
cudaError_t launch_incr(int* a, int n, cudaStream_t st) { incr_k<<<1, 32, 0, st>>>(a, n); return cudaGetLastError(); }
cudaError_t launch_loss(const float* rgb, const float* rgb_gt, const float* img, const float* const* img_pp, const int64_t* ray_idx, int HW,
                        const float* dp, const float* dg, const uint8_t* mask, int N, float w_rgb, float w_depth, int l2, float gscale, float* out,
                        float* g_rgb, float* g_dp, float* g_dg, const float* w_dev, cudaStream_t st) {
  loss_rgb_depth_k<<<1, 1024, 0, st>>>(rgb, rgb_gt, img, img_pp, ray_idx, HW, dp, dg, mask, N, w_rgb, w_depth, l2, gscale, out, g_rgb, g_dp, g_dg,
                                       w_dev);
  return cudaGetLastError();
}
// Scratch of the chamfer: the search keys (64-bit, P + Q), then with adjoints acc [P + Q][3] (64-bit) and bad [P + Q] (32-bit)
static size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }
size_t chamfer_workspace_bytes(int P, int Q) {
  const size_t n = (size_t)P + (size_t)Q;
  return align256(n * sizeof(unsigned long long)) + n * (3 * sizeof(unsigned long long) + sizeof(unsigned));
}

// ws: caller scratch of chamfer_workspace_bytes(P, Q) bytes, or (P + Q) 64-bit keys when gX / gY are null; optional int32 index
// outputs for the C ABI
cudaError_t launch_chamfer_full(const float* X, int P, const float* Y, int Q, void* ws, float* loss, float weight, const float* weight_dev,
                                float* gX, float* gY, int* ixy, int* iyx, cudaStream_t st) {
  const int n = P + Q;
  unsigned long long* kxy = static_cast<unsigned long long*>(ws); unsigned long long* kyx = kxy + P;
  cudaError_t e = cudaMemsetAsync(kxy, 0xff, sizeof(unsigned long long) * (size_t)n, st);
  if (e != cudaSuccess) return e;
  unsigned long long* acc = nullptr; unsigned* bad = nullptr;
  if (gX) {
    acc = reinterpret_cast<unsigned long long*>(static_cast<char*>(ws) + align256((size_t)n * sizeof(unsigned long long)));
    bad = reinterpret_cast<unsigned*>(acc + 3 * (size_t)n);
    e = cudaMemsetAsync(acc, 0, (size_t)n * (3 * sizeof(unsigned long long) + sizeof(unsigned)), st);
    if (e != cudaSuccess) return e;
  }
  const int per_block = NS_THREADS * NS_QPT, mx = P > Q ? P : Q;
  const int bx = (mx + per_block - 1) / per_block;
  int splits = (2 * 148 + bx - 1) / bx;                       // ~4 resident blocks per SM over both directions
  const int mn = P < Q ? P : Q;
  if (splits > (mn + NS_CHUNK - 1) / NS_CHUNK) splits = (mn + NS_CHUNK - 1) / NS_CHUNK;
  if (splits < 1) splits = 1;
  int per_split = (mx + splits - 1) / splits;
  per_split = (per_split + 3) & ~3;
  nn_search_k<<<dim3(bx, splits, 2), NS_THREADS, 0, st>>>(X, P, Y, Q, kxy, kyx, per_split);
  const int nb = (n + CH_THREADS - 1) / CH_THREADS;
  chamfer_pairs_k<<<nb, CH_THREADS, 0, st>>>(X, P, Y, Q, kxy, weight, weight_dev, gX, gY, ixy, iyx, acc, bad);
  if (gX) chamfer_finish_k<<<nb, CH_THREADS, 0, st>>>(P, Q, acc, bad, weight, weight_dev, gX, gY, kxy, nb, loss);
  else chamfer_loss_k<<<1, 32, 0, st>>>(kxy, nb, loss);
  return cudaGetLastError();
}
cudaError_t launch_chamfer_dev(const float* X, int P, const float* Y, int Q, void* ws, float* loss, const float* weight_dev, float* gX, float* gY,
                               cudaStream_t st) {
  return launch_chamfer_full(X, P, Y, Q, ws, loss, 1.f, weight_dev, gX, gY, nullptr, nullptr, st);
}
cudaError_t launch_adam(float* p, const float* g, float* m, float* v, int64_t n, int step, float lr, float b1, float b2, float eps, cudaStream_t st) {
  double bc1 = 1.0 - pow((double)b1, step), bc2 = 1.0 - pow((double)b2, step);
  adam_k<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(p, g, m, v, n, (float)(lr / bc1), (float)(1.0 / sqrt(bc2)), b1, b2, eps);
  return cudaGetLastError();
}
