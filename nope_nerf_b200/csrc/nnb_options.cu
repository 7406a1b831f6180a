// Kernels of the training options that the whole-step CUDA graph runs beside the default terms:
//   * the scale / shift invariant depth term (training.depth_loss_type = invariant, model/losses.py:34-57), forward + adjoint;
//   * the learned focal lengths (pose.learn_focal, model/intrinsics.py) into the camera matrix, and their adjoint;
//   * the pose-smoothness terms (training.weight_dist_1st_loss / weight_dist_2nd_loss, model/losses.py:103-112), forward + adjoint.
// Every launch is one CTA: per-step values (loss weights, parameters) are read from device memory, every sum runs in a fixed order
// (thread-strided partials, then a fixed shuffle tree), and no float atomics are used, so the results are reproducible bit for bit.
#include "nnb_common.cuh"

namespace {

constexpr int OPT_THREADS = 1024;

// sum over the block in a fixed order; every thread gets the result
__device__ float block_sum_fixed(float v, float* sh) {
  v = warp_sum(v);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();
  if (l == 0) sh[w] = v;
  __syncthreads();
  float t = (threadIdx.x < (blockDim.x >> 5)) ? sh[threadIdx.x] : 0.f;
  if (w == 0) t = warp_sum(t);
  if (threadIdx.x == 0) sh[32] = t;
  __syncthreads();
  return sh[32];
}

__device__ __forceinline__ float sgn(float x) { return x > 0.f ? 1.f : (x < 0.f ? -1.f : 0.f); }

// order-preserving unsigned key of a float (-0 and +0 share the key of +0, as they compare equal)
__device__ __forceinline__ unsigned order_key(float x) {
  const unsigned u = __float_as_uint(x + 0.f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_value(unsigned k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }

// k-th smallest (0-based) of the masked x[0..N): four 8-bit radix passes over the order-preserving keys (shared-memory histograms,
// integer counts, so the result does not depend on the order of the adds)
__device__ float select_kth(const float* __restrict__ x, const uint8_t* __restrict__ mask, int N, unsigned k, unsigned* hist, unsigned* st) {
  unsigned prefix = 0u, pmask = 0u;
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int i = threadIdx.x; i < 256; i += blockDim.x) hist[i] = 0u;
    __syncthreads();
    for (int n = threadIdx.x; n < N; n += blockDim.x)
      if (mask[n]) {
        const unsigned key = order_key(x[n]);
        if ((key & pmask) == prefix) atomicAdd(&hist[(key >> shift) & 255u], 1u);
      }
    __syncthreads();
    if (threadIdx.x == 0) {
      unsigned c = 0u, b = 0u;
      for (; b < 255u; ++b) { if (c + hist[b] > k) break; c += hist[b]; }
      st[0] = b; st[1] = k - c;
    }
    __syncthreads();
    prefix |= st[0] << shift; pmask |= 255u << shift; k = st[1];
    __syncthreads();
  }
  return key_value(prefix);
}

// Loss.depth_loss_dpt over the masked rays, forward and adjoint.  With n masked rays, a = (p - t_p) / s_p, b = (g - t_g) / s_g
// (t = lower median, s = mean |x - t|), L = mean (a - b)^2 and d_i = a_i - b_i:
//   dL/dp_i = u_i / s_p + G_s sign(p_i - t_p) / n + [p_i == t_p] G_t / c_p,   u_i = 2 c d_i / n (c = w * grad_scale)
//   G_s = dL/ds_p = -sum u_i a_i / s_p,   G_t = dL/dt_p = -sum u_i / s_p - G_s sum sign(p_i - t_p) / n
// and the same for g with u -> -u; c_p = number of masked rays equal to the median (torch.median spreads the gradient evenly over
// them).
__global__ void __launch_bounds__(OPT_THREADS, 1) depth_invariant_k(const float* __restrict__ dp, const float* __restrict__ dg,
                                                                 const uint8_t* __restrict__ mask, int N, const float* w_dev, float grad_scale,
                                                                 float* out, float* g_dp, float* g_dg) {
  __shared__ unsigned hist[256], st[2];
  __shared__ float sh[33];
  const float w = *w_dev;
  if (w == 0.f) return;                                  // the term is off at this point of the annealing schedule
  float c0 = 0.f;
  for (int i = threadIdx.x; i < N; i += blockDim.x) c0 += mask[i] ? 1.f : 0.f;
  const float cnt = block_sum_fixed(c0, sh);
  if (cnt == 0.f) return;
  const unsigned k = ((unsigned)cnt - 1u) / 2u;
  const float tp = select_kth(dp, mask, N, k, hist, st);
  const float tg = select_kth(dg, mask, N, k, hist, st);
  float ap = 0.f, ag = 0.f, cp = 0.f, cg = 0.f;
  for (int i = threadIdx.x; i < N; i += blockDim.x)
    if (mask[i]) {
      ap += fabsf(dp[i] - tp); ag += fabsf(dg[i] - tg);
      cp += dp[i] == tp ? 1.f : 0.f; cg += dg[i] == tg ? 1.f : 0.f;
    }
  ap = block_sum_fixed(ap, sh); ag = block_sum_fixed(ag, sh); cp = block_sum_fixed(cp, sh); cg = block_sum_fixed(cg, sh);
  const float sp = ap / cnt, sg = ag / cnt;
  float l = 0.f, sd = 0.f, sda = 0.f, sdb = 0.f, sgp = 0.f, sgg = 0.f;
  for (int i = threadIdx.x; i < N; i += blockDim.x)
    if (mask[i]) {
      const float a = (dp[i] - tp) / sp, b = (dg[i] - tg) / sg, d = a - b;
      l += d * d; sd += d; sda += d * a; sdb += d * b;
      sgp += sgn(dp[i] - tp); sgg += sgn(dg[i] - tg);
    }
  l = block_sum_fixed(l, sh); sd = block_sum_fixed(sd, sh); sda = block_sum_fixed(sda, sh); sdb = block_sum_fixed(sdb, sh);
  sgp = block_sum_fixed(sgp, sh); sgg = block_sum_fixed(sgg, sh);
  const float L = l / cnt;
  if (threadIdx.x == 0) { out[2] = L; out[0] += w * L; }
  const float coef = 2.f * w * grad_scale / cnt;         // u_i = coef * d_i
  const float gs_p = -coef * sda / sp, gt_p = -coef * sd / sp - gs_p * sgp / cnt;
  const float gs_g = coef * sdb / sg, gt_g = coef * sd / sg - gs_g * sgg / cnt;
  for (int i = threadIdx.x; i < N; i += blockDim.x)
    if (mask[i]) {
      const float a = (dp[i] - tp) / sp, b = (dg[i] - tg) / sg, u = coef * (a - b);
      g_dp[i] += u / sp + gs_p * sgn(dp[i] - tp) / cnt + (dp[i] == tp ? gt_p / cp : 0.f);
      if (g_dg) g_dg[i] += -u / sg + gs_g * sgn(dg[i] - tg) / cnt + (dg[i] == tg ? gt_g / cg : 0.f);
    }
}

// LearnFocal.forward into the camera matrix (training.py:247-252): cam = diag(fx', -fy', -1, 1), (fx', fy') = (fx, fy), squared at
// order 2; fy = fx when fy is null (fx_only)
__global__ void focal_fwd_k(const float* fx, const float* fy, int order, float* cam) {
  const int i = threadIdx.x;
  if (i >= 16) return;
  float a = *fx, b = fy ? *fy : a;
  if (order == 2) { a = a * a; b = b * b; }
  cam[i] = i == 0 ? a : (i == 5 ? -b : (i == 10 ? -1.f : (i == 15 ? 1.f : 0.f)));
}

// its adjoint: d/dfx' = g_cam[0] + g_kxy[0], d/dfy' = -(g_cam[5] + g_kxy[1]), chained through the square at order 2
__global__ void focal_bwd_k(const float* fx, const float* fy, int order, const float* g_cam, const float* g_kxy, float* g_fx, float* g_fy) {
  if (threadIdx.x != 0) return;
  float ga = g_cam[0] + (g_kxy ? g_kxy[0] : 0.f), gb = -(g_cam[5] + (g_kxy ? g_kxy[1] : 0.f));
  const float a = *fx, b = fy ? *fy : a;
  if (order == 2) { ga *= 2.f * a; gb *= 2.f * b; }
  if (fy) { *g_fx += ga; *g_fy += gb; }
  else *g_fx += ga + gb;                                 // fx_only: both diagonal entries come from fx
}

// |t_i - t_{i-1}| and its unit direction (0 at zero length, like the norm's autograd sub-gradient)
__device__ __forceinline__ float seg(const float* t, int i, float u[3]) {
  const float x = t[3 * i] - t[3 * i - 3], y = t[3 * i + 1] - t[3 * i - 2], z = t[3 * i + 2] - t[3 * i - 1];
  const float d = sqrtf(x * x + y * y + z * z);
  const float r = d > 0.f ? 1.f / d : 0.f;
  u[0] = x * r; u[1] = y * r; u[2] = z * r;
  return d;
}

// d (w1 * mean_i dist_i + w2 * mean_j (dist_j - dist_{j-1})^2) / d dist_i, i in [1, V)
__device__ __forceinline__ float dist_grad(const float* t, int V, int i, float w1, float w2) {
  float g = w1 / (float)(V - 1);
  if (V > 2) {
    float u[3];
    const float di = seg(t, i, u);
    float e = 0.f;
    if (i >= 2) e += di - seg(t, i - 1, u);
    if (i + 1 < V) e -= seg(t, i + 1, u) - di;
    g += 2.f * w2 * e / (float)(V - 2);
  }
  return g;
}

// Loss.get_weight_dist_loss: dist_i = |t_i - t_{i-1}| (i = 1..V-1), loss_dist_1st = mean dist, loss_dist_2nd = mean over j = 2..V-1 of
// (dist_j - dist_{j-1})^2 (NaN at V = 2, torch's mean of nothing).  out2 = {1st, 2nd}; loss_total += grad_scale (w1 1st + w2 2nd);
// g_t += grad_scale d(w1 1st + w2 2nd)/dt, one writer per row.  Skipped while both weights are 0.
__global__ void __launch_bounds__(256) pose_smooth_k(const float* __restrict__ t, int V, const float* w_dev, float grad_scale, float* out2,
                                                     float* loss_total, float* g_t) {
  __shared__ float sh[33];
  const float w1 = w_dev[0], w2 = w_dev[1];
  if (w1 == 0.f && w2 == 0.f) return;
  float s1 = 0.f, s2 = 0.f, u[3];
  for (int i = 1 + threadIdx.x; i < V; i += blockDim.x) {
    const float d = seg(t, i, u);
    s1 += d;
    if (i >= 2) { const float e = d - seg(t, i - 1, u); s2 += e * e; }
  }
  s1 = block_sum_fixed(s1, sh); s2 = block_sum_fixed(s2, sh);
  if (threadIdx.x == 0) {
    const float d1 = s1 / (float)(V - 1), d2 = s2 / (float)(V - 2);
    out2[0] = d1; out2[1] = d2;
    if (loss_total) *loss_total += grad_scale * (w1 * d1 + w2 * d2);
  }
  if (!g_t) return;
  for (int r = threadIdx.x; r < V; r += blockDim.x) {
    float g[3] = {0.f, 0.f, 0.f}, v[3];
    if (r >= 1) { const float c = dist_grad(t, V, r, w1, w2); seg(t, r, v); for (int q = 0; q < 3; ++q) g[q] += c * v[q]; }
    if (r + 1 < V) { const float c = dist_grad(t, V, r + 1, w1, w2); seg(t, r + 1, v); for (int q = 0; q < 3; ++q) g[q] -= c * v[q]; }
    for (int q = 0; q < 3; ++q) g_t[3 * r + q] += grad_scale * g[q];
  }
}

}  // namespace

cudaError_t launch_depth_invariant(const float* dp, const float* dg, const uint8_t* mask, int N, const float* w_dev, float grad_scale, float* out,
                                   float* g_dp, float* g_dg, cudaStream_t st) {
  depth_invariant_k<<<1, OPT_THREADS, 0, st>>>(dp, dg, mask, N, w_dev, grad_scale, out, g_dp, g_dg);
  return cudaGetLastError();
}
cudaError_t launch_focal_fwd(const float* fx, const float* fy, int order, float* cam, cudaStream_t st) {
  focal_fwd_k<<<1, 32, 0, st>>>(fx, fy, order, cam);
  return cudaGetLastError();
}
cudaError_t launch_focal_bwd(const float* fx, const float* fy, int order, const float* g_cam, const float* g_kxy, float* g_fx, float* g_fy,
                             cudaStream_t st) {
  focal_bwd_k<<<1, 32, 0, st>>>(fx, fy, order, g_cam, g_kxy, g_fx, g_fy);
  return cudaGetLastError();
}
cudaError_t launch_pose_smooth(const float* t, int V, const float* w_dev, float grad_scale, float* out2, float* loss_total, float* g_t,
                               cudaStream_t st) {
  pose_smooth_k<<<1, 256, 0, st>>>(t, V, w_dev, grad_scale, out2, loss_total, g_t);
  return cudaGetLastError();
}
