// Shared device code of both engines: ray generation, prior-depth gather, sampling,
// positional encoding, alpha compositing (forward + adjoint) and the flat parameter layout.
// Reference semantics: model/rendering.py:36-197, model/common.py:13-39,112-160,632-675,
// model/network.py:19-33, model/official_nerf.py:99-119 (SURVEY.md appendix A).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>
#include "../../include/nope_nerf_b200.h"

#define NNB_EPS 1e-6f  // model/rendering.py:9

// ---- flat parameter layout (floats), OfficialStaticNerf.parameters() order, for hidden width D -------------
namespace nnb {
constexpr int PE = 63;   // (2*10+1)*3
constexpr int DE = 27;   // (2*4+1)*3
// widths with a kernel instantiation (model.hidden_dim); nnb_render_args.hidden_dim == 0 means 256
__host__ __device__ constexpr bool dim_supported(int D) { return D == 64 || D == 128 || D == 256; }
// trunk layer l = 0..7 (layers0.{0,2,4,6}, layers1.{0,2,4,6}): weight (D x w_ld) then bias (D)
__host__ __device__ constexpr int w_ld(int D, int l) { return l == 0 ? PE : (l == 4 ? D + PE : D); }
__host__ __device__ constexpr int w_off(int D, int l) {
  return l == 0 ? 0
       : (l < 4 ? D * PE + D + (l - 1) * (D * D + D)
       : (l == 4 ? D * PE + D + 3 * (D * D + D)
       : D * PE + D + 3 * (D * D + D) + D * (D + PE) + D + (l - 5) * (D * D + D)));
}
__host__ __device__ constexpr int b_off(int D, int l) { return w_off(D, l) + D * w_ld(D, l); }
__host__ __device__ constexpr int W_SIG(int D) { return b_off(D, 7) + D; }               // fc_density (1 x D)
__host__ __device__ constexpr int B_SIG(int D) { return W_SIG(D) + D; }
__host__ __device__ constexpr int W_FEAT(int D) { return B_SIG(D) + 1; }                 // fc_feature (D x D)
__host__ __device__ constexpr int B_FEAT(int D) { return W_FEAT(D) + D * D; }
__host__ __device__ constexpr int W_RGBH(int D) { return B_FEAT(D) + D; }                // rgb_layers.0 (D/2 x (D + 27))
__host__ __device__ constexpr int B_RGBH(int D) { return W_RGBH(D) + (D / 2) * (D + DE); }
__host__ __device__ constexpr int W_RGB(int D) { return B_RGBH(D) + D / 2; }             // fc_rgb (3 x D/2)
__host__ __device__ constexpr int B_RGB(int D) { return W_RGB(D) + 3 * (D / 2); }
__host__ __device__ constexpr int num_params(int D) { return B_RGB(D) + 3; }
static_assert(W_SIG(256) == 493056 && B_SIG(256) == 493312 && W_FEAT(256) == 493313 && B_FEAT(256) == 558849 && W_RGBH(256) == 559105 &&
              B_RGBH(256) == 595329 && W_RGB(256) == 595457 && B_RGB(256) == 595841, "layout");
static_assert(w_off(256, 3) == 147968 && b_off(256, 3) == 213504 && w_off(256, 7) == 427264 && b_off(256, 7) == 492800 &&
              b_off(256, 4) == 295424, "layout");
static_assert(num_params(256) == NNB_NUM_PARAMS && num_params(128) == 158660 && num_params(64) == 44516, "layout");
}  // namespace nnb

struct Ray {
  float x, y;             // pixel in [-1,1]
  float kx, ky;
  float R[9], t[3];
  float dc[3];            // camera-space direction (x/kx, y/ky, -1)
  float dt[3];            // R dc  (ray_vector before normalisation)
  float nrm;              // |R dc|
  float d[3];             // sampling direction (normalised if NNB_NORMALISE)
  float depth_raw, depth; // prior depth before/after distortion
  float g;                // prior distance d_i_gt (rendering.py:57-60,70-71)
  bool mask;
  // NDC (common.py:632-675)
  float O[3], Dn[3], o2[3], tau;
};

__device__ __forceinline__ float ld_scalar(const float* p, float dflt) { return p ? __ldg(p) : dflt; }

__device__ inline void setup_ray(const nnb_render_args& a, int n, Ray& r) {
  if (a.pixels) {
    r.x = __ldg(a.pixels + 2 * n); r.y = __ldg(a.pixels + 2 * n + 1);
  } else {  // arange_pixels (common.py:29-39) evaluated at ray_idx
    long long idx = a.ray_idx[n];
    int row = (int)(idx / a.W), col = (int)(idx % a.W);
    r.x = __fsub_rn(__fdiv_rn(2.f * (float)col, (float)(a.W - 1)), 1.f);
    r.y = __fsub_rn(__fdiv_rn(2.f * (float)row, (float)(a.H - 1)), 1.f);
  }
  r.kx = __ldg(a.cam + 0); r.ky = __ldg(a.cam + 5);
#pragma unroll
  for (int i = 0; i < 3; ++i) {
#pragma unroll
    for (int j = 0; j < 3; ++j) r.R[3 * i + j] = __ldg(a.c2w + 4 * i + j);
    r.t[i] = __ldg(a.c2w + 4 * i + 3);
  }
  r.dc[0] = __fdiv_rn(r.x, r.kx); r.dc[1] = __fdiv_rn(r.y, r.ky); r.dc[2] = -1.f;
#pragma unroll
  for (int i = 0; i < 3; ++i)
    r.dt[i] = __fadd_rn(__fadd_rn(__fmul_rn(r.R[3 * i], r.dc[0]), __fmul_rn(r.R[3 * i + 1], r.dc[1])),
                        __fmul_rn(r.R[3 * i + 2], r.dc[2]));
  r.nrm = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(r.dt[0], r.dt[0]), __fmul_rn(r.dt[1], r.dt[1])), __fmul_rn(r.dt[2], r.dt[2])));
  const bool normalise = a.flags & NNB_NORMALISE;
#pragma unroll
  for (int i = 0; i < 3; ++i) r.d[i] = normalise ? __fdiv_rn(r.dt[i], r.nrm) : r.dt[i];
  if (a.depth) {
    r.depth_raw = __ldg(a.depth + n); r.depth = r.depth_raw;
  } else {  // F.interpolate(depth,(H,W),'nearest')[ray_idx] (network.py:22-24; ATen nearest_idx)
    long long idx = a.ray_idx[n];
    int row = (int)(idx / a.W), col = (int)(idx % a.W);
    float sh = (float)a.h_d / (float)a.H, sw = (float)a.w_d / (float)a.W;
    int sr = min((int)floorf(__fmul_rn((float)row, sh)), a.h_d - 1);
    int sc = min((int)floorf(__fmul_rn((float)col, sw)), a.w_d - 1);
    r.depth_raw = __ldg(a.depth_map + (size_t)sr * a.w_d + sc);
    float sc_ = ld_scalar(a.scale, 1.f), sf_ = ld_scalar(a.shift, 0.f);
    r.depth = (a.flags & NNB_SHIFT_FIRST) ? __fmul_rn(__fadd_rn(r.depth_raw, sf_), sc_)
                                          : __fadd_rn(__fmul_rn(r.depth_raw, sc_), sf_);
  }
  float gd = fabsf(r.depth);
  r.g = normalise ? __fmul_rn(gd, r.nrm) : gd;
  r.mask = isfinite(r.g) && (r.g != 0.f);
  if (a.flags & NNB_NDC) {  // get_ndc_rays_fxfy, near = 1 (rendering.py:170-171)
    r.tau = -(1.f + r.t[2]) / r.d[2];
#pragma unroll
    for (int i = 0; i < 3; ++i) r.o2[i] = __fadd_rn(r.t[i], __fmul_rn(r.tau, r.d[i]));
    float ox = r.o2[0] / r.o2[2], oy = r.o2[1] / r.o2[2];
    r.O[0] = -r.kx * ox; r.O[1] = -r.ky * oy; r.O[2] = 1.f + 2.f / r.o2[2];
    r.Dn[0] = -r.kx * (r.d[0] / r.d[2] - ox); r.Dn[1] = -r.ky * (r.d[1] / r.d[2] - oy); r.Dn[2] = 1.f - r.O[2];
  }
}

// torch.linspace(0,1,S)[i] (symmetric evaluation)
__device__ __forceinline__ float lin01(int i, int S) {
  float step = 1.f / (float)(S - 1);
  return (i < S / 2) ? __fmul_rn(step, (float)i) : __fsub_rn(1.f, __fmul_rn(step, (float)(S - 1 - i)));
}
__device__ __forceinline__ float z_plain(const nnb_render_args& a, int i) {
  float u = lin01(i, a.S);
  if (a.flags & NNB_NDC) return u;  // depth_range literal [0,1] (rendering.py:99)
  return __fadd_rn(__fmul_rn(a.near_, __fsub_rn(1.f, u)), __fmul_rn(a.far_, u));
}
// sample_uniform / sample_ndc z value of sample i of ray n (rendering.py:168-197)
__device__ inline float sample_z(const nnb_render_args& a, int n, int i) {
  float z = z_plain(a, i);
  if (a.noise && !(a.flags & NNB_NDC)) {
    float lo = (i > 0) ? __fmul_rn(0.5f, __fadd_rn(z, z_plain(a, i - 1))) : z;
    float hi = (i < a.S - 1) ? __fmul_rn(0.5f, __fadd_rn(z_plain(a, i + 1), z)) : z;
    z = __fadd_rn(lo, __fmul_rn(__fsub_rn(hi, lo), __ldg(a.noise + (size_t)n * a.S + i)));
  }
  return z;
}
__device__ __forceinline__ void sample_point(const nnb_render_args& a, const Ray& r, float z, float p[3]) {
  if (a.flags & NNB_NDC) {
#pragma unroll
    for (int i = 0; i < 3; ++i) p[i] = __fadd_rn(r.O[i], __fmul_rn(r.Dn[i], z));
  } else {
#pragma unroll
    for (int i = 0; i < 3; ++i) p[i] = __fadd_rn(r.t[i], __fmul_rn(r.d[i], z));
  }
}
__device__ __forceinline__ void view_dir(const nnb_render_args& a, const Ray& r, float v[3]) {
#pragma unroll
  for (int i = 0; i < 3; ++i) v[i] = (a.flags & NNB_USE_DIR) ? -r.d[i] : 1.f;
}

// encode_position (official_nerf.py:99-119): out[0:3]=x, out[3+6l+c]=sin(2^l x_c), out[6+6l+c]=cos(2^l x_c)
template <int L, typename F>
__device__ __forceinline__ void encode(const float x[3], F&& put) {
#pragma unroll
  for (int c = 0; c < 3; ++c) put(c, x[c]);
  float f = 1.f;
#pragma unroll
  for (int l = 0; l < L; ++l) {
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float s, co;
      sincosf(__fmul_rn(f, x[c]), &s, &co);
      put(3 + 6 * l + c, s); put(6 + 6 * l + c, co);
    }
    f *= 2.f;
  }
}
// adjoint of encode: g(k) -> gx
template <int L, typename F>
__device__ __forceinline__ void encode_bwd(const float x[3], F&& get, float gx[3]) {
#pragma unroll
  for (int c = 0; c < 3; ++c) gx[c] = get(c);
  float f = 1.f;
#pragma unroll
  for (int l = 0; l < L; ++l) {
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float s, co;
      sincosf(__fmul_rn(f, x[c]), &s, &co);
      gx[c] += f * (co * get(3 + 6 * l + c) - s * get(6 + 6 * l + c));
    }
    f *= 2.f;
  }
}

__device__ __forceinline__ float softplus_f(float s) { return s > 20.f ? s : log1pf(expf(s)); }
__device__ __forceinline__ float sigmoid_f(float s) { return 1.f / (1.f + expf(-s)); }
// density logit -> MLP output a (alpha if !dist_alpha else sigma) (official_nerf.py:77-83)
__device__ __forceinline__ float density_act(float s, uint32_t flags, float* sigma_out) {
  if (flags & NNB_RAW_DENSITY) { *sigma_out = s; return s; }      // explicit-point queries for infer_occ / gradient(): the logit itself
  float sigma = (flags & NNB_SOFTPLUS) ? softplus_f(s) : fmaxf(s, 0.f);
  *sigma_out = sigma;
  return (flags & NNB_DIST_ALPHA) ? sigma : 1.f - expf(-sigma);
}
// d a / d s
__device__ __forceinline__ float density_act_grad(float s, uint32_t flags) {
  if (flags & NNB_RAW_DENSITY) return 1.f;
  float sigma = (flags & NNB_SOFTPLUS) ? softplus_f(s) : fmaxf(s, 0.f);
  float ds = (flags & NNB_SOFTPLUS) ? (s > 20.f ? 1.f : sigmoid_f(s)) : (s > 0.f ? 1.f : 0.f);
  return (flags & NNB_DIST_ALPHA) ? ds : expf(-sigma) * ds;
}

// warp-level inclusive scans over 32 lanes
__device__ __forceinline__ float warp_incl_prod(float v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { float u = __shfl_up_sync(0xffffffffu, v, o); if (lane >= o) v *= u; }
  return v;
}
__device__ __forceinline__ float warp_incl_sum_rev(float v, int lane) {  // suffix-inclusive sum
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { float u = __shfl_down_sync(0xffffffffu, v, o); if (lane + o < 32) v += u; }
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// per-sample record written by the MLP stage, read by compositing / backward
struct __align__(16) SampleRec { float r, g, b, a; float s, z, pad0, pad1; };

// ---- the arithmetic of composite_fwd (rendering.py:122-158) for the tensor-core frame renderer (tc_frame, frame_finish) ----
// composite_alpha is composite_fwd's own (through sample_alpha).  composite_chunk and composite_tail are the statements of its loop body and
// of its end, in the same order; composite_fwd keeps its own copy of them, because nvcc 12.9 allocates composite_fwd's registers
// differently when it calls them, and its SASS is kept as it was.  tests/test_gpu_render_frame.py checks that the two give the same bits.
// alpha of sample i from its MLP output a_i and depth z_i; z_next() is the depth of sample i + 1, read only with NNB_DIST_ALPHA and i < S - 1
template <typename ZNext>
__device__ __forceinline__ float composite_alpha(const nnb_render_args& a, int i, float a_i, float z_i, ZNext&& z_next) {
  if (!(a.flags & NNB_DIST_ALPHA)) return a_i;
  if (i == a.S - 1) return 1.f;  // alpha[:, -1] = 1 (rendering.py:128)
  float delta = __fsub_rn(z_next(), z_i);
  return 1.f - expf(-a_i * delta);
}
// one 32-sample chunk of a ray, one warp, lane = sample (valid: inside the ray; an invalid lane has alpha = r = g = b = z = 0): carry is
// the transmittance before the chunk on entry and after it on return (the same in every lane); C0..C2, Dist and acc are this lane's
// partial sums of the weighted colour, depth and weight
__device__ __forceinline__ void composite_chunk(float alpha, bool valid, float r, float g, float b, float z, int lane, float& carry, float& C0,
                                                float& C1, float& C2, float& Dist, float& acc) {
  float om = valid ? __fadd_rn(__fsub_rn(1.f, alpha), NNB_EPS) : 1.f;
  float incl = warp_incl_prod(om, lane);
  float excl = __shfl_up_sync(0xffffffffu, incl, 1); if (lane == 0) excl = 1.f;
  float T = carry * excl;
  carry *= __shfl_sync(0xffffffffu, incl, 31);
  float wgt = alpha * T;
  C0 += wgt * r; C1 += wgt * g; C2 += wgt * b; Dist += wgt * z; acc += wgt;
}
// the ray's outputs from the lane partials: warp sums, white background, the EVAL | NORMALISE division, NDC depth_gt, mask
__device__ __forceinline__ void composite_tail(const nnb_render_args& a, int n, const Ray& ray, float C0, float C1, float C2, float Dist, float acc,
                                               int lane) {
  C0 = warp_sum(C0); C1 = warp_sum(C1); C2 = warp_sum(C2); Dist = warp_sum(Dist); acc = warp_sum(acc);
  if (lane == 0) {
    if (a.flags & NNB_WHITE_BG) { float bg = 1.f - acc; C0 += bg; C1 += bg; C2 += bg; }
    float g = ray.g;
    if ((a.flags & NNB_EVAL) && (a.flags & NNB_NORMALISE)) { Dist = Dist / ray.nrm; g = g / ray.nrm; }
    if (a.flags & NNB_NDC) g = 1.f - 1.f / g;
    a.rgb[3 * n] = C0; a.rgb[3 * n + 1] = C1; a.rgb[3 * n + 2] = C2;
    a.depth_pred[n] = Dist; a.depth_gt[n] = g; a.mask[n] = ray.mask ? 1 : 0;
  }
}
