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

// ---- the per-ray geometry adjoint (SURVEY.md A.6) of ray_bwd, from the ray's sums over its samples of the point adjoint (so), the
// depth-weighted point adjoint (sd) and the view-direction adjoint (sv): red[0..8] d R, [9..11] d t, [12,13] d kx, ky, [14,15] d scale, shift
// -> rayred[n][16], and b.g_depth[n]: the statements of ray_bwd's lane-0 block, for the differentiable frame (frame_ray_finish,
// nnb_frame.cuh).  ray_bwd keeps its own copy: nvcc 12.9 schedules ray_bwd differently when it calls this, and its SASS is kept as it was.
__device__ __forceinline__ void ray_adjoint(const nnb_render_bwd_args& b, int n, const Ray& r, const float so[3], const float sd[3],
                                            const float sv[3], float* rayred) {
  const nnb_render_args& a = b.fwd;
  float red[16];
#pragma unroll
  for (int k = 0; k < 16; ++k) red[k] = 0.f;
  const bool normalise = a.flags & NNB_NORMALISE, ev = (a.flags & NNB_EVAL) && normalise;
  float g_nrm = 0.f;
  float gDo = b.g_depth_pred ? __ldg(b.g_depth_pred + n) : 0.f;
  float g_g = b.g_depth_gt ? __ldg(b.g_depth_gt + n) : 0.f;
  float gcur = ev ? r.g / r.nrm : r.g;
  if (a.flags & NNB_NDC) g_g = g_g / (gcur * gcur);
  if (ev) {
    float Dist = a.depth_pred[n] * r.nrm;  // stored output is Dist / nrm
    g_nrm -= gDo * Dist / (r.nrm * r.nrm);
    g_nrm -= g_g * r.g / (r.nrm * r.nrm);
    g_g = g_g / r.nrm;
  }
  float g_gdepth;
  if (normalise) { g_gdepth = g_g * r.nrm; g_nrm += g_g * fabsf(r.depth); } else g_gdepth = g_g;
  float g_depth = g_gdepth * (r.depth > 0.f ? 1.f : (r.depth < 0.f ? -1.f : 0.f));
  float g_o[3], g_d[3], g_kx = 0.f, g_ky = 0.f;
  if (a.flags & NNB_NDC) {
    const float* d = r.d; const float* o2 = r.o2;
    float ox = o2[0] / o2[2], oy = o2[1] / o2[2];
    float gO[3] = {so[0], so[1], so[2]}, gDn[3] = {sd[0], sd[1], sd[2]};
    float g_Oz = gO[2] - gDn[2];
    float g_ox = -r.kx * gO[0] + r.kx * gDn[0];
    float g_oy = -r.ky * gO[1] + r.ky * gDn[1];
    g_d[0] = -r.kx * gDn[0] / d[2];
    g_d[1] = -r.ky * gDn[1] / d[2];
    g_d[2] = (r.kx * gDn[0] * d[0] + r.ky * gDn[1] * d[1]) / (d[2] * d[2]);
    g_kx = -ox * gO[0] - (d[0] / d[2] - ox) * gDn[0];
    g_ky = -oy * gO[1] - (d[1] / d[2] - oy) * gDn[1];
    float g_o2[3];
    g_o2[0] = g_ox / o2[2]; g_o2[1] = g_oy / o2[2];
    g_o2[2] = -(g_ox * ox + g_oy * oy) / o2[2] - 2.f * g_Oz / (o2[2] * o2[2]);
    float g_tau = g_o2[0] * d[0] + g_o2[1] * d[1] + g_o2[2] * d[2];
#pragma unroll
    for (int c = 0; c < 3; ++c) { g_o[c] = g_o2[c]; g_d[c] += g_o2[c] * r.tau; }
    g_o[2] += -g_tau / d[2];
    g_d[2] += g_tau * (1.f + r.t[2]) / (d[2] * d[2]);
  } else {
#pragma unroll
    for (int c = 0; c < 3; ++c) { g_o[c] = so[c]; g_d[c] = sd[c]; }
  }
  if (a.flags & NNB_USE_DIR) {
#pragma unroll
    for (int c = 0; c < 3; ++c) g_d[c] -= sv[c];
  }
  float g_dt[3];
  if (normalise) {
    float dot = r.d[0] * g_d[0] + r.d[1] * g_d[1] + r.d[2] * g_d[2];
#pragma unroll
    for (int c = 0; c < 3; ++c) g_dt[c] = (g_d[c] - r.d[c] * dot) / r.nrm;
  } else {
#pragma unroll
    for (int c = 0; c < 3; ++c) g_dt[c] = g_d[c];
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) g_dt[c] += (g_nrm / r.nrm) * r.dt[c];
  // g_R[a][b] = g_dt[a] * dc[b]; g_t = g_o
#pragma unroll
  for (int i = 0; i < 3; ++i) {
#pragma unroll
    for (int j = 0; j < 3; ++j) red[3 * i + j] = g_dt[i] * r.dc[j];
    red[9 + i] = g_o[i];
  }
  float g_dc0 = g_dt[0] * r.R[0] + g_dt[1] * r.R[3] + g_dt[2] * r.R[6];
  float g_dc1 = g_dt[0] * r.R[1] + g_dt[1] * r.R[4] + g_dt[2] * r.R[7];
  g_kx += g_dc0 * (-r.x / (r.kx * r.kx));
  g_ky += g_dc1 * (-r.y / (r.ky * r.ky));
  red[12] = g_kx; red[13] = g_ky;
  if (b.g_depth) b.g_depth[n] = g_depth;
  if (!a.depth) {  // depth = raw*scale + shift  |  (raw + shift)*scale
    float sc = ld_scalar(a.scale, 1.f), sf = ld_scalar(a.shift, 0.f);
    if (a.flags & NNB_SHIFT_FIRST) { red[14] = g_depth * (r.depth_raw + sf); red[15] = g_depth * sc; }
    else { red[14] = g_depth * r.depth_raw; red[15] = g_depth; }
  }
#pragma unroll
  for (int k = 0; k < 16; ++k) rayred[(size_t)n * 16 + k] = red[k];
}

// ---- the compositing adjoint of one 32-sample chunk of a ray (the differentiable frame, nnb_render_frame_bwd): the statements of
// composite_bwd's reverse sweep for chunk c, in the same order, from the transmittance `carry` into the chunk instead of composite_bwd's
// forward sweep (the frame's forward stores it with the bits that sweep has).  composite_bwd keeps its own copy so that its SASS is kept as
// it was.  carry_s is the suffix sum of w gw over the later chunks on entry, and includes this chunk on return; it is carried from chunk to
// chunk and never formed as total - prefix (DESIGN.md §4).  df = d alpha / d a.  Returns (w gC0, w gC1, w gC2, d L / d a) of the lane's
// sample, zeros for an invalid lane.
// FUSED: d L / d alpha = T gw - suffix / om as one fma, which is what nvcc 12.9 makes of composite_bwd's statement; the exact engine's frame
// (FUSED = true) spells it so that at S <= 32 its gradients are nnb_render_bwd's bits.  FUSED = false is the statement as written, which
// this copy compiles to a product and a subtraction: the tensor-core frame's form, kept as it was.
template <bool FUSED = false>
__device__ __forceinline__ float4 composite_chunk_bwd(float alpha, bool valid, float r, float g, float b, float z, float df, int lane, float carry,
                                                      float gC0, float gC1, float gC2, float gD, float gsum, float& carry_s) {
  const float om = valid ? __fadd_rn(__fsub_rn(1.f, alpha), NNB_EPS) : 1.f;
  const float incl_p = warp_incl_prod(om, lane);
  float excl_p = __shfl_up_sync(0xffffffffu, incl_p, 1); if (lane == 0) excl_p = 1.f;
  const float T = carry * excl_p;
  const float w = alpha * T;
  const float gw = fmaf(gD, z, fmaf(gC2, b, fmaf(gC1, g, gC0 * r))) - gsum;
  const float wg = valid ? w * gw : 0.f;
  const float incl = warp_incl_sum_rev(wg, lane);
  float excl = __shfl_down_sync(0xffffffffu, incl, 1); if (lane == 31) excl = 0.f;
  const float suffix = excl + carry_s;
  carry_s += __shfl_sync(0xffffffffu, incl, 0);
  const float g_alpha = FUSED ? fmaf(T, gw, -(suffix / om)) : T * gw - suffix / om;
  return valid ? make_float4(w * gC0, w * gC1, w * gC2, g_alpha * df) : make_float4(0.f, 0.f, 0.f, 0.f);
}
