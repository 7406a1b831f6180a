// Reference-image stage of Trainer.compute_loss (model/training.py:280-365): per-point arithmetic of the point-cloud
// (chamfer) and warped-RGB terms, written as __host__ __device__ functions so the SAME code is checked on the CPU against
// oracle.ref_stage (tests/test_host.py builds tools/refstage_host_check.cu with nvcc) and runs inside the kernels of
// nnb_refstage.cu (GPU parity: tests/test_gpu_parity.py::test_native_ref_stage_vs_oracle and the full-loss trainer goldens).
#pragma once
#include <cmath>
#include <cstdint>

#if defined(__CUDACC__)
#define NNB_HD __host__ __device__ __forceinline__
#else
#define NNB_HD inline
#endif

namespace refstage {

struct Geom {            // everything a point needs besides the image / depth pointers
  int H, W, hd, wd, rh, rw;      // full frame, DPT map, low-resolution grid (hd / ratio, wd / ratio)
  float kx, ky, nl;              // K00, K11 (model/common.py:436-457), nearest_limit
  float s_cur, h_cur, s_ref, h_ref;   // effective distortion (scale, shift) of the current / reference view
  float M[12];                   // relative transform [R | t] (row-major 3 x 4), training.py:296-313
  float s2;                      // scale both clouds are divided by (scale_pcs), training.py:357-359
  int is_last, scale_pcs, detach_rgbs_scale, shift_first;
  float w_pc, w_rgb_s;           // loss weights (annealed per epoch, training.py:208-217)
  int with_ssim;                 // warped-RGB term 0.15 L1 + 0.85 SSIM (training.with_ssim, losses.py:150-157)
  int grad_ref;                  // gradients into the reference view too (training.detach_ref_img = False, training.py:288-292)
};
constexpr int kAcc = 17;         // reduced sums: gR (9) | gt (3) | g_s2 | g_scale_cur | g_shift_cur | g_kx | g_ky
constexpr int kAccRef = 2;       // with grad_ref, after those: g_scale_ref (through the reference depth) | g_shift_ref

// F.interpolate(..., mode='nearest') source index: floor(dst * in/out), scale in float32 (training.py:318-319)
NNB_HD int nearest_src(int dst, int n_in, int n_out) {
  int s = (int)floorf((float)dst * ((float)n_in / (float)n_out));
  return s < n_in - 1 ? s : n_in - 1;
}

// one pixel of F.interpolate(img, (rh, rw), mode='bilinear', align_corners=False) for plane `c` of a (3,H,W) image
NNB_HD float lowres_pixel(const float* img, int H, int W, int rh, int rw, int c, int y, int x) {
  float sy = ((float)y + 0.5f) * ((float)H / (float)rh) - 0.5f; if (sy < 0.f) sy = 0.f;
  float sx = ((float)x + 0.5f) * ((float)W / (float)rw) - 0.5f; if (sx < 0.f) sx = 0.f;
  int y0 = (int)floorf(sy); if (y0 > H - 1) y0 = H - 1;
  int x0 = (int)floorf(sx); if (x0 > W - 1) x0 = W - 1;
  const int y1 = y0 + 1 < H ? y0 + 1 : H - 1, x1 = x0 + 1 < W ? x0 + 1 : W - 1;
  const float ly = sy - (float)y0, lx = sx - (float)x0;
  const float* p = img + (size_t)c * H * W;
  const float top = p[(size_t)y0 * W + x0] * (1.f - lx) + p[(size_t)y0 * W + x1] * lx;
  const float bot = p[(size_t)y1 * W + x0] * (1.f - lx) + p[(size_t)y1 * W + x1] * lx;
  return top * (1.f - ly) + bot * ly;
}

// F.grid_sample(lowres(img), xy, bilinear, zeros padding, align_corners=True) for the 3 channels, optionally with the
// derivative of  sum_c g[c] * value[c]  w.r.t. xy
NNB_HD void sample_lowres(const float* img, const Geom& G, float x, float y, float out[3], const float* g, float gxy[2]) {
  const float fx = (x + 1.f) * 0.5f * (float)(G.rw - 1), fy = (y + 1.f) * 0.5f * (float)(G.rh - 1);
  const float x0f = floorf(fx), y0f = floorf(fy);
  const float lx = fx - x0f, ly = fy - y0f;
  const int x0 = (int)x0f, y0 = (int)y0f;
  float dfx = 0.f, dfy = 0.f;
  for (int c = 0; c < 3; ++c) {
    float v[4];
    for (int k = 0; k < 4; ++k) {
      const int yy = y0 + (k >> 1), xx = x0 + (k & 1);
      v[k] = (xx >= 0 && xx < G.rw && yy >= 0 && yy < G.rh) ? lowres_pixel(img, G.H, G.W, G.rh, G.rw, c, yy, xx) : 0.f;
    }
    out[c] = v[0] * (1.f - lx) * (1.f - ly) + v[1] * lx * (1.f - ly) + v[2] * (1.f - lx) * ly + v[3] * lx * ly;
    if (g) {
      dfx += g[c] * ((v[1] - v[0]) * (1.f - ly) + (v[3] - v[2]) * ly);
      dfy += g[c] * ((v[2] - v[0]) * (1.f - lx) + (v[3] - v[1]) * lx);
    }
  }
  if (g) { gxy[0] = dfx * 0.5f * (float)(G.rw - 1); gxy[1] = dfy * 0.5f * (float)(G.rh - 1); }
}

struct Point {           // forward state of one low-resolution pixel
  float px, py;          // arange_pixels coordinates in [-1,1] (model/common.py:13-39)
  float raw_cur;         // raw DPT depth of the current view at this pixel (d scale / d shift need it)
  int live_cur;          // current view's depth not clamped to nearest_limit
  float raw_ref;         // the same for the reference view
  int live_ref;
  float pc1[3], pc2[3];  // back-projected clouds (transform_to_world with the identity pose, model/common.py:112-160)
  float X[3];            // R pc1 + t
  int bad, valid;        // behind-camera fix-up (training.py:334-335), |xy| <= 1 (project_to_cam)
  float Xc[3], xy[2];    // fixed-up point and its projection
};

NNB_HD void point_forward(const Geom& G, const float* dpt_cur, const float* dpt_ref, int i, Point& p) {
  const int row = i / G.rw, col = i - row * G.rw;
  p.px = 2.f * (float)col / (float)(G.rw - 1) - 1.f; p.py = 2.f * (float)row / (float)(G.rh - 1) - 1.f;
  const int sr = nearest_src(row, G.hd, G.rh), sc = nearest_src(col, G.wd, G.rw);
  p.raw_cur = dpt_cur[(size_t)sr * G.wd + sc];
  p.raw_ref = dpt_ref[(size_t)sr * G.wd + sc];
  float dc = G.shift_first ? (p.raw_cur + G.h_cur) * G.s_cur : p.raw_cur * G.s_cur + G.h_cur;           // training.py:241-245
  float dr = G.shift_first ? (p.raw_ref + G.h_ref) * G.s_ref : p.raw_ref * G.s_ref + G.h_ref;           // training.py:283-287
  p.live_cur = dc >= G.nl;
  if (!p.live_cur) dc = G.nl;                                                                          // d[d < nl] = nl (training.py:320-321)
  p.live_ref = !(dr < G.nl);
  if (!p.live_ref) dr = G.nl;
  const float d1 = G.is_last ? dr : dc, d2 = G.is_last ? dc : dr;
  p.pc1[0] = p.px * d1 / G.kx; p.pc1[1] = p.py * d1 / G.ky; p.pc1[2] = -d1;
  p.pc2[0] = p.px * d2 / G.kx; p.pc2[1] = p.py * d2 / G.ky; p.pc2[2] = -d2;
  for (int r = 0; r < 3; ++r) p.X[r] = G.M[4 * r] * p.pc1[0] + G.M[4 * r + 1] * p.pc1[1] + G.M[4 * r + 2] * p.pc1[2] + G.M[4 * r + 3];
  p.bad = (-p.X[2] < G.nl);
  for (int r = 0; r < 3; ++r) p.Xc[r] = p.bad ? G.nl : p.X[r];
  const float z = -p.Xc[2];
  p.xy[0] = G.kx * p.Xc[0] / z; p.xy[1] = G.ky * p.Xc[1] / z;
  p.valid = fmaxf(fabsf(p.xy[0]), fabsf(p.xy[1])) <= 1.f;
}

// warped-RGB residual of a point: diff[c] = rgb_pc1[c] - rgb_pc1_proj[c]  (training.py:326-337)
NNB_HD void point_rgb_diff(const Geom& G, const float* img1, const float* img2, const Point& p, float diff[3]) {
  float a[3], b[3];
  sample_lowres(img1, G, p.px, p.py, a, nullptr, nullptr);
  sample_lowres(img2, G, p.xy[0], p.xy[1], b, nullptr, nullptr);
  for (int c = 0; c < 3; ++c) diff[c] = a[c] - b[c];
}

// the two colours of a point: rgb_pc1 (img1 on the fixed grid) and rgb_pc1_proj (img2 at the projection), training.py:326-333
NNB_HD void point_rgb(const Geom& G, const float* img1, const float* img2, const Point& p, float a[3], float b[3]) {
  sample_lowres(img1, G, p.px, p.py, a, nullptr, nullptr);
  sample_lowres(img2, G, p.xy[0], p.xy[1], b, nullptr, nullptr);
}

// ---- SSIM of the warped-RGB term (class SSIM, losses.py:222-253) ----
// training.py:338-343 hands Loss channel-last (1, rh, rw, 3) maps, so SSIM sees rh channels of (rw x 3) images: its 3x3 windows slide
// over (column, colour channel) inside ONE low-resolution row, with reflection padding of both axes.  x, y: one row, element
// (col, ch) at [3 col + ch]; x = rgb_pc1 (data), y = rgb_pc1_proj (the only input with a gradient).
constexpr float kSsimC1 = 0.01f * 0.01f, kSsimC2 = 0.03f * 0.03f;
NNB_HD int reflect_idx(int i, int n) { return i < 0 ? -i : (i >= n ? 2 * n - 2 - i : i); }

// map value clamp((1 - SSIM) / 2, 0, 1) of the window centred at (col, ch).  With coef: the window's adjoint for a cotangent g on the
// map value, as coefficients of (E[y], E[y^2], E[xy]) divided by 9, so that d map / d y_tap = coef0 + 2 coef1 y_tap + coef2 x_tap
NNB_HD float ssim_window(const float* x, const float* y, int rw, int col, int ch, float g, float* coef) {
  float sx = 0.f, sy = 0.f, sxx = 0.f, syy = 0.f, sxy = 0.f;
  for (int i = -1; i <= 1; ++i) {
    const int cc = reflect_idx(col + i, rw);
    for (int j = -1; j <= 1; ++j) {
      const int k = 3 * cc + reflect_idx(ch + j, 3);
      const float a = x[k], b = y[k];
      sx += a; sy += b; sxx += a * a; syy += b * b; sxy += a * b;
    }
  }
  const float mx = sx / 9.f, my = sy / 9.f;
  const float vx = sxx / 9.f - mx * mx, vy = syy / 9.f - my * my, cxy = sxy / 9.f - mx * my;
  const float a1 = 2.f * mx * my + kSsimC1, a2 = 2.f * cxy + kSsimC2;
  const float b1 = mx * mx + my * my + kSsimC1, b2 = vx + vy + kSsimC2;
  const float S = a1 * a2 / (b1 * b2);
  const float raw = (1.f - S) * 0.5f;
  if (coef) {
    coef[0] = coef[1] = coef[2] = 0.f;
    if (g != 0.f && raw >= 0.f && raw <= 1.f) {               // torch.clamp passes the gradient on [0, 1]
      const float gs = -0.5f * g;
      const float d_my = gs * (2.f * mx * a2 / (b1 * b2) - S * 2.f * my / b1);
      const float d_vy = gs * (-S / b2);
      const float d_cxy = gs * (2.f * a1 / (b1 * b2));
      coef[0] = (d_my - 2.f * my * d_vy - mx * d_cxy) / 9.f; coef[1] = d_vy / 9.f; coef[2] = d_cxy / 9.f;
    }
  }
  return raw < 0.f ? 0.f : (raw > 1.f ? 1.f : raw);
}

// gather form of the SSIM adjoint: d loss / d y at the three channels of column `col`, summed over every window that reads them
// (a reflected tap reads an element twice and counts twice).  coef: one row, 3 coefficients per window centre at [9 col + 3 ch].
NNB_HD void ssim_gather(const float* x, const float* y, const float* coef, int rw, int col, float g[3]) {
  g[0] = g[1] = g[2] = 0.f;
  for (int xc = col - 1; xc <= col + 1; ++xc) {
    if (xc < 0 || xc >= rw) continue;
    const int ncol = (reflect_idx(xc - 1, rw) == col) + (xc == col) + (reflect_idx(xc + 1, rw) == col);
    if (!ncol) continue;
    for (int cc = 0; cc < 3; ++cc) {
      const float* k = coef + 9 * xc + 3 * cc;
      for (int ch = 0; ch < 3; ++ch) {
        const int nch = (reflect_idx(cc - 1, 3) == ch) + (cc == ch) + (reflect_idx(cc + 1, 3) == ch);
        if (nch) g[ch] += (float)(ncol * nch) * (k[0] + 2.f * k[1] * y[3 * col + ch] + k[2] * x[3 * col + ch]);
      }
    }
  }
}

// Adjoint of one point.  gXs, gYs: d(w_pc * chamfer) / d(scaled clouds) of this point (already weighted); inv_nv: w_rgb_s /
// (3 * #valid) or 0; g_rgb2: with G.with_ssim, d(SSIM part) / d rgb_pc1_proj of this point (ssim_gather), else unused.
// Accumulates into acc = { gR (9, row-major), gt (3), g_s2, g_scale_cur, g_shift_cur, g_kx, g_ky } and, with G.grad_ref,
// { g_scale_ref, g_shift_ref } after them (kAcc + kAccRef entries).
NNB_HD void point_backward(const Geom& G, const float* img1, const float* img2, const Point& p, const float gXs[3], const float gYs[3],
                           float inv_nv, const float* g_rgb2, float* acc) {
  float gX[3] = {0.f, 0.f, 0.f}, gXr[3] = {0.f, 0.f, 0.f}, gY[3];
  const float s2 = G.scale_pcs ? G.s2 : 1.f;
  float gs2 = 0.f;
  for (int r = 0; r < 3; ++r) {
    gX[r] = gXs[r] / s2; gY[r] = gYs[r] / s2;
    if (G.scale_pcs) gs2 -= (gXs[r] * (p.X[r] / s2) + gYs[r] * (p.pc2[r] / s2)) / s2;
  }
  if (inv_nv != 0.f && (p.valid || G.with_ssim)) {       // SSIM windows also read the warped colour of invalid points
    float diff[3], gp[3], dummy[3], gxy[2];
    point_rgb_diff(G, img1, img2, p, diff);
    for (int c = 0; c < 3; ++c) gp[c] = (p.valid && fabsf(diff[c]) < 1.f) ? -(diff[c] > 0.f ? 1.f : (diff[c] < 0.f ? -1.f : 0.f)) * inv_nv : 0.f;
    if (G.with_ssim) for (int c = 0; c < 3; ++c) gp[c] = 0.15f * gp[c] + g_rgb2[c];
    sample_lowres(img2, G, p.xy[0], p.xy[1], dummy, gp, gxy);
    {                                                      // xy = (kx Xc_x, ky Xc_y) / z: the projection's own d/dK (also for fixed-up points)
      const float z = -p.Xc[2];
      acc[15] += gxy[0] * p.Xc[0] / z; acc[16] += gxy[1] * p.Xc[1] / z;
    }
    if (!p.bad) {
      const float z = -p.Xc[2];
      gXr[0] = gxy[0] * G.kx / z; gXr[1] = gxy[1] * G.ky / z;
      gXr[2] = (gxy[0] * G.kx * p.Xc[0] + gxy[1] * G.ky * p.Xc[1]) / (z * z);
    }
  }
  float gpc1[3] = {0.f, 0.f, 0.f};
  for (int r = 0; r < 3; ++r) {
    const float gt_r = gX[r] + gXr[r];
    for (int k = 0; k < 3; ++k) acc[3 * r + k] += gt_r * p.pc1[k];
    acc[9 + r] += gt_r;
    const float gp1 = gX[r] + (G.detach_rgbs_scale ? 0.f : gXr[r]);
    for (int k = 0; k < 3; ++k) gpc1[k] += G.M[4 * r + k] * gp1;
  }
  acc[12] += gs2;
  const float* gd_src = G.is_last ? gY : gpc1;          // which cloud was built from the current view's depth
  float gd = gd_src[0] * p.px / G.kx + gd_src[1] * p.py / G.ky - gd_src[2];
  if (!p.live_cur) gd = 0.f;
  if (G.shift_first) { acc[13] += gd * (p.raw_cur + G.h_cur); acc[14] += gd * G.s_cur; }
  else { acc[13] += gd * p.raw_cur; acc[14] += gd; }
  if (G.grad_ref) {                                     // the other cloud was built from the reference view's depth
    const float* gr_src = G.is_last ? gpc1 : gY;
    float gdr = gr_src[0] * p.px / G.kx + gr_src[1] * p.py / G.ky - gr_src[2];
    if (!p.live_ref) gdr = 0.f;
    if (G.shift_first) { acc[kAcc] += gdr * (p.raw_ref + G.h_ref); acc[kAcc + 1] += gdr * G.s_ref; }
    else { acc[kAcc] += gdr * p.raw_ref; acc[kAcc + 1] += gdr; }
  }
  // back-projection (x d / kx, y d / ky, -d): d pc_x / d kx = -pc_x / kx, for both clouds
  acc[15] -= (gpc1[0] * p.pc1[0] + gY[0] * p.pc2[0]) / G.kx;
  acc[16] -= (gpc1[1] * p.pc1[1] + gY[1] * p.pc2[1]) / G.ky;
}

// rigid inverse of a 4x4 pose [R t; 0 1]
NNB_HD void rigid_inverse(const float* A, float* out) {
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) out[4 * r + c] = A[4 * c + r];
    out[4 * r + 3] = -(A[0 * 4 + r] * A[3] + A[1 * 4 + r] * A[7] + A[2 * 4 + r] * A[11]);
  }
  out[12] = 0.f; out[13] = 0.f; out[14] = 0.f; out[15] = 1.f;
}
NNB_HD void mat4_mul(const float* A, const float* B, float* C) {
  for (int r = 0; r < 4; ++r) for (int c = 0; c < 4; ++c) {
    float s = 0.f;
    for (int k = 0; k < 4; ++k) s += A[4 * r + k] * B[4 * k + c];
    C[4 * r + c] = s;
  }
}

// relative transform and scale2 (training.py:296-313): M = inv(c2w_ref) c2w  |  last view: inv(c2w) c2w_ref
NNB_HD void prepare(Geom& G, const float* c2w_cur, const float* c2w_ref) {
  float inv[16], M[16];
  if (!G.is_last) { rigid_inverse(c2w_ref, inv); mat4_mul(inv, c2w_cur, M); G.s2 = G.s_ref; }
  else { rigid_inverse(c2w_cur, inv); mat4_mul(inv, c2w_ref, M); G.s2 = G.s_cur; }
  for (int i = 0; i < 12; ++i) G.M[i] = M[i];
}

// reduced sums acc[15] -> gradients w.r.t. the current view's c2w (16, row-major), effective scale and shift
NNB_HD void finish(const Geom& G, const float* c2w_cur, const float* c2w_ref, const float acc[kAcc], float g_c2w[16], float* g_scale, float* g_shift) {
  float gM[16], inv[16], invT[16], tmp[16], tmp2[16];
  for (int r = 0; r < 3; ++r) { for (int c = 0; c < 3; ++c) gM[4 * r + c] = acc[3 * r + c]; gM[4 * r + 3] = acc[9 + r]; }
  gM[12] = gM[13] = gM[14] = gM[15] = 0.f;
  if (!G.is_last) {
    rigid_inverse(c2w_ref, inv);
    for (int r = 0; r < 4; ++r) for (int c = 0; c < 4; ++c) invT[4 * r + c] = inv[4 * c + r];
    mat4_mul(invT, gM, g_c2w);                                     // M = inv(c2w_ref) c2w
    *g_scale = acc[13];
  } else {
    rigid_inverse(c2w_cur, inv);
    for (int r = 0; r < 4; ++r) for (int c = 0; c < 4; ++c) { invT[4 * r + c] = inv[4 * c + r]; tmp[4 * r + c] = c2w_ref[4 * c + r]; }
    mat4_mul(gM, tmp, tmp2);                                       // d loss / d inv(c2w) = gM c2w_ref^T
    mat4_mul(invT, tmp2, tmp); mat4_mul(tmp, invT, g_c2w);         // d inv(A) = -A^-1 dA A^-1
    for (int i = 0; i < 16; ++i) g_c2w[i] = -g_c2w[i];
    *g_scale = acc[13] + acc[12];                                  // scale2 is the current view's own scale
  }
  *g_shift = acc[14];
}

// with G.grad_ref: reduced sums -> gradients w.r.t. the reference view's c2w (16, row-major), effective scale and shift
NNB_HD void finish_ref(const Geom& G, const float* c2w_cur, const float* c2w_ref, const float* acc, float g_c2w_ref[16], float* g_scale,
                       float* g_shift) {
  float gM[16], inv[16], invT[16], tmp[16], tmp2[16];
  for (int r = 0; r < 3; ++r) { for (int c = 0; c < 3; ++c) gM[4 * r + c] = acc[3 * r + c]; gM[4 * r + 3] = acc[9 + r]; }
  gM[12] = gM[13] = gM[14] = gM[15] = 0.f;
  if (!G.is_last) {
    rigid_inverse(c2w_ref, inv);
    for (int r = 0; r < 4; ++r) for (int c = 0; c < 4; ++c) { invT[4 * r + c] = inv[4 * c + r]; tmp[4 * r + c] = c2w_cur[4 * c + r]; }
    mat4_mul(gM, tmp, tmp2);                                       // d loss / d inv(c2w_ref) = gM c2w^T
    mat4_mul(invT, tmp2, tmp); mat4_mul(tmp, invT, g_c2w_ref);     // d inv(A) = -A^-1 dA A^-1
    for (int i = 0; i < 16; ++i) g_c2w_ref[i] = -g_c2w_ref[i];
    *g_scale = acc[kAcc] + acc[12];                                // scale2 is the reference view's scale
  } else {
    rigid_inverse(c2w_cur, inv);
    for (int r = 0; r < 4; ++r) for (int c = 0; c < 4; ++c) invT[4 * r + c] = inv[4 * c + r];
    mat4_mul(invT, gM, g_c2w_ref);                                 // M = inv(c2w) c2w_ref
    *g_scale = acc[kAcc];
  }
  *g_shift = acc[kAcc + 1];
}

}  // namespace refstage
