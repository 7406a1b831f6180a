// Host-side check of nope_nerf_b200/csrc/nnb_refstage.cuh: runs the SAME __host__ __device__ per-point functions the CUDA
// kernels use, serially on the CPU, so tests/test_host.py can compare them with oracle.ref_stage without a GPU.
//   refstage_host_check <in.bin> <out.bin>
// in : int32[8] {H,W,hd,wd,ratio,is_last,scale_pcs,detach_rgbs_scale}, float32[9] {kx,ky,nl,s_cur,h_cur,s_ref,h_ref,w_pc,w_rgb_s},
//      c2w_cur[16], c2w_ref[16], img_cur[3HW], img_ref[3HW], dpt_cur[hd*wd], dpt_ref[hd*wd]
// out: float32 {loss_pc, loss_rgb_s, g_c2w[16], g_scale, g_shift, g_kx, g_ky} [+ {g_c2w_ref[16], g_scale_ref, g_shift_ref} with flag 16]
// optional 3rd argument '1': shift_first; optional 4th argument: nnb_refstage flags 8 (with_ssim) | 16 (gradients into the reference view)
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "../nope_nerf_b200/csrc/nnb_refstage.cuh"

int main(int argc, char** argv) {
  if (argc < 3) return 2;
  FILE* f = fopen(argv[1], "rb");
  if (!f) return 3;
  int hi[8]; float hf[9], c2w_cur[16], c2w_ref[16];
  if (fread(hi, 4, 8, f) != 8 || fread(hf, 4, 9, f) != 9 || fread(c2w_cur, 4, 16, f) != 16 || fread(c2w_ref, 4, 16, f) != 16) return 4;
  refstage::Geom G{};
  G.H = hi[0]; G.W = hi[1]; G.hd = hi[2]; G.wd = hi[3]; G.rh = hi[2] / hi[4]; G.rw = hi[3] / hi[4];
  G.is_last = hi[5]; G.scale_pcs = hi[6]; G.detach_rgbs_scale = hi[7];
  G.kx = hf[0]; G.ky = hf[1]; G.nl = hf[2]; G.s_cur = hf[3]; G.h_cur = hf[4]; G.s_ref = hf[5]; G.h_ref = hf[6];
  const float w_pc = hf[7], w_rgb_s = hf[8];
  G.shift_first = (argc > 3 && argv[3][0] == '1') ? 1 : 0; G.w_pc = w_pc; G.w_rgb_s = w_rgb_s;
  const int xflags = argc > 4 ? atoi(argv[4]) : 0;
  G.with_ssim = (xflags & 8) ? 1 : 0; G.grad_ref = (xflags & 16) ? 1 : 0;
  std::vector<float> img_cur(3 * (size_t)G.H * G.W), img_ref(img_cur.size()), dpt_cur((size_t)G.hd * G.wd), dpt_ref(dpt_cur.size());
  if (fread(img_cur.data(), 4, img_cur.size(), f) != img_cur.size() || fread(img_ref.data(), 4, img_ref.size(), f) != img_ref.size() ||
      fread(dpt_cur.data(), 4, dpt_cur.size(), f) != dpt_cur.size() || fread(dpt_ref.data(), 4, dpt_ref.size(), f) != dpt_ref.size()) return 5;
  fclose(f);
  const float* img1 = G.is_last ? img_ref.data() : img_cur.data();
  const float* img2 = G.is_last ? img_cur.data() : img_ref.data();
  refstage::prepare(G, c2w_cur, c2w_ref);
  const int P = G.rh * G.rw;
  const float s2 = G.scale_pcs ? G.s2 : 1.f;
  std::vector<refstage::Point> pts(P);
  std::vector<float> Xs(3 * P), Ys(3 * P), gXs(3 * P, 0.f), gYs(3 * P, 0.f);
  float sum_abs = 0.f; int nvalid = 0;
  std::vector<float> rgb1(3 * P), rgb2(3 * P), coef(9 * (size_t)P, 0.f);
  for (int i = 0; i < P; ++i) {
    refstage::point_forward(G, dpt_cur.data(), dpt_ref.data(), i, pts[i]);
    for (int r = 0; r < 3; ++r) { Xs[3 * i + r] = pts[i].X[r] / s2; Ys[3 * i + r] = pts[i].pc2[r] / s2; }
    if (G.with_ssim) refstage::point_rgb(G, img1, img2, pts[i], &rgb1[3 * i], &rgb2[3 * i]);
    if (w_rgb_s != 0.f && pts[i].valid) {
      float diff[3];
      refstage::point_rgb_diff(G, img1, img2, pts[i], diff);
      for (int c = 0; c < 3; ++c) { float a = fabsf(diff[c]); sum_abs += a > 1.f ? 1.f : a; }
      ++nvalid;
    }
  }
  // dense chamfer (model/losses.py:114-148), the nearest neighbours and terms of nn_search_k / chamfer_pairs_k
  float loss_pc = 0.f;
  if (w_pc != 0.f) {
    for (int dir = 0; dir < 2; ++dir) {
      const std::vector<float>& A = dir ? Ys : Xs; const std::vector<float>& B = dir ? Xs : Ys;
      std::vector<float>& gA = dir ? gYs : gXs; std::vector<float>& gB = dir ? gXs : gYs;
      float tot = 0.f;
      for (int i = 0; i < P; ++i) {
        float best = INFINITY; int bi = 0;
        for (int q = 0; q < P; ++q) {
          const float dx = A[3 * i] - B[3 * q], dy = A[3 * i + 1] - B[3 * q + 1], dz = A[3 * i + 2] - B[3 * q + 2];
          const float d = sqrtf(dx * dx + dy * dy + dz * dz);
          if (d < best) { best = d; bi = q; }
        }
        tot += best;
        if (best > 0.f) for (int r = 0; r < 3; ++r) {
          const float g = w_pc * (A[3 * i + r] - B[3 * bi + r]) / (best * (float)P);
          gA[3 * i + r] += g; gB[3 * bi + r] -= g;
        }
      }
      loss_pc += tot / (float)P;
    }
  }
  const float inv_nv = (w_rgb_s != 0.f && nvalid > 0) ? w_rgb_s / (3.f * (float)nvalid) : 0.f;
  float sum_ssim = 0.f;
  if (G.with_ssim) {                     // SSIM map over every row (sums over valid centres) and the per-window adjoint coefficients
    for (int i = 0; i < P; ++i) {
      const int row = i / G.rw, col = i - row * G.rw;
      const size_t ro = (size_t)row * 3 * G.rw;
      for (int c = 0; c < 3; ++c) {
        const float g = pts[i].valid ? 0.85f * inv_nv : 0.f;
        const float m = refstage::ssim_window(&rgb1[ro], &rgb2[ro], G.rw, col, c, g, &coef[9 * (size_t)i + 3 * c]);
        if (pts[i].valid) sum_ssim += m;
      }
    }
  }
  float acc[refstage::kAcc + refstage::kAccRef] = {0};
  for (int i = 0; i < P; ++i) {
    float g2[3] = {0.f, 0.f, 0.f};
    if (G.with_ssim) {
      const int row = i / G.rw, col = i - row * G.rw;
      const size_t ro = (size_t)row * 3 * G.rw;
      refstage::ssim_gather(&rgb1[ro], &rgb2[ro], &coef[3 * ro], G.rw, col, g2);
    }
    refstage::point_backward(G, img1, img2, pts[i], &gXs[3 * i], &gYs[3 * i], inv_nv, g2, acc);
  }
  float out[40];
  out[0] = loss_pc;
  out[1] = nvalid > 0 ? (G.with_ssim ? (0.15f * sum_abs + 0.85f * sum_ssim) : sum_abs) / (3.f * (float)nvalid) : 0.f;
  refstage::finish(G, c2w_cur, c2w_ref, acc, out + 2, out + 18, out + 19);
  f = fopen(argv[2], "wb");
  if (!f) return 6;
  out[20] = acc[15]; out[21] = acc[16];
  if (G.grad_ref) refstage::finish_ref(G, c2w_cur, c2w_ref, acc, out + 22, out + 38, out + 39);
  fwrite(out, 4, G.grad_ref ? 40 : 22, f); fclose(f);
  return 0;
}
