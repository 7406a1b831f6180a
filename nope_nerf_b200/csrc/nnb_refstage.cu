// Reference-image stage of Trainer.compute_loss (model/training.py:280-365) as four small kernels around the dense chamfer:
//   prep (relative pose, scale2)  ->  points forward (clouds, warped-RGB residual)  ->  nnb chamfer (nearest neighbours, d/dX, d/dY)
//   ->  points backward (one row of partial sums per block)  ->  finish (the rows summed in a fixed order; gradients of the current
//   view's pose matrix and distortion).  No float atomics: the same inputs give the same bits on every run.
// With SSIM (flag 8) the points forward also stores both colours of every point and one more kernel (rs_ssim_k) evaluates the SSIM
// windows before the chamfer; the points backward gathers the windows' adjoint per point.  With flag 16 the same reduction carries
// two more sums and finish also writes the reference view's gradients.  With both flags clear the launches are those of before.
// The per-point arithmetic lives in nnb_refstage.cuh and is checked on the CPU against oracle.ref_stage; the kernels are
// checked on hardware by tests/test_gpu_parity.py (test_native_ref_stage_vs_oracle, full-loss trainer goldens).
#include "nnb_common.cuh"
#include "nnb_refstage.cuh"
#include "../../include/nope_nerf_b200.h"

cudaError_t launch_chamfer_dev(const float*, int, const float*, int, void*, float*, const float*, float*, float*, cudaStream_t);
size_t chamfer_workspace_bytes(int P, int Q);

namespace {
using refstage::Geom;
using refstage::Point;
using refstage::kAcc;
using refstage::kAccRef;

struct Scratch {       // device-resident state of one call (512 B at the start of the workspace)
  Geom G;
  const float* img1; const float* img2;    // the two frames in the order of the warp (training.py:296-313)
  float loss_pc, w_pc;                     // w_pc sits next to loss_pc: the chamfer reads its weight from device memory
};
static_assert(sizeof(Scratch) <= 512, "scratch layout");

// Every sum over the points is reproducible bit for bit: each block stores its K partials in its own row of a [blocks][K] array, and
// the consumers add the rows up in one fixed order (warp_total).
constexpr int kFwdK = 2;                   // sum_abs, nvalid                                  (rs_points_fwd_k)
constexpr int kSsimK = 1;                  // SSIM map over valid points and channels           (rs_ssim_k, flag 8)
constexpr int kBwdK = kAcc + kAccRef;      // row stride of the adjoint sums                   (rs_points_bwd_k)
struct Partials { float* fwd; float* ssim; float* bwd; int nb; };

// Everything that changes from step to step may come from DEVICE memory (img_pp, cam, cam_idx, weights), so a captured CUDA
// graph of the full-loss training step can be replayed for every frame pair (model/training.py: _GraphStep).
__global__ void rs_prep_k(Scratch* S, Geom G0, nnb_refstage_args a) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  Geom G = G0;
  G.s_cur = a.dist_cur[0]; G.h_cur = a.dist_cur[1]; G.s_ref = a.dist_ref[0]; G.h_ref = a.dist_ref[1];
  if (a.cam) { G.kx = a.cam[0]; G.ky = a.cam[5]; }
  if (a.cam_idx_dev) G.is_last = (*a.cam_idx_dev == a.num_cams - 1) ? 1 : 0;
  if (a.weights_dev) { G.w_pc = a.weights_dev[0]; G.w_rgb_s = a.weights_dev[1]; }
  refstage::prepare(G, a.c2w_cur, a.c2w_ref);
  const float* cur = a.img_pp ? a.img_pp[0] : a.img_cur;
  const float* ref = a.img_pp ? a.img_pp[1] : a.img_ref;
  S->G = G; S->img1 = G.is_last ? ref : cur; S->img2 = G.is_last ? cur : ref;
  S->loss_pc = 0.f; S->w_pc = G.w_pc;
}

template <int K>
__device__ void block_store(float (&v)[K], float* row) {   // sum v[k] over the block into this block's row (row[k], k < K)
  __shared__ float sh[K][32];
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = blockDim.x >> 5;
#pragma unroll
  for (int k = 0; k < K; ++k) { const float s = warp_sum(v[k]); if (l == 0) sh[k][w] = s; }
  __syncthreads();
  if (w == 0) {
#pragma unroll
    for (int k = 0; k < K; ++k) { float s = warp_sum(l < nw ? sh[k][l] : 0.f); if (l == 0) row[k] = s; }
  }
}

// column k of a [nb][K] partial array, summed by one full warp in a fixed order (lane l adds rows l, l + 32, ... in turn, then a fixed
// butterfly); every lane returns the same bits
__device__ __forceinline__ float warp_total(const float* part, int nb, int K, int k) {
  float s = 0.f;
  for (int b = threadIdx.x & 31; b < nb; b += 32) s += part[(size_t)b * K + k];
  return warp_sum(s);
}

// the same for a whole block: warp 0 sums, every thread gets the value
__device__ float block_total(const float* part, int nb, int K, int k) {
  __shared__ float t;
  if (threadIdx.x < 32) { const float s = warp_total(part, nb, K, k); if (threadIdx.x == 0) t = s; }
  __syncthreads();
  return t;
}

// rgb1 / rgb2 / vmask: with SSIM, both colours and the validity of EVERY point (the SSIM windows also read invalid points)
__global__ void rs_points_fwd_k(Scratch* S, const float* dpt_cur, const float* dpt_ref, float* Xs, float* Ys, float* rgb1, float* rgb2,
                                float* vmask, Partials pt) {
  const Geom& G = S->G;
  const int P = G.rh * G.rw, i = blockIdx.x * blockDim.x + threadIdx.x;
  float part[2] = {0.f, 0.f};
  if (i < P) {
    Point p;
    refstage::point_forward(G, dpt_cur, dpt_ref, i, p);
    const float s2 = G.scale_pcs ? G.s2 : 1.f;
#pragma unroll
    for (int r = 0; r < 3; ++r) { Xs[3 * i + r] = p.X[r] / s2; Ys[3 * i + r] = p.pc2[r] / s2; }
    if (G.with_ssim) {
      float a[3], b[3];
      refstage::point_rgb(G, S->img1, S->img2, p, a, b);
#pragma unroll
      for (int c = 0; c < 3; ++c) { rgb1[3 * i + c] = a[c]; rgb2[3 * i + c] = b[c]; }
      vmask[i] = p.valid ? 1.f : 0.f;
      if (G.w_rgb_s != 0.f && p.valid) {
#pragma unroll
        for (int c = 0; c < 3; ++c) part[0] += fminf(fabsf(a[c] - b[c]), 1.f);
        part[1] = 1.f;
      }
    } else if (G.w_rgb_s != 0.f && p.valid) {
      float diff[3];
      refstage::point_rgb_diff(G, S->img1, S->img2, p, diff);
#pragma unroll
      for (int c = 0; c < 3; ++c) part[0] += fminf(fabsf(diff[c]), 1.f);
      part[1] = 1.f;
    }
  }
  block_store<kFwdK>(part, pt.fwd + (size_t)blockIdx.x * kFwdK);
}

// SSIM map of every valid point's three windows (summed into the ssim partials) and the adjoint coefficients of every window
// (coef [P][3][3]); a window centred on an invalid point has no loss and zero coefficients
__global__ void rs_ssim_k(Scratch* S, const float* rgb1, const float* rgb2, const float* vmask, float* coef, Partials pt) {
  const Geom& G = S->G;
  const int P = G.rh * G.rw, i = blockIdx.x * blockDim.x + threadIdx.x;
  const float nvalid = block_total(pt.fwd, pt.nb, kFwdK, 1);
  float part[1] = {0.f};
  if (i < P) {
    const int row = i / G.rw, col = i - row * G.rw;
    const size_t ro = (size_t)row * 3 * G.rw;
    const bool valid = vmask[i] != 0.f;
    const float g = (valid && G.w_rgb_s != 0.f && nvalid > 0.f) ? 0.85f * (G.w_rgb_s / (3.f * nvalid)) : 0.f;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float m = refstage::ssim_window(rgb1 + ro, rgb2 + ro, G.rw, col, c, g, coef + 9 * (size_t)i + 3 * c);
      if (valid) part[0] += m;
    }
  }
  block_store<kSsimK>(part, pt.ssim + (size_t)blockIdx.x * kSsimK);
}

// NA = kAcc, or kAcc + kAccRef with gradients into the reference view.  With SSIM, each point first gathers d loss / d rgb_pc1_proj
// from the windows that read it (rgb1 / rgb2 / coef non-null).
template <int NA>
__global__ void rs_points_bwd_k(Scratch* S, const float* dpt_cur, const float* dpt_ref, const float* gXs, const float* gYs, const float* rgb1,
                                const float* rgb2, const float* coef, Partials pt) {
  const Geom& G = S->G;
  const int P = G.rh * G.rw, i = blockIdx.x * blockDim.x + threadIdx.x;
  const float nvalid = block_total(pt.fwd, pt.nb, kFwdK, 1);
  float acc[NA];
#pragma unroll
  for (int k = 0; k < NA; ++k) acc[k] = 0.f;
  if (i < P) {
    Point p;
    refstage::point_forward(G, dpt_cur, dpt_ref, i, p);
    const float inv_nv = (G.w_rgb_s != 0.f && nvalid > 0.f) ? G.w_rgb_s / (3.f * nvalid) : 0.f;
    float g2[3] = {0.f, 0.f, 0.f};
    if (G.with_ssim) {
      const int row = i / G.rw, col = i - row * G.rw;
      const size_t ro = (size_t)row * 3 * G.rw;
      refstage::ssim_gather(rgb1 + ro, rgb2 + ro, coef + 3 * ro, G.rw, col, g2);
    }
    refstage::point_backward(G, S->img1, S->img2, p, gXs + 3 * i, gYs + 3 * i, inv_nv, g2, acc);
  }
  block_store<NA>(acc, pt.bwd + (size_t)blockIdx.x * kBwdK);
}

// one warp per sum (the adjoint sums, then sum_abs, nvalid, sum_ssim) adds up its column of partials, then thread 0 finishes
constexpr int kFinishWarps = kBwdK + 3;
__global__ void __launch_bounds__(32 * kFinishWarps) rs_finish_k(const Scratch* S, nnb_refstage_args a, Partials pt) {
  __shared__ float tot[kFinishWarps];
  const int w = threadIdx.x >> 5;
  const int na = S->G.grad_ref ? kAcc + kAccRef : kAcc;
  float s = 0.f;
  if (w < kBwdK) { if (w < na) s = warp_total(pt.bwd, pt.nb, kBwdK, w); }
  else if (w < kBwdK + 2) s = warp_total(pt.fwd, pt.nb, kFwdK, w - kBwdK);
  else if (S->G.with_ssim) s = warp_total(pt.ssim, pt.nb, kSsimK, 0);
  if ((threadIdx.x & 31) == 0) tot[w] = s;
  __syncthreads();
  if (threadIdx.x != 0) return;
  float acc[kAcc + kAccRef];
#pragma unroll
  for (int k = 0; k < kAcc + kAccRef; ++k) acc[k] = tot[k];
  const float sum_abs = tot[kBwdK], nvalid = tot[kBwdK + 1], sum_ssim = tot[kBwdK + 2];
  float g[16], gs, gh;
  refstage::finish(S->G, a.c2w_cur, a.c2w_ref, acc, g, &gs, &gh);
  const float l_pc = S->G.w_pc != 0.f ? S->loss_pc : 0.f;
  const float l_rgbs = nvalid > 0.f ? (S->G.with_ssim ? 0.15f * sum_abs + 0.85f * sum_ssim : sum_abs) / (3.f * nvalid) : 0.f;
  a.losses[0] = l_pc; a.losses[1] = l_rgbs;
  if (a.loss_total) atomicAdd(a.loss_total, S->G.w_pc * l_pc + S->G.w_rgb_s * l_rgbs);
  const float gsc = a.grad_scale == 0.f ? 1.f : a.grad_scale;
  // One add per output element, from this one thread.  They are atomic so that a caller may run the stage beside other work that
  // adds into the same buffers; the sum is then still correct, and it is reproducible bit for bit whenever that other work is
  // ordered before or after this kernel (the Trainer joins the render backward first: model/training.py, _GraphStep.body_a).
  if (a.g_c2w) for (int i = 0; i < 12; ++i) atomicAdd(a.g_c2w + i, gsc * g[i]);
  if (a.g_dist) { atomicAdd(a.g_dist, gsc * gs); atomicAdd(a.g_dist + 1, gsc * gh); }
  if (a.g_kxy) { atomicAdd(a.g_kxy, gsc * acc[15]); atomicAdd(a.g_kxy + 1, gsc * acc[16]); }
  if (S->G.grad_ref) {
    float gr[16], grs, grh;
    refstage::finish_ref(S->G, a.c2w_cur, a.c2w_ref, acc, gr, &grs, &grh);
    for (int i = 0; i < 12; ++i) atomicAdd(a.g_c2w_ref + i, gsc * gr[i]);
    atomicAdd(a.g_dist_ref, gsc * grs); atomicAdd(a.g_dist_ref + 1, gsc * grh);
  }
}

}  // namespace

// Workspace: Scratch (512 B) | Xs, Ys, gXs, gYs [P][3] | partials fwd [nb][2], ssim [nb][1], bwd [nb][19] | the chamfer's scratch
// (256-aligned) | with flag 8 (SSIM): rgb1 [P][3], rgb2 [P][3], vmask [P], window coefficients [P][3][3]
constexpr int kRsThreads = 128;
static size_t rs_chamfer_offset(size_t P) {
  const size_t nb = (P + kRsThreads - 1) / kRsThreads;
  return (512 + P * 4 * 3 * sizeof(float) + nb * (kFwdK + kSsimK + kBwdK) * sizeof(float) + 255) & ~(size_t)255;
}

size_t refstage_workspace_bytes(int hd, int wd, int ratio) {
  const size_t P = (size_t)(hd / ratio) * (size_t)(wd / ratio);
  const size_t ch = chamfer_workspace_bytes((int)P, (int)P);
  return ch == 0 ? 0 : rs_chamfer_offset(P) + ch;
}

size_t refstage_workspace_bytes_flags(int hd, int wd, int ratio, unsigned flags) {
  const size_t P = (size_t)(hd / ratio) * (size_t)(wd / ratio);
  const size_t b = refstage_workspace_bytes(hd, wd, ratio);
  return b == 0 ? 0 : b + ((flags & 8u) ? P * (3 + 3 + 1 + 9) * sizeof(float) : 0);
}

cudaError_t launch_refstage(const nnb_refstage_args& a, cudaStream_t st) {
  Geom G0{};
  G0.H = a.H; G0.W = a.W; G0.hd = a.h_d; G0.wd = a.w_d; G0.rh = a.h_d / a.pc_ratio; G0.rw = a.w_d / a.pc_ratio;
  G0.kx = a.kx; G0.ky = a.ky; G0.nl = a.nearest_limit; G0.w_pc = a.w_pc; G0.w_rgb_s = a.w_rgb_s;
  G0.is_last = a.is_last ? 1 : 0; G0.scale_pcs = (a.flags & 1u) ? 1 : 0; G0.detach_rgbs_scale = (a.flags & 2u) ? 1 : 0;
  G0.shift_first = (a.flags & 4u) ? 1 : 0; G0.with_ssim = (a.flags & 8u) ? 1 : 0; G0.grad_ref = (a.flags & 16u) ? 1 : 0;
  const int P = G0.rh * G0.rw;
  char* base = static_cast<char*>(a.workspace);
  Scratch* S = reinterpret_cast<Scratch*>(base);
  float* Xs = reinterpret_cast<float*>(base + 512); float* Ys = Xs + 3 * (size_t)P;
  float* gXs = Ys + 3 * (size_t)P; float* gYs = gXs + 3 * (size_t)P;
  const int nb = (P + kRsThreads - 1) / kRsThreads;
  Partials pt;
  pt.nb = nb; pt.fwd = gYs + 3 * (size_t)P; pt.ssim = pt.fwd + (size_t)nb * kFwdK; pt.bwd = pt.ssim + (size_t)nb * kSsimK;
  const size_t ch_bytes = chamfer_workspace_bytes(P, P);
  if (ch_bytes == 0) return cudaErrorInvalidValue;
  void* ch_ws = base + rs_chamfer_offset((size_t)P);
  float* rgb1 = nullptr; float* rgb2 = nullptr; float* vmask = nullptr; float* coef = nullptr;
  if (G0.with_ssim) {
    rgb1 = reinterpret_cast<float*>(static_cast<char*>(ch_ws) + ch_bytes); rgb2 = rgb1 + 3 * (size_t)P; vmask = rgb2 + 3 * (size_t)P;
    coef = vmask + P;
  }
  rs_prep_k<<<1, 32, 0, st>>>(S, G0, a);
  rs_points_fwd_k<<<nb, kRsThreads, 0, st>>>(S, a.dpt_cur, a.dpt_ref, Xs, Ys, rgb1, rgb2, vmask, pt);
  if (G0.with_ssim) rs_ssim_k<<<nb, kRsThreads, 0, st>>>(S, rgb1, rgb2, vmask, coef, pt);
  cudaError_t e = cudaMemsetAsync(gXs, 0, sizeof(float) * 6 * (size_t)P, st);
  if (e != cudaSuccess) return e;
  if (a.w_pc != 0.f || a.weights_dev) {      // device-resident weights: the term is always evaluated (a weight of 0 zeroes its gradients)
    e = launch_chamfer_dev(Xs, P, Ys, P, ch_ws, &S->loss_pc, &S->w_pc, gXs, gYs, st);
    if (e != cudaSuccess) return e;
  }
  if (G0.grad_ref) rs_points_bwd_k<kAcc + kAccRef><<<nb, kRsThreads, 0, st>>>(S, a.dpt_cur, a.dpt_ref, gXs, gYs, rgb1, rgb2, coef, pt);
  else rs_points_bwd_k<kAcc><<<nb, kRsThreads, 0, st>>>(S, a.dpt_cur, a.dpt_ref, gXs, gYs, rgb1, rgb2, coef, pt);
  rs_finish_k<<<1, 32 * kFinishWarps, 0, st>>>(S, a, pt);
  return cudaGetLastError();
}
