// Exact-fp32 SIMT engine (NNB_ENGINE_SIMT): the reference arithmetic (nn.Linear = fp32 FMA)
// with the whole field evaluated tile-by-tile out of shared memory.  It is the bit-faithful
// engine used for small batches and as the on-device cross-check of the tensor-core engine.
// Every MLP kernel is instantiated once per supported hidden width D (64 | 128 | 256) and dispatched on nnb_render_args.hidden_dim.
//   F1 simt_mlp_fwd     : ray-gen + sampling + encoding + 8xD MLP + heads  (64 samples / CTA)
//   F2 composite_fwd    : alpha compositing, one warp per ray (shared with the TC engine)
//   B1 composite_bwd    : compositing adjoint -> per-sample (g_rgb, g_a)
//   B2 simt_mlp_dgrad   : data-gradient chain through the MLP, emits dY per layer
//   B3 simt_wgrad       : dW = dY^T X as split-M tiles, one partial per split, summed in order by wgrad_reduce
//      head_wgrad       : the same arithmetic for the TC engine's narrow head jobs, streamed at memory speed
//   B4 ray_bwd          : per-ray geometry adjoint -> d c2w, d K, d depth, d scale/shift
#include "nnb_tc_common.cuh"   // mbarrier / bulk-copy wrappers (head_wgrad)
#include "nnb_march.cuh"
#include "nnb_frame.cuh"

void nnb_prof_mark(cudaStream_t st);

namespace {

constexpr int TM = 64;         // samples per CTA tile
template <int D> constexpr int ldb() { return D + 68; }   // activation buffer row stride (D hidden + 64 enc + 4 pad)
constexpr int WS_LD = 260;     // staged weight row stride
constexpr int KC = 16;         // reduction chunk

// out[m][n] (+)= act( sum_k in[m][k] * B[k][n] + bias[n] ), m < 64, n < 64*NJ
//   !TRANS: B[k][n] = W[n*ldw + k]   (forward: W is nn.Linear (out,in) row-major)
//    TRANS: B[k][n] = W[k*ldw + n]   (dgrad:   g_in = g_out @ W)
template <int NJ, bool TRANS, int ACT, bool ACCUM>
__device__ __forceinline__ void tile_gemm(const float* in, int ldi, int K, const float* __restrict__ W, int ldw,
                                          int nvalid, int kvalid, const float* __restrict__ bias, float* out, int ldo,
                                          float* Ws) {
  constexpr int NOUT = 64 * NJ;
  constexpr int NST = NJ * 4;  // staged elements per thread per chunk
  const int tid = threadIdx.x, ng = tid & 15, mg = tid >> 4;
  float acc[4][4 * NJ];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 4 * NJ; ++c) acc[r][c] = 0.f;
  float stage[NST];
  auto gload = [&](int k0) {
#pragma unroll
    for (int e = 0; e < NST; ++e) {
      int idx = tid + 256 * e, kk, n;
      if (!TRANS) { kk = idx & 15; n = idx >> 4; } else { n = idx % NOUT; kk = idx / NOUT; }
      int k = k0 + kk;
      float v = 0.f;
      if (k < kvalid && n < nvalid) v = TRANS ? __ldg(W + (size_t)k * ldw + n) : __ldg(W + (size_t)n * ldw + k);
      stage[e] = v;
    }
  };
  auto sstore = [&](float* dst) {
#pragma unroll
    for (int e = 0; e < NST; ++e) {
      int idx = tid + 256 * e, kk, n;
      if (!TRANS) { kk = idx & 15; n = idx >> 4; } else { n = idx % NOUT; kk = idx / NOUT; }
      dst[kk * WS_LD + n] = stage[e];
    }
  };
  const int nchunks = K / KC;
  gload(0); sstore(Ws); __syncthreads();
  for (int c = 0; c < nchunks; ++c) {
    const float* cur = Ws + (c & 1) * KC * WS_LD;
    if (c + 1 < nchunks) gload((c + 1) * KC);
#pragma unroll
    for (int k4 = 0; k4 < 4; ++k4) {
      float4 a[4];
#pragma unroll
      for (int r = 0; r < 4; ++r) a[r] = *reinterpret_cast<const float4*>(in + (mg * 4 + r) * ldi + c * KC + k4 * 4);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float* wrow = cur + (k4 * 4 + q) * WS_LD + ng * 4;
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
          float4 w = *reinterpret_cast<const float4*>(wrow + 64 * j);
#pragma unroll
          for (int r = 0; r < 4; ++r) {
            float av = q == 0 ? a[r].x : (q == 1 ? a[r].y : (q == 2 ? a[r].z : a[r].w));
            acc[r][4 * j + 0] = fmaf(av, w.x, acc[r][4 * j + 0]);
            acc[r][4 * j + 1] = fmaf(av, w.y, acc[r][4 * j + 1]);
            acc[r][4 * j + 2] = fmaf(av, w.z, acc[r][4 * j + 2]);
            acc[r][4 * j + 3] = fmaf(av, w.w, acc[r][4 * j + 3]);
          }
        }
      }
    }
    if (c + 1 < nchunks) sstore(Ws + ((c + 1) & 1) * KC * WS_LD);
    __syncthreads();
  }
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    int n = ng * 4 + 64 * j;
    float b[4] = {0.f, 0.f, 0.f, 0.f};
    if (bias) {
#pragma unroll
      for (int cc = 0; cc < 4; ++cc) if (n + cc < nvalid) b[cc] = __ldg(bias + n + cc);
    }
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      float* o = out + (mg * 4 + r) * ldo + n;
      float4 v = make_float4(acc[r][4 * j] + b[0], acc[r][4 * j + 1] + b[1], acc[r][4 * j + 2] + b[2], acc[r][4 * j + 3] + b[3]);
      if (ACT == 1) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
      if (ACCUM) { float4 p = *reinterpret_cast<float4*>(o); v.x += p.x; v.y += p.y; v.z += p.z; v.w += p.w; }
      *reinterpret_cast<float4*>(o) = v;
    }
  }
}

// copy a [64][ncols] SMEM tile (row stride lds) to global rows m0.. (row stride ncols)
__device__ __forceinline__ void tile_to_global(const float* s, int lds, float* g, size_t m0, int ncols) {
  const int per_row = ncols / 4;
  for (int idx = threadIdx.x; idx < TM * per_row; idx += 256) {
    int row = idx / per_row, c4 = idx % per_row;
    float4 v = *reinterpret_cast<const float4*>(s + row * lds + c4 * 4);
    *reinterpret_cast<float4*>(g + (m0 + row) * ncols + c4 * 4) = v;
  }
}

__device__ __forceinline__ void row_view_dir(const nnb_render_args& a, size_t m, size_t M, const Ray& ray, float v[3]) {
  if (a.pts) {
    size_t mm = m < M ? m : M - 1;
#pragma unroll
    for (int c = 0; c < 3; ++c) v[c] = a.dirs ? __ldg(a.dirs + 3 * mm + c) : 1.f;
    return;
  }
  view_dir(a, ray, v);
}

struct SimtPtrs {
  SampleRec* rec;
  float *h[8], *feat, *hr, *enc, *denc;
  float *dy[8], *dfeat, *dyr;
  float4 *dyc, *gs, *gp, *gv;
  float *rayred, *wpart;
};

__device__ __forceinline__ void row_geometry(const nnb_render_args& a, size_t m, size_t M, Ray& ray, int& n, int& i, float& z,
                                             float p[3]) {
  size_t mm = m < M ? m : M - 1;
  if (a.pts) {   // explicit-point field query: no ray, the point is given
    n = (int)mm; i = 0; z = 0.f;
    p[0] = __ldg(a.pts + 3 * mm); p[1] = __ldg(a.pts + 3 * mm + 1); p[2] = __ldg(a.pts + 3 * mm + 2);
    return;
  }
  n = (int)(mm / a.S); i = (int)(mm % a.S);
  setup_ray(a, n, ray);
  z = sample_z(a, n, i);
  sample_point(a, ray, z, p);
}

// MODE of simt_fwd_tile: SF_RAYS (simt_mlp_fwd: the render's samples, or explicit points a.pts) writes records and the stash.
// SF_MARCH / SF_SECANT (simt_march / simt_secant, nnb_ray_march on this engine) are occupancy-only tiles whose points come from q: the
// colour branch is skipped and the density head's occupancy - tau goes to the march's back end instead of a record.
//   SF_MARCH: row r is step 128 q.block + 64 pass + r of ray `mray` (clamped to its last step); the value goes to s_val[64 pass + r].
//   SF_SECANT: row r is the secant iterate of hit ray q.list[m0 + r] (rows past M: the point 0, ignored); pass = the secant pass.
// SF_FRAME (simt_frame, nnb_render_frame on this engine): SF_RAYS on the rows frame_row gives (M = N S), with nothing stashed and no
// record.  The colour head puts each row's (r, g, b, a) in a row area at the start of oth, and the CTA's warps take the tile's
// ray-chunks in turn through frame_step (nnb_frame.cuh).  fr / n_live: the round and its ray-chunk count.
// SF_CHUNK (simt_frame_stash, nnb_render_frame_bwd on this engine): SF_RAYS with the stash and records on the rows of chunk fr.k of every
// ray (chunk_row); geometry, view direction and the record's z come from the row's sample, stores go to the row.
// SF_PACK (simt_stash_pack, nnb_render_fwd_tmin_engine on this engine): SF_CHUNK on the rows of round fr.k's list (pack_row), n_live of
// them; the caller offsets P to the round's first row of the packed stash.
enum : int { SF_RAYS = 0, SF_MARCH = 1, SF_SECANT = 2, SF_FRAME = 3, SF_CHUNK = 4, SF_PACK = 5 };

// Row `row` of frame tile `tile`: a ray-chunk is R = min(S, 32) rows and a tile holds 64 / R of them, so row r is sample 32 fr.k + r % R
// of the ray in slot (64 / R) tile + r / R of the round.  Slots past the round's last repeat it, rows past a ray's last sample evaluate
// that sample, and the rows past the tile's last whole ray-chunk (64 % R of them) evaluate some sample; frame_step reads none of them.
__device__ __forceinline__ size_t frame_row(const nnb_render_args& a, const FramePtrs& fr, unsigned tile, int row, int n_live) {
  const int R = min(a.S, 32);
  const int slot = min((TM / R) * (int)tile + row / R, n_live - 1);
  const int n = fr.list ? fr.list[slot] : slot;
  return (size_t)n * a.S + min(32 * fr.k + row % R, a.S - 1);
}

// Row m of chunk k's stash (nnb_render_frame_bwd on this engine, nnb_frame.cuh): ray n owns R = min(S, 32) consecutive rows, row R n + j
// is sample 32 k + j of ray n, clamped to the ray's last sample; rows past the last ray (the Mpad tail) repeat row R N - 1, and no later
// stage reads them.  Returns the sample's row n S + i in nnb_render_fwd's order, which is m itself at S <= 32.
__device__ __forceinline__ size_t chunk_row(const nnb_render_args& a, int k, size_t m) {
  const int R = min(a.S, 32);
  const size_t last = (size_t)a.N * R - 1;
  if (m > last) m = last;
  return (m / R) * a.S + min(32 * k + (int)(m % R), a.S - 1);
}

// ---- the packed stash of nnb_render_fwd_tmin_engine / nnb_render_bwd_tmin_engine on this engine ------------------------------------
// Round k evaluates chunk k of the rays lists[k] ([C][N], increasing n, frame_live_list) with counts[k] of them.  Its rows start at
// base_k = sum over j < k of 64 ceil(R count_j / 64) (R = min(S, 32); each round padded to the 64-row tile), and row base_k + R slot + j is
// sample 32 k + j of ray lists[k][slot].  At S <= 32 there is one round and row n S + j is nnb_render_fwd's row.  Counts are clamped to
// 0..N where they are read, so every row stays below the stash's C 64 ceil(R N / 64) rows.
__device__ __forceinline__ size_t pack_round_base(const int* counts, int k, int N, int R) {
  size_t r = 0;
  for (int j = 0; j < k; ++j) r += (size_t)TM * ((R * frame_live_count(counts + j, N) + TM - 1) / TM);
  return r;
}
// sample row n S + i (nnb_render_fwd's order) of row m of round fr.k (n_live >= 1 rays): slots past the list's last repeat it
__device__ __forceinline__ size_t pack_row(const nnb_render_args& a, const FramePtrs& fr, size_t m, int n_live) {
  const int R = min(a.S, 32);
  const int slot = min((int)(m / R), n_live - 1);
  return (size_t)fr.list[slot] * a.S + min(32 * fr.k + (int)(m % R), a.S - 1);
}
// sample row of packed row m: the round whose rows hold m (the last round past them), the slot's ray (padding rows take the list's last
// ray; their cotangent is zero)
__device__ __forceinline__ size_t pack_row_sample(const nnb_render_args& a, const int* lists, const int* counts, int C, size_t m) {
  const int R = min(a.S, 32);
  size_t r = 0;
  int k = 0;
  for (; k < C - 1; ++k) {
    const size_t rows = (size_t)TM * ((R * frame_live_count(counts + k, a.N) + TM - 1) / TM);
    if (m < r + rows) break;
    r += rows;
  }
  const int slot = min((int)((m - r) / R), max(frame_live_count(counts + k, a.N) - 1, 0));
  const int n = min(max(lists[(size_t)k * a.N + slot], 0), a.N - 1);
  return (size_t)n * a.S + min(32 * k + (int)((m - r) % R), a.S - 1);
}

// one 64-row tile of the exact forward: rows m0 = 64 tile .. m0 + 63 of M
template <int D, int MODE>
__device__ __forceinline__ void simt_fwd_tile(const nnb_render_args& a, const SimtPtrs& P, size_t M, int stash, unsigned tile, const MarchPtrs& q,
                                              int mray, int pass, float* s_val, const FramePtrs& fr = FramePtrs{}, int n_live = 0) {
  constexpr int LDB = ldb<D>(), NJ = D / 64, NJR = D >= 128 ? D / 128 : 1;   // output column blocks of the trunk / rgb hidden layers
  extern __shared__ __align__(16) float smem[];
  float* buf0 = smem; float* buf1 = buf0 + TM * LDB; float* Ws = buf1 + TM * LDB;
  const int tid = threadIdx.x;
  const size_t m0 = (size_t)tile * TM;
  const float* w = a.weights;
  auto row_m = [&](int row) {
    return MODE == SF_FRAME ? frame_row(a, fr, tile, row, n_live) : MODE == SF_CHUNK ? chunk_row(a, fr.k, m0 + row)
         : MODE == SF_PACK ? pack_row(a, fr, m0 + row, n_live) : m0 + row;
  };
  {  // prologue: encode positions into columns D..D+63 of both buffers
    int row = tid & 63, part = tid >> 6;
    Ray ray; int n, i; float z, p[3];
    if constexpr (MODE == SF_MARCH) {
      march_point(q, mray, march_depth(q.near, __ldg(q.far + mray), __ldg(q.frac + min(q.block * MARCH_BLOCK + pass * TM + row, q.n_steps - 1))), p);
    } else if constexpr (MODE == SF_SECANT) {
      p[0] = p[1] = p[2] = 0.f;
      if (m0 + row < M) {
        const int r = q.list[m0 + row];
        march_point(q, r, secant_depth((pass == 0 ? q.brk0 : q.brk1)[r]), p);
      }
    } else {
      row_geometry(a, row_m(row), M, ray, n, i, z, p);
    }
    float* e0 = buf0 + row * LDB + D; float* e1 = buf1 + row * LDB + D;
    if (part == 0) {
#pragma unroll
      for (int c = 0; c < 3; ++c) { e0[c] = p[c]; e1[c] = p[c]; }
      e0[63] = 0.f; e1[63] = 0.f;
    }
    for (int l = part; l < 10; l += 4) {
      float f = (float)(1 << l);
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        float s, co; sincosf(__fmul_rn(f, p[c]), &s, &co);
        e0[3 + 6 * l + c] = s; e1[3 + 6 * l + c] = s; e0[6 + 6 * l + c] = co; e1[6 + 6 * l + c] = co;
      }
    }
  }
  __syncthreads();
  if ((MODE == SF_RAYS || MODE == SF_CHUNK || MODE == SF_PACK) && stash) {
    for (int idx = tid; idx < TM * 16; idx += 256) {
      int row = idx >> 4, c4 = idx & 15;
      *reinterpret_cast<float4*>(P.enc + (m0 + row) * 64 + c4 * 4) = *reinterpret_cast<const float4*>(buf0 + row * LDB + D + c4 * 4);
    }
  }
  float* cur = buf0; float* oth = buf1;
  for (int l = 0; l < 8; ++l) {
    const float* in = (l == 0) ? cur + D : cur;
    int K = (l == 0) ? 64 : (l == 4 ? D + 64 : D);
    int kvalid = (l == 0) ? 63 : (l == 4 ? D + 63 : D);
    tile_gemm<NJ, false, 1, false>(in, LDB, K, w + nnb::w_off(D, l), nnb::w_ld(D, l), D, kvalid, w + nnb::b_off(D, l), oth, LDB, Ws);
    __syncthreads();
    if ((MODE == SF_RAYS || MODE == SF_CHUNK || MODE == SF_PACK) && stash) tile_to_global(oth, LDB, P.h[l], m0, D);
    float* t_ = cur; cur = oth; oth = t_;
  }
  // cur = h8.  density head: 4 threads per row
  const int hrow = tid >> 2, hc = tid & 3;
  float s_logit;
  {
    float acc = 0.f;
    const float* hr_ = cur + hrow * LDB + hc * (D / 4);
    const float* ws_ = w + nnb::W_SIG(D) + hc * (D / 4);
#pragma unroll 8
    for (int k = 0; k < D / 4; ++k) acc = fmaf(hr_[k], __ldg(ws_ + k), acc);
    acc += __shfl_xor_sync(0xffffffffu, acc, 1);
    acc += __shfl_xor_sync(0xffffffffu, acc, 2);
    s_logit = acc + __ldg(w + nnb::B_SIG(D));
  }
  if constexpr (MODE == SF_MARCH || MODE == SF_SECANT) {   // occupancy only: the colour branch does not enter the march
    if (hc == 0) {
      float sigma;
      auto f = [&] { return __fsub_rn(density_act(s_logit, a.flags, &sigma), q.tau); };
      if (MODE == SF_MARCH) s_val[pass * TM + hrow] = f();
      else if (m0 + hrow < M) secant_update(q, q.list[m0 + hrow], pass == 0, f);
    }
    return;
  }
  // feature layer (no activation) -> oth, then dir encoding into cols D..D+31
  tile_gemm<NJ, false, 0, false>(cur, LDB, D, w + nnb::W_FEAT(D), D, D, D, w + nnb::B_FEAT(D), oth, LDB, Ws);
  if (tid < TM) {
    Ray ray; int n, i; float z, p[3], v[3];
    row_geometry(a, row_m(tid), M, ray, n, i, z, p);
    row_view_dir(a, row_m(tid), M, ray, v);
    float* de = oth + tid * LDB + D;
    encode<4>(v, [&](int k, float val) { de[k] = val; });
#pragma unroll
    for (int k = 27; k < 32; ++k) de[k] = 0.f;
  }
  __syncthreads();
  if (stash) {
    tile_to_global(oth, LDB, P.feat, m0, D);
    for (int idx = tid; idx < TM * 8; idx += 256) {
      int row = idx >> 3, c4 = idx & 7;
      *reinterpret_cast<float4*>(P.denc + (m0 + row) * 32 + c4 * 4) = *reinterpret_cast<const float4*>(oth + row * LDB + D + c4 * 4);
    }
  }
  // rgb hidden layer: D / 2 columns (at D = 64 one 64-column block with the upper 32 columns zero)
  tile_gemm<NJR, false, 1, false>(oth, LDB, D + 32, w + nnb::W_RGBH(D), D + 27, D / 2, D + 27, w + nnb::B_RGBH(D), cur, LDB, Ws);
  __syncthreads();
  if (stash) tile_to_global(cur, LDB, P.hr, m0, D / 2);
  {  // colour head + record
    float val = 0.f;
    if (hc < 3) {
      const float* hr_ = cur + hrow * LDB; const float* wc = w + nnb::W_RGB(D) + hc * (D / 2);
      float acc = 0.f;
#pragma unroll 8
      for (int k = 0; k < D / 2; ++k) acc = fmaf(hr_[k], __ldg(wc + k), acc);
      val = sigmoid_f(acc + __ldg(w + nnb::B_RGB(D) + hc));
    }
    if constexpr (MODE == SF_FRAME) {   // row area: (r, g, b, a) of row hrow; oth was last read by the rgb hidden layer
      float sigma;
      oth[hrow * 4 + hc] = hc < 3 ? val : density_act(s_logit, a.flags, &sigma);
    } else {
      float* rec = reinterpret_cast<float*>(P.rec + m0 + hrow);
      if (hc < 3) rec[hc] = val;
      else {
        Ray ray; int n, i; float z, p[3], sigma;
        row_geometry(a, row_m(hrow), M, ray, n, i, z, p);
        rec[3] = density_act(s_logit, a.flags, &sigma);
        rec[4] = s_logit; rec[5] = z; rec[6] = 0.f; rec[7] = 0.f;
      }
    }
  }
  if constexpr (MODE == SF_FRAME) {
    __syncthreads();   // every row is in the row area
    const int R = min(a.S, 32), per = TM / R;
    for (int c = tid >> 5; c < per; c += 8)
      frame_step(a, fr, per * (int)tile + c, n_live, reinterpret_cast<const unsigned char*>(oth + c * R * 4), tid & 31);
  }
}

template <int D>
__global__ void __launch_bounds__(256, 1) simt_mlp_fwd(nnb_render_args a, SimtPtrs P, size_t M, int stash) {
  simt_fwd_tile<D, SF_RAYS>(a, P, M, stash, blockIdx.x, MarchPtrs{}, 0, 0, nullptr);
}

// Device-count form of simt_mlp_fwd on explicit points (nnb_geometry_frame on this engine): the rows are points off .. off + n - 1 of the
// compacted list, n = min(*count - off, cap), read when the kernel starts; a.pts / a.dirs and the outputs start at row off.  A CTA past
// the n rows exits before any barrier.
template <int D>
__global__ void __launch_bounds__(256, 1) simt_mlp_fwd_n(nnb_render_args a, SimtPtrs P, const int* __restrict__ count, int off, int cap,
                                                         int stash) {
  const int n = min(*count - off, cap);
  if ((int)blockIdx.x * TM >= n) return;
  simt_fwd_tile<D, SF_RAYS>(a, P, (size_t)n, stash, blockIdx.x, MarchPtrs{}, 0, 0, nullptr);
}

// one round of nnb_ray_march on this engine: block q.block of every ray of q.list (n_rays rays when q.count is NULL), one ray per CTA
// and iteration, its 128 steps as two 64-row tiles (the second only when the ray has steps there); march_scan reduces them
template <int D>
__global__ void __launch_bounds__(256, 1) simt_march(nnb_render_args a, const __grid_constant__ MarchPtrs q, int n_rays) {
  __shared__ __align__(16) float s_val[MARCH_BLOCK];
  const int n_tiles = q.count ? *q.count : n_rays;
  for (int t = blockIdx.x; t < n_tiles; t += gridDim.x) {
    const int ray = q.list ? q.list[t] : t;
    for (int pass = 0; pass < 2 && q.block * MARCH_BLOCK + pass * TM < q.n_steps; ++pass) {
      simt_fwd_tile<D, SF_MARCH>(a, SimtPtrs{}, 0, 0, 0u, q, ray, pass, s_val);
      __syncthreads();
    }
    if (threadIdx.x < 32) march_scan(q, ray, s_val, threadIdx.x);
    __syncthreads();
  }
}

// the q.n_secant secant passes of nnb_ray_march over the *q.count hit rays of q.list, 64 rays per tile; a pass reads the brackets the
// previous pass of the same CTA wrote
template <int D>
__global__ void __launch_bounds__(256, 1) simt_secant(nnb_render_args a, const __grid_constant__ MarchPtrs q) {
  const size_t M = (size_t)*q.count;
  for (unsigned tile = blockIdx.x; (size_t)tile * TM < M; tile += gridDim.x)
    for (int pass = 0; pass < q.n_secant; ++pass) {
      simt_fwd_tile<D, SF_SECANT>(a, SimtPtrs{}, M, 0, tile, q, 0, pass, nullptr);
      __syncthreads();
    }
}

// one round of nnb_render_frame on this engine: chunk f.k of every ray of f.list (of every ray when f.list is NULL), 64 / min(S, 32)
// ray-chunks per 64-row tile; the ray-chunk count is read when the kernel starts
template <int D>
__global__ void __launch_bounds__(256, 1) simt_frame(nnb_render_args a, const __grid_constant__ FramePtrs f) {
  const int n_live = f.count ? *f.count : a.N, per = TM / min(a.S, 32);
  const unsigned n_tiles = (unsigned)((n_live + per - 1) / per);
  for (unsigned tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    simt_fwd_tile<D, SF_FRAME>(a, SimtPtrs{}, (size_t)a.N * a.S, 0, tile, MarchPtrs{}, 0, 0, nullptr, f, n_live);
    __syncthreads();   // the back end is done with the row area before the next tile's prologue writes the buffers
  }
}

// one reverse round of nnb_render_frame_bwd on this engine: chunk f.k of every ray, records and the training stash of its R N rows
// (chunk_row), one 64-row tile per CTA
template <int D>
__global__ void __launch_bounds__(256, 1) simt_frame_stash(nnb_render_args a, SimtPtrs P, const __grid_constant__ FramePtrs f) {
  simt_fwd_tile<D, SF_CHUNK>(a, P, (size_t)a.N * a.S, 1, blockIdx.x, MarchPtrs{}, 0, 0, nullptr, f);
}

// one forward round of nnb_render_fwd_tmin_engine on this engine: chunk f.k of the f.count rays of f.list, records and the training stash
// of its R count rows (SF_PACK) into the packed stash from row base_k on, one 64-row tile per CTA.  The count is read when the kernel
// starts; a CTA past the round's rows exits before any barrier.
template <int D>
__global__ void __launch_bounds__(256, 1) simt_stash_pack(nnb_render_args a, SimtPtrs P, const __grid_constant__ FramePtrs f) {
  const int R = min(a.S, 32), n_live = frame_live_count(f.count, a.N);
  if ((int)blockIdx.x * TM >= R * n_live) return;
  const size_t mo = pack_round_base(f.count - f.k, f.k, a.N, R);
  P.rec += mo; P.feat += mo * D; P.hr += mo * (D / 2); P.enc += mo * 64; P.denc += mo * 32;
  for (int l = 0; l < 8; ++l) P.h[l] += mo * D;
  simt_fwd_tile<D, SF_PACK>(a, P, (size_t)a.N * a.S, 1, blockIdx.x, MarchPtrs{}, 0, 0, nullptr, f, n_live);
}

// ---------------------------------------------------------------------------------------
// compositing (rendering.py:122-158), one warp per ray; shared by both engines
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ float sample_alpha(const nnb_render_args& a, const SampleRec* rr, int i, const SampleRec& me) {
  return composite_alpha(a, i, me.a, me.z, [&] { return rr[i + 1].z; });
}

__global__ void composite_fwd(nnb_render_args a, const SampleRec* recs) {
  const int lane = threadIdx.x & 31, n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (n >= a.N) return;
  Ray ray; setup_ray(a, n, ray);
  const SampleRec* rr = recs + (size_t)n * a.S;
  float carry = 1.f, C0 = 0.f, C1 = 0.f, C2 = 0.f, Dist = 0.f, acc = 0.f;
  for (int c = 0; c * 32 < a.S; ++c) {
    int i = c * 32 + lane; bool valid = i < a.S;
    SampleRec me = valid ? rr[i] : SampleRec{0, 0, 0, 0, 0, 0, 0, 0};
    float alpha = valid ? sample_alpha(a, rr, i, me) : 0.f;
    float om = valid ? __fadd_rn(__fsub_rn(1.f, alpha), NNB_EPS) : 1.f;
    float incl = warp_incl_prod(om, lane);
    float excl = __shfl_up_sync(0xffffffffu, incl, 1); if (lane == 0) excl = 1.f;
    float T = carry * excl;
    carry *= __shfl_sync(0xffffffffu, incl, 31);
    float wgt = alpha * T;
    C0 += wgt * me.r; C1 += wgt * me.g; C2 += wgt * me.b; Dist += wgt * me.z; acc += wgt;
    if (valid) {
      if (a.z_vals) a.z_vals[(size_t)n * a.S + i] = me.z;
      if (a.alpha) a.alpha[(size_t)n * a.S + i] = alpha;
    }
  }
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

__global__ void composite_bwd(nnb_render_bwd_args b, const SampleRec* recs, float4* gs) {
  const nnb_render_args& a = b.fwd;
  const int lane = threadIdx.x & 31, n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (n >= a.N) return;
  Ray ray; setup_ray(a, n, ray);
  const SampleRec* rr = recs + (size_t)n * a.S;
  float gD = b.g_depth_pred ? __ldg(b.g_depth_pred + n) : 0.f;
  if ((a.flags & NNB_EVAL) && (a.flags & NNB_NORMALISE)) gD = gD / ray.nrm;
  const float gC0 = __ldg(b.g_rgb + 3 * n), gC1 = __ldg(b.g_rgb + 3 * n + 1), gC2 = __ldg(b.g_rgb + 3 * n + 2);
  const float gsum = (a.flags & NNB_WHITE_BG) ? (gC0 + gC1 + gC2) : 0.f;
  // chunk c's terms from its records: alpha, om = 1 - alpha + eps, the inclusive product of om over the chunk, and the transmittance
  // T given the carry into the chunk
  auto chunk = [&](int c, float carry, float& alpha, float& om, float& incl, float& T) {
    const int i = c * 32 + lane; const bool valid = i < a.S;
    const SampleRec me = valid ? rr[i] : SampleRec{0, 0, 0, 0, 0, 0, 0, 0};
    alpha = valid ? sample_alpha(a, rr, i, me) : 0.f;
    om = valid ? __fadd_rn(__fsub_rn(1.f, alpha), NNB_EPS) : 1.f;
    incl = warp_incl_prod(om, lane);
    float excl = __shfl_up_sync(0xffffffffu, incl, 1); if (lane == 0) excl = 1.f;
    T = carry * excl;
    return me;
  };
  // forward sweep: only the transmittance carried into each chunk of 32 samples; lane c keeps chunk c's, hence S <= 32 * 32 = 1024
  float carry = 1.f, carry_c = 1.f;
  const int C = (a.S + 31) / 32;
  for (int c = 0; c < C; ++c) {
    if (lane == c) carry_c = carry;
    float alpha, om, incl, T;
    chunk(c, carry, alpha, om, incl, T);
    carry *= __shfl_sync(0xffffffffu, incl, 31);
  }
  // reverse sweep: each chunk's terms recomputed from the records with the same operations, then the in-chunk suffix scan with the
  // suffix of the later chunks carried in
  float carry_s = 0.f;
  for (int c = C - 1; c >= 0; --c) {
    const int i = c * 32 + lane; const bool valid = i < a.S;
    float alpha, om, incl_p, T;
    const SampleRec me = chunk(c, __shfl_sync(0xffffffffu, carry_c, c), alpha, om, incl_p, T);
    const float w = alpha * T;
    // d L / d w with its multiply-adds spelled out: a contracted a*b + c*d may fuse either product, and the choice would otherwise
    // depend on how the compiler schedules this loop
    const float gw = fmaf(gD, me.z, fmaf(gC2, me.b, fmaf(gC1, me.g, gC0 * me.r))) - gsum;
    float df = 1.f;  // d alpha / d a
    if (a.flags & NNB_DIST_ALPHA) {
      if (i >= a.S - 1) df = 0.f;
      else { float delta = __fsub_rn(rr[i + 1].z, me.z); df = delta * expf(-me.a * delta); }
    }
    float wg = valid ? w * gw : 0.f;
    float incl = warp_incl_sum_rev(wg, lane);
    float excl = __shfl_down_sync(0xffffffffu, incl, 1); if (lane == 31) excl = 0.f;
    float suffix = excl + carry_s;
    carry_s += __shfl_sync(0xffffffffu, incl, 0);
    float g_alpha = T * gw - suffix / om;
    if (valid) gs[(size_t)n * a.S + i] = make_float4(w * gC0, w * gC1, w * gC2, g_alpha * df);
  }
}

// The per-ray kernels of nnb_render_fwd_tmin_engine / nnb_render_bwd_tmin_engine on the packed stash.  They are the statements of the
// tensor-core pair's stash_frame_step, stash_chunk_adjoint and stash_ray_acc (nnb_tc.cu) on this engine's rows (R = min(S, 32) rows per
// slot, rounds padded to 64 rows), copied rather than shared so that those kernels keep their SASS; the adjoint takes composite_bwd's fused
// d L / d alpha (composite_chunk_bwd<true>), as the exact frame pair does, so that at S <= 32 the gradients are nnb_render_bwd's bits.

// back end of forward round f.k: one warp per slot, frame_step's arithmetic on the round's records, from the ray's carry and lane partials
// of the rounds before.  Lane 0 stores the carry, its checkpoint ckpt[k][n] and c_n: k + 1 when the ray stops, C while it stays live.
__global__ void simt_pack_step(nnb_render_args a, const __grid_constant__ FramePtrs f, const SampleRec* __restrict__ rec,
                               float* __restrict__ ckpt, int C) {
  const int lane = threadIdx.x & 31, slot = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (slot >= frame_live_count(f.count, a.N)) return;
  const int n = f.list[slot], R = min(a.S, 32);
  const int i = 32 * f.k + lane;
  const bool valid = i < a.S;   // implies lane < R
  float4 me = make_float4(0.f, 0.f, 0.f, 0.f);
  float z = 0.f, alpha = 0.f;
  if (valid) {
    const SampleRec r = rec[pack_round_base(f.count - f.k, f.k, a.N, R) + (size_t)slot * R + lane];
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

// slot of ray n in a round's list (increasing n): the first slot whose ray is not below n, clamped to the list
__device__ __forceinline__ int pack_slot(const int* list, int count, int n) {
  int lo = 0, hi = count;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (list[mid] < n) lo = mid + 1; else hi = mid;
  }
  return min(lo, max(count - 1, 0));
}

// Compositing adjoint of the packed stash, one warp per ray: chunks c_n - 1 .. 0, the suffix carry starting at 0 in the ray's last chunk.
// Lanes past a ray's R rows (S < 32 only) have no row and write nothing.  Warps N .. N + 2 C - 1 zero the cotangents of round
// (w - N) / 2's padding rows base_k + R count_k .. base_k+1 - 1 (fewer than 64).  Thread 0 stores counts[C] = base_C-1 + R count_C-1, the
// rows of the weight-gradient stage (N S at S <= 32).
__global__ void simt_pack_adjoint(nnb_render_bwd_args b, const __grid_constant__ FrameBwdPtrs f, const int* __restrict__ chunks,
                                  const int* __restrict__ lists, int* __restrict__ counts) {
  const nnb_render_args& a = b.fwd;
  const int C = f.rounds, R = min(a.S, 32);
  const int lane = threadIdx.x & 31, w = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (w == 0 && lane == 0)
    counts[C] = (int)(pack_round_base(counts, C - 1, a.N, R) + (size_t)R * frame_live_count(counts + C - 1, a.N));
  if (w >= a.N) {
    const int k = (w - a.N) / 2;
    if (k >= C) return;
    const int rows = R * frame_live_count(counts + k, a.N), r = rows + 32 * ((w - a.N) % 2) + lane;
    if (r < (rows + TM - 1) / TM * TM) f.gs[pack_round_base(counts, k, a.N, R) + r] = make_float4(0.f, 0.f, 0.f, 0.f);
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
    const int slot = pack_slot(lists + (size_t)k * a.N, frame_live_count(counts + k, a.N), n);
    const size_t m = pack_round_base(counts, k, a.N, R) + (size_t)slot * R + lane;
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
    const float4 g = composite_chunk_bwd<true>(alpha, valid, me.r, me.g, me.b, me.z, df, lane, carry, gC0, gC1, gC2, gD, gsum, carry_s);
    if (lane < R) f.gs[m] = g;
  }
}

// ray_bwd's lane sums on the packed stash, one warp per ray: the terms of chunks c_n - 1 .. 0 added in that order (frame_ray_acc<true>'s)
// to lane partials that start at 0, stored once for frame_ray_finish
__global__ void simt_pack_ray_acc(nnb_render_args a, const __grid_constant__ FrameBwdPtrs f, const int* __restrict__ chunks,
                                  const int* __restrict__ lists, const int* __restrict__ counts) {
  const int lane = threadIdx.x & 31, n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (n >= a.N) return;
  const int R = min(a.S, 32);
  float v[9];
#pragma unroll
  for (int c = 0; c < 9; ++c) v[c] = 0.f;
  for (int k = frame_ray_chunks(chunks, n, f.rounds) - 1; k >= 0; --k) {
    if (32 * k + lane >= a.S) continue;   // implies lane < R
    const int slot = pack_slot(lists + (size_t)k * a.N, frame_live_count(counts + k, a.N), n);
    const size_t m = pack_round_base(counts, k, a.N, R) + (size_t)slot * R + lane;
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

// ---------------------------------------------------------------------------------------
// B2: data-gradient chain
// ---------------------------------------------------------------------------------------
// MODE of simt_dgrad_tile: DG_ROWS (simt_mlp_dgrad): row m is sample m.  DG_CHUNK (simt_dgrad_chunk, nnb_render_frame_bwd on this engine):
// the rows of chunk `chunk`'s stash as simt_frame_stash wrote them: row_geometry and row_view_dir take the row's sample chunk_row(a,
// chunk, m), everything else the row.  DG_PACK (simt_dgrad_pack, nnb_render_bwd_tmin_engine on this engine): the rows of the packed stash,
// whose samples are pack_row_sample(a, lists, counts, chunk, m) (chunk = C).
enum : int { DG_ROWS = 0, DG_CHUNK = 1, DG_PACK = 2 };

// one 64-row tile of the chain: rows m0 = 64 tile .. m0 + 63 of M
template <int D, int MODE = DG_ROWS>
__device__ __forceinline__ void simt_dgrad_tile(const nnb_render_args& a, const SimtPtrs& P, size_t M, int write_dy, unsigned tile,
                                                int chunk = 0, const int* lists = nullptr, const int* counts = nullptr) {
  constexpr int LDB = ldb<D>(), NJ = D / 64, DR = D / 2;
  extern __shared__ __align__(16) float smem[];
  float* bufA = smem; float* bufB = bufA + TM * LDB; float* Ws = bufB + TM * LDB;
  float* genc = Ws + 2 * KC * WS_LD;          // [64][64]
  float* gyc = genc + TM * 64;                // [64][4]
  const int tid = threadIdx.x;
  const size_t m0 = (size_t)tile * TM;
  const float* w = a.weights;
  // the row's sample for the geometry (DG_CHUNK: M counts the chunk's rows, the samples are the N S of the render)
  auto row_s = [&](int row) {
    return MODE == DG_CHUNK ? chunk_row(a, chunk, m0 + row)
         : MODE == DG_PACK ? pack_row_sample(a, lists, counts, chunk, m0 + row) : m0 + row;
  };
  const size_t MS = MODE == DG_CHUNK || MODE == DG_PACK ? (size_t)a.N * a.S : M;
  {  // 1. head adjoints
    int row = tid >> 2, c = tid & 3; size_t m = m0 + row;
    float4 g = (m < M) ? P.gs[m] : make_float4(0, 0, 0, 0);
    const float* rec = reinterpret_cast<const float*>(P.rec + m);
    float v;
    if (c < 3) { float rgb = rec[c]; float gc = c == 0 ? g.x : (c == 1 ? g.y : g.z); v = gc * rgb * (1.f - rgb); }
    else v = g.w * density_act_grad(rec[4], a.flags);
    gyc[row * 4 + c] = v;
    if (write_dy) reinterpret_cast<float*>(P.dyc + m)[c] = v;
  }
  __syncthreads();
  // 2. g_yr = (g_yc @ Wc) * (hr > 0)
  for (int idx = tid; idx < TM * DR; idx += 256) {
    int row = idx / DR, j = idx % DR; size_t m = m0 + row;
    float v = gyc[row * 4] * __ldg(w + nnb::W_RGB(D) + j) + gyc[row * 4 + 1] * __ldg(w + nnb::W_RGB(D) + DR + j) +
              gyc[row * 4 + 2] * __ldg(w + nnb::W_RGB(D) + 2 * DR + j);
    v = (P.hr[m * DR + j] > 0.f) ? v : 0.f;
    bufA[row * LDB + j] = v;
    if (write_dy) P.dyr[m * DR + j] = v;
  }
  __syncthreads();
  // 3. g_xr = g_yr @ Wr : feature part -> bufB[:, :D], dir-encoding part -> bufB[:, D:D+64]
  tile_gemm<NJ, true, 0, false>(bufA, LDB, DR, w + nnb::W_RGBH(D), D + 27, D, DR, nullptr, bufB, LDB, Ws);
  tile_gemm<1, true, 0, false>(bufA, LDB, DR, w + nnb::W_RGBH(D) + D, D + 27, 27, DR, nullptr, bufB + D, LDB, Ws);
  __syncthreads();
  if (write_dy) tile_to_global(bufB, LDB, P.dfeat, m0, D);
  if (tid < TM) {
    Ray ray; int n, i; float z, p[3], v[3], gvd[3];
    row_geometry(a, row_s(tid), MS, ray, n, i, z, p);
    row_view_dir(a, row_s(tid), MS, ray, v);
    const float* ge = bufB + tid * LDB + D;
    encode_bwd<4>(v, [&](int k) { return ge[k]; }, gvd);
    P.gv[m0 + tid] = make_float4(gvd[0], gvd[1], gvd[2], 0.f);
  }
  // 4. g_h8 = g_feat @ Wf + g_s * w_sigma
  tile_gemm<NJ, true, 0, false>(bufB, LDB, D, w + nnb::W_FEAT(D), D, D, D, nullptr, bufA, LDB, Ws);
  __syncthreads();
  for (int idx = tid; idx < TM * D; idx += 256) {
    int row = idx / D, k = idx % D;
    bufA[row * LDB + k] += gyc[row * 4 + 3] * __ldg(w + nnb::W_SIG(D) + k);
  }
  __syncthreads();
  // 5. trunk
  float* X = bufA; float* Y = bufB;
  for (int l = 7; l >= 0; --l) {
    for (int idx = tid; idx < TM * (D / 4); idx += 256) {
      int row = idx / (D / 4), c4 = idx % (D / 4); size_t m = m0 + row;
      float4 hv = *reinterpret_cast<const float4*>(P.h[l] + m * D + c4 * 4);
      float4* xp = reinterpret_cast<float4*>(X + row * LDB + c4 * 4);
      float4 g = *xp;
      g.x = hv.x > 0.f ? g.x : 0.f; g.y = hv.y > 0.f ? g.y : 0.f; g.z = hv.z > 0.f ? g.z : 0.f; g.w = hv.w > 0.f ? g.w : 0.f;
      *xp = g;
      if (write_dy) *reinterpret_cast<float4*>(P.dy[l] + m * D + c4 * 4) = g;
    }
    __syncthreads();
    if (l == 0) {
      tile_gemm<1, true, 0, true>(X, LDB, D, w + nnb::w_off(D, 0), 63, 63, D, nullptr, genc, 64, Ws);
    } else {
      tile_gemm<NJ, true, 0, false>(X, LDB, D, w + nnb::w_off(D, l), nnb::w_ld(D, l), D, D, nullptr, Y, LDB, Ws);
      if (l == 4) tile_gemm<1, true, 0, false>(X, LDB, D, w + nnb::w_off(D, 4) + D, D + 63, 63, D, nullptr, genc, 64, Ws);
      float* t_ = X; X = Y; Y = t_;
    }
    __syncthreads();
  }
  // 6. encoding adjoint
  if (tid < TM) {
    Ray ray; int n, i; float z, p[3], gp[3];
    row_geometry(a, row_s(tid), MS, ray, n, i, z, p);
    const float* ge = genc + tid * 64;
    encode_bwd<10>(p, [&](int k) { return ge[k]; }, gp);
    P.gp[m0 + tid] = make_float4(gp[0], gp[1], gp[2], 0.f);
  }
}

template <int D>
__global__ void __launch_bounds__(256, 1) simt_mlp_dgrad(nnb_render_args a, SimtPtrs P, size_t M, int write_dy) {
  simt_dgrad_tile<D>(a, P, M, write_dy, blockIdx.x);
}

// the chain of one reverse round of nnb_render_frame_bwd on this engine, on chunk k's stash (M = R N rows, R = min(S, 32))
template <int D>
__global__ void __launch_bounds__(256, 1) simt_dgrad_chunk(nnb_render_args a, SimtPtrs P, size_t M, int write_dy, int k) {
  simt_dgrad_tile<D, DG_CHUNK>(a, P, M, write_dy, blockIdx.x, k);
}

// the chain of nnb_render_bwd_tmin_engine on this engine on the packed stash of cap rows, over its first counts[C] rows (clamped to
// 0..cap), read when the kernel starts; a CTA past them exits before any barrier
template <int D>
__global__ void __launch_bounds__(256, 1) simt_dgrad_pack(nnb_render_args a, SimtPtrs P, size_t cap, int write_dy, int C,
                                                          const int* __restrict__ counts, const int* __restrict__ lists) {
  const size_t M = min((size_t)max(counts[C], 0), cap);
  if ((size_t)blockIdx.x * TM >= M) return;
  simt_dgrad_tile<D, DG_PACK>(a, P, M, write_dy, blockIdx.x, C, lists, counts);
}

// Device-count form of simt_mlp_dgrad (the normals of nnb_geometry_frame on this engine), rows as in simt_mlp_fwd_n: the chain on the
// stash simt_mlp_fwd_n wrote, without the dY stash.  A CTA past the n rows exits before any barrier.
template <int D>
__global__ void __launch_bounds__(256, 1) simt_mlp_dgrad_n(nnb_render_args a, SimtPtrs P, const int* __restrict__ count, int off, int cap) {
  const int n = min(*count - off, cap);
  if ((int)blockIdx.x * TM >= n) return;
  simt_dgrad_tile<D>(a, P, (size_t)n, 0, blockIdx.x);
}

// ---------------------------------------------------------------------------------------
// H: second-order field backward (nnb_field_hvp, DESIGN.md §4).  For a cotangent u on n = d s / d p, s' = u . n is the derivative
// of the logit along u: the tangent chain e' = J_enc(p) u, z'_l = W_l x'_{l-1} (no bias; [h'3 | e'] into layer 4), h'_l = [h_l > 0] z'_l,
// s' = w_sigma . h'7.  The ReLU masks are piecewise constant, so d s' / d W_l = dy_l (x) x'_{l-1} with dy_l the gated output gradient
// of the data-gradient chain for a cotangent 1 on the logit, d s' / d w_sigma = h'7, no bias term, and d s' / d p only the encoding's
// own second derivative.
// ---------------------------------------------------------------------------------------
struct TangentPtrs {
  float* th[8]; float* tenc;   // tangent stash [Mpad][D] / [Mpad][64]
  const float4* u;             // [M] cotangent on n (xyz)
  float4* gp;                  // [M] d s' / d p, or nullptr
};

// cotangent (0, 0, 0, 1) on out_rgba: 1 on the logit (NNB_RAW_DENSITY)
__global__ void logit_seed(float4* gs, size_t M) {
  const size_t m = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (m < M) gs[m] = make_float4(0.f, 0.f, 0.f, 1.f);
}

// one 64-row tile: e' and h'0..h'7 into the tangent stash (whole tile, Mpad rows), then delta_enc = dy4 W4[:, D:] + dy0 W0 (the data-
// gradient kernel's order) and the point term, written for rows m < M only.  Reads the stash of simt_mlp_fwd (h) and simt_mlp_dgrad (dy).
template <int D>
__global__ void __launch_bounds__(256, 1) simt_field_tangent(nnb_render_args a, SimtPtrs P, TangentPtrs T, size_t M) {
  constexpr int LDB = ldb<D>(), NJ = D / 64;
  extern __shared__ __align__(16) float smem[];
  float* buf0 = smem; float* buf1 = buf0 + TM * LDB; float* Ws = buf1 + TM * LDB;
  float* genc = Ws + 2 * KC * WS_LD;          // [64][64]
  const int tid = threadIdx.x;
  const size_t m0 = (size_t)blockIdx.x * TM;
  const float* w = a.weights;
  {  // 1. e' = J_enc(p) u into columns D..D+63 of both buffers (tail rows: u = 0)
    const int row = tid & 63, part = tid >> 6;
    const size_t m = m0 + row;
    Ray ray; int n, i; float z, p[3];
    row_geometry(a, m, M, ray, n, i, z, p);
    const float4 uv = m < M ? T.u[m] : make_float4(0.f, 0.f, 0.f, 0.f);
    const float u[3] = {uv.x, uv.y, uv.z};
    float* e0 = buf0 + row * LDB + D; float* e1 = buf1 + row * LDB + D;
    if (part == 0) {
#pragma unroll
      for (int c = 0; c < 3; ++c) { e0[c] = u[c]; e1[c] = u[c]; }
      e0[63] = 0.f; e1[63] = 0.f;
    }
    for (int l = part; l < 10; l += 4) {
      const float f = (float)(1 << l);
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        float s, co; sincosf(__fmul_rn(f, p[c]), &s, &co);
        const float ds = __fmul_rn(__fmul_rn(f, co), u[c]), dc = -__fmul_rn(__fmul_rn(f, s), u[c]);   // d sin(f p) / d p, d cos(f p) / d p
        e0[3 + 6 * l + c] = ds; e1[3 + 6 * l + c] = ds; e0[6 + 6 * l + c] = dc; e1[6 + 6 * l + c] = dc;
      }
    }
  }
  __syncthreads();
  for (int idx = tid; idx < TM * 16; idx += 256) {
    const int row = idx >> 4, c4 = idx & 15;
    *reinterpret_cast<float4*>(T.tenc + (m0 + row) * 64 + c4 * 4) = *reinterpret_cast<const float4*>(buf0 + row * LDB + D + c4 * 4);
  }
  // 2. h'_l = [h_l > 0] (W_l x'_{l-1}), the forward's layer loop without bias
  float* cur = buf0; float* oth = buf1;
  for (int l = 0; l < 8; ++l) {
    const float* in = (l == 0) ? cur + D : cur;
    const int K = (l == 0) ? 64 : (l == 4 ? D + 64 : D);
    const int kvalid = (l == 0) ? 63 : (l == 4 ? D + 63 : D);
    tile_gemm<NJ, false, 0, false>(in, LDB, K, w + nnb::w_off(D, l), nnb::w_ld(D, l), D, kvalid, nullptr, oth, LDB, Ws);
    __syncthreads();
    for (int idx = tid; idx < TM * (D / 4); idx += 256) {
      const int row = idx / (D / 4), c4 = idx % (D / 4); const size_t m = m0 + row;
      const float4 hv = *reinterpret_cast<const float4*>(P.h[l] + m * D + c4 * 4);
      float4* xp = reinterpret_cast<float4*>(oth + row * LDB + c4 * 4);
      float4 g = *xp;
      g.x = hv.x > 0.f ? g.x : 0.f; g.y = hv.y > 0.f ? g.y : 0.f; g.z = hv.z > 0.f ? g.z : 0.f; g.w = hv.w > 0.f ? g.w : 0.f;
      *xp = g;
      *reinterpret_cast<float4*>(T.th[l] + m * D + c4 * 4) = g;
    }
    __syncthreads();
    float* t_ = cur; cur = oth; oth = t_;
  }
  if (!T.gp) return;
  // 3. delta_enc = d s / d enc from the dy stash: dy4 into buf0, dy0 into buf1
  for (int idx = tid; idx < TM * (D / 4); idx += 256) {
    const int row = idx / (D / 4), c4 = idx % (D / 4); const size_t m = m0 + row;
    *reinterpret_cast<float4*>(buf0 + row * LDB + c4 * 4) = *reinterpret_cast<const float4*>(P.dy[4] + m * D + c4 * 4);
    *reinterpret_cast<float4*>(buf1 + row * LDB + c4 * 4) = *reinterpret_cast<const float4*>(P.dy[0] + m * D + c4 * 4);
  }
  __syncthreads();
  tile_gemm<1, true, 0, false>(buf0, LDB, D, w + nnb::w_off(D, 4) + D, D + 63, 63, D, nullptr, genc, 64, Ws);
  tile_gemm<1, true, 0, true>(buf1, LDB, D, w + nnb::w_off(D, 0), 63, 63, D, nullptr, genc, 64, Ws);
  __syncthreads();
  // 4. d s' / d p_c = -u_c sum_l f^2 (delta_sin sin(f p_c) + delta_cos cos(f p_c)), f = 2^l; the identity columns contribute nothing
  if (tid < TM && m0 + tid < M) {
    const size_t m = m0 + tid;
    Ray ray; int n, i; float z, p[3];
    row_geometry(a, m, M, ray, n, i, z, p);
    const float4 uv = T.u[m];
    const float u[3] = {uv.x, uv.y, uv.z};
    const float* ge = genc + tid * 64;
    float gp[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float acc = 0.f;
      for (int l = 0; l < 10; ++l) {
        const float f = (float)(1 << l);
        float s, co; sincosf(__fmul_rn(f, p[c]), &s, &co);
        acc = fmaf(__fmul_rn(f, f), fmaf(ge[3 + 6 * l + c], s, __fmul_rn(ge[6 + 6 * l + c], co)), acc);
      }
      gp[c] = -__fmul_rn(acc, u[c]);
    }
    T.gp[m] = make_float4(gp[0], gp[1], gp[2], 0.f);
  }
}

// ---------------------------------------------------------------------------------------
// B3: weight gradients.  dW[n][k] += sum_m dY[m][n] X[m][k]
// ---------------------------------------------------------------------------------------
struct WJob {
  const float* dY; const float* X; float* dW; float* db;
  int ldy, Nn, ldx, Kk, ldw, tiles_k, tile_start, ntiles;
  size_t part_off;   // this job's partials in the split buffer
};
struct WJobs { WJob j[16]; int njobs; };

// split blockIdx.y of job j writes its partial dW / db to part (layout of RedJob; wgrad_reduce sums the splits in order)
__device__ __forceinline__ void simt_wgrad_body(const WJobs& jobs, size_t M, int msplit, float* part) {
  __shared__ __align__(16) float Ys[16][64];
  __shared__ __align__(16) float Xs[16][64];
  int ji = 0;
  while (ji + 1 < jobs.njobs && (int)blockIdx.x >= jobs.j[ji + 1].tile_start) ++ji;
  const WJob& J = jobs.j[ji];
  int t = blockIdx.x - J.tile_start;
  int tn = t / J.tiles_k, tk = t % J.tiles_k;
  int n0 = tn * 64, k0 = tk * 64;
  size_t chunk = (M + msplit - 1) / msplit; chunk = (chunk + 15) / 16 * 16;
  size_t mb = (size_t)blockIdx.y * chunk, me = mb + chunk < M ? mb + chunk : M;
  const int tid = threadIdx.x, ni = tid >> 4, ki = tid & 15;
  float acc[4][4] = {}, bs[4] = {};
  for (size_t mc = mb; mc < me; mc += 16) {
    for (int idx = tid; idx < 16 * 64; idx += 256) {
      int mm = idx >> 6, c = idx & 63; size_t m = mc + mm;
      Ys[mm][c] = (m < me && n0 + c < J.Nn) ? __ldg(J.dY + m * J.ldy + n0 + c) : 0.f;
      Xs[mm][c] = (m < me && k0 + c < J.Kk) ? __ldg(J.X + m * J.ldx + k0 + c) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int mm = 0; mm < 16; ++mm) {
      float4 y = *reinterpret_cast<const float4*>(&Ys[mm][ni * 4]);
      float4 x = *reinterpret_cast<const float4*>(&Xs[mm][ki * 4]);
      float yv[4] = {y.x, y.y, y.z, y.w}, xv[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        bs[r] += yv[r];
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[r][c] = fmaf(yv[r], xv[c], acc[r][c]);
      }
    }
    __syncthreads();
  }
  float* pp = part + J.part_off + (size_t)blockIdx.y * ((size_t)J.Nn * J.Kk + J.Nn);
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    int n = n0 + ni * 4 + r;
    if (n >= J.Nn) continue;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      int k = k0 + ki * 4 + c;
      if (k < J.Kk) pp[(size_t)n * J.Kk + k] = acc[r][c];
    }
    if (tk == 0 && ki == 0) pp[(size_t)J.Nn * J.Kk + n] = bs[r];
  }
  if (blockIdx.x == gridDim.x - 1 && blockIdx.y == gridDim.y - 1) pdl_wait();   // chained launch: see tc_wgrad_all
}
__global__ void __launch_bounds__(256) simt_wgrad(WJobs jobs, size_t M, int msplit, float* part) { simt_wgrad_body(jobs, M, msplit, part); }
// simt_wgrad on the first *mrows rows (clamped to 0..cap), read on the device, at simt_wgrad_msplit of that count (at most the launch's
// gridDim.y splits): the splits past it store zeros, so at *mrows = M the partials are simt_wgrad's at M
__global__ void __launch_bounds__(256) simt_wgrad_live(WJobs jobs, size_t cap, float* part, const int* __restrict__ mrows) {
  const size_t M = min((size_t)max(*mrows, 0), cap);
  const int msplit = min(max((int)((M + 4095) / 4096), 1), min((int)gridDim.y, 16));
  simt_wgrad_body(jobs, M, msplit, part);
}

// The head jobs of the TC engine's weight-gradient stage (fc_density, fc_rgb: 1 and 3 rows of dW; the direction slice of
// rgb_layers.0: 27 columns), at the arithmetic of simt_wgrad: per element acc = fmaf(y, x, acc) from 0 over its split's samples in
// increasing order, the bias in the same order, the same splits and partial layout.  They are narrow, so they read 0.29 GB at C2 size
// for 0.6 GFLOP, and simt_wgrad's 64 x 64 tiles would stage and discard 63 of 64 dY columns (or most X columns).  Here a CTA is one
// split of one job with all of its Nn x Kk outputs: one thread streams the split's rows, which are contiguous, into a HW_NSTG-deep
// shared-memory ring with cp.async.bulk (whole dY and X rows, completion on an mbarrier), and thread t owns column k = t % KW
// (KW = Kk rounded up to a power of two >= 32) and RN rows starting at RN (t / KW).  Warps release a slot through a second mbarrier.
struct HJob { const float* dY; const float* X; int ldy, yoff, Nn, ldx, Kk, kw, rn; size_t part_off; };
struct HJobs { HJob j[4]; int njobs; };
constexpr int HW_CH = 16, HW_NSTG = 4, HW_MAX_LDX = 256, HW_MAX_LDY = 128;        // samples per chunk, ring depth, row limits
constexpr int HW_SY = HW_CH * HW_MAX_LDX * 4, HW_STG = HW_SY + HW_CH * HW_MAX_LDY * 4;   // slot: X [CH][ldx] | dY [CH][ldy]
constexpr int HW_SMEM = HW_NSTG * HW_STG + 2 * HW_NSTG * 8;

template <int RN>
__device__ __forceinline__ void head_wgrad_split(const HJob& J, size_t mb, size_t me, float* pp, unsigned char* smem) {
  using namespace tcu;
  const int tid = threadIdx.x, k = tid % J.kw, n0 = (tid / J.kw) * RN;
  const int nv = J.Nn - n0 < RN ? J.Nn - n0 : RN;   // rows of this thread (<= 0: none)
  const bool kv = k < J.Kk, bias = k < nv;   // column k valid; this thread sums the bias of row n0 + k
  const int nch = mb < me ? (int)((me - mb + HW_CH - 1) / HW_CH) : 0;
  const uint32_t bar0 = smem_u32(smem + HW_NSTG * HW_STG);
  auto FULL = [&](int i) { return bar0 + 8u * i; };
  auto EMPTY = [&](int i) { return bar0 + 8u * (HW_NSTG + i); };
  const float* ybase = J.dY - J.yoff;   // 16-byte aligned rows
  auto issue = [&](int c) {
    const size_t s0 = mb + (size_t)c * HW_CH;
    const uint32_t rows = (uint32_t)(me - s0 < (size_t)HW_CH ? me - s0 : HW_CH);
    const uint32_t bx = rows * J.ldx * 4, by = rows * J.ldy * 4, sl = c % HW_NSTG;
    mbar_expect_tx(FULL(sl), bx + by);
    bulk_g2s(smem_u32(smem + sl * HW_STG), J.X + s0 * J.ldx, bx, FULL(sl));
    bulk_g2s(smem_u32(smem + sl * HW_STG + HW_SY), ybase + s0 * J.ldy, by, FULL(sl));
  };
  if (tid == 0) {
    for (int i = 0; i < HW_NSTG; ++i) { mbar_init(FULL(i), 1); mbar_init(EMPTY(i), blockDim.x / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    for (int c = 0; c < HW_NSTG && c < nch; ++c) issue(c);
  }
  __syncthreads();
  float acc[RN], bsum = 0.f;
#pragma unroll
  for (int r = 0; r < RN; ++r) acc[r] = 0.f;
  for (int c = 0; c < nch; ++c) {
    const int sl = c % HW_NSTG;
    if (tid == 0 && c > 0 && c - 1 + HW_NSTG < nch) {   // refill the slot of chunk c - 1 once every warp has released it
      mbar_wait(EMPTY((c - 1) % HW_NSTG), (uint32_t)((c - 1) / HW_NSTG) & 1u);
      issue(c - 1 + HW_NSTG);
    }
    mbar_wait(FULL(sl), (uint32_t)(c / HW_NSTG) & 1u);
    const size_t s0 = mb + (size_t)c * HW_CH;
    const int rows = me - s0 < (size_t)HW_CH ? (int)(me - s0) : HW_CH;
    const float* sx = reinterpret_cast<const float*>(smem + sl * HW_STG) + k;
    const float* sy = reinterpret_cast<const float*>(smem + sl * HW_STG + HW_SY) + J.yoff + n0;
    if (nv > 0) {
#pragma unroll 2
      for (int i = 0; i < rows; ++i) {
        const float* yr = sy + i * J.ldy;
        if (kv) {
          const float x = sx[i * J.ldx];
          float y[RN];
          if constexpr (RN >= 4) {   // 16-byte aligned: yoff = 0 and n0 a multiple of RN (launch_head_wgrad)
#pragma unroll
            for (int q = 0; q < RN / 4; ++q) {
              const float4 v = reinterpret_cast<const float4*>(yr)[q];
              y[4 * q] = v.x; y[4 * q + 1] = v.y; y[4 * q + 2] = v.z; y[4 * q + 3] = v.w;
            }
          } else {
#pragma unroll
            for (int r = 0; r < RN; ++r) y[r] = r < nv ? yr[r] : 0.f;
          }
#pragma unroll
          for (int r = 0; r < RN; ++r)
            if (r < nv) acc[r] = fmaf(y[r], x, acc[r]);
        }
        bsum += yr[bias ? k : 0];   // lane k < nv: the bias of row n0 + k
      }
    }
    __syncwarp();
    if ((tid & 31) == 0) mbar_arrive(EMPTY(sl));
  }
#pragma unroll
  for (int r = 0; r < RN; ++r)
    if (r < nv && kv) pp[(size_t)(n0 + r) * J.Kk + k] = acc[r];
  if (bias) pp[(size_t)J.Nn * J.Kk + n0 + k] = bsum;
}

// grid (msplit, jobs): split blockIdx.x of job blockIdx.y; chained launch as simt_wgrad
__device__ __forceinline__ void head_wgrad_body(const HJobs& jobs, size_t M, int msplit, float* part) {
  extern __shared__ __align__(128) unsigned char hsmem[];
  const HJob& J = jobs.j[blockIdx.y];
  size_t chunk = (M + msplit - 1) / msplit; chunk = (chunk + 15) / 16 * 16;
  const size_t mb = (size_t)blockIdx.x * chunk, me = mb + chunk < M ? mb + chunk : M;
  float* pp = part + J.part_off + (size_t)blockIdx.x * ((size_t)J.Nn * J.Kk + J.Nn);
  switch (J.rn) {
    case 1: head_wgrad_split<1>(J, mb, me, pp, hsmem); break;
    case 2: head_wgrad_split<2>(J, mb, me, pp, hsmem); break;
    case 4: head_wgrad_split<4>(J, mb, me, pp, hsmem); break;
    case 8: head_wgrad_split<8>(J, mb, me, pp, hsmem); break;
    default: head_wgrad_split<16>(J, mb, me, pp, hsmem); break;
  }
  if (blockIdx.x == gridDim.x - 1 && blockIdx.y == gridDim.y - 1) pdl_wait();   // chained launch: see tc_wgrad_all
}
__global__ void __launch_bounds__(256) head_wgrad(const __grid_constant__ HJobs jobs, size_t M, int msplit, float* part) {
  head_wgrad_body(jobs, M, msplit, part);
}
// head_wgrad on the first min(32 *mcount, M) rows (the live rays of a reverse round of nnb_render_frame_train_bwd_tmin), read on the
// device, at the launch's split count: the splits past those rows store zeros, and at *mcount = M / 32 the splits are head_wgrad's
__global__ void __launch_bounds__(256) head_wgrad_live(const __grid_constant__ HJobs jobs, size_t M, int msplit, float* part,
                                                       const int* __restrict__ mcount) {
  const size_t m = (size_t)max(*mcount, 0) * 32;
  head_wgrad_body(jobs, m < M ? m : M, msplit, part);
}

// dW[n][k] += sum over splits (fixed order); one thread per element of all jobs
struct RedJobs { RedJob j[16]; int e0[17]; int njobs; };
__global__ void wgrad_reduce(RedJobs J, const float* __restrict__ part) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= J.e0[J.njobs]) return;
  int ji = 0;
  while (ji + 1 < J.njobs && e >= J.e0[ji + 1]) ++ji;
  const RedJob r = J.j[ji];
  const int le = e - J.e0[ji], nk = r.Nn * r.Kk;
  float s = 0.f;
  if (le < nk) {
    for (int y = 0; y < r.nsplit; ++y) s += part[r.off + (size_t)y * r.stride + le];
    r.dW[(size_t)(le / r.Kk) * r.ldw + le % r.Kk] += s;
  } else {
    for (int y = 0; y < r.nsplit; ++y)
      for (int q = 0; q < r.dbslots; ++q) s += part[r.off + (size_t)y * r.stride + nk + (size_t)q * r.Nn + (le - nk)];
    r.db[le - nk] += s;
  }
}

// ---------------------------------------------------------------------------------------
// B4: per-ray geometry adjoint (SURVEY.md A.6)
// ---------------------------------------------------------------------------------------
// per ray: red[0..8] d R, [9..11] d t, [12,13] d kx, ky, [14,15] d scale, shift -> rayred[n][16]; ray_reduce sums over the rays
__global__ void ray_bwd(nnb_render_bwd_args b, const SampleRec* recs, const float4* gp, const float4* gv, float* rayred) {
  const nnb_render_args& a = b.fwd;
  const int lane = threadIdx.x & 31, n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (n < a.N) {
    Ray r; setup_ray(a, n, r);
    float so[3] = {0, 0, 0}, sd[3] = {0, 0, 0}, sv[3] = {0, 0, 0};
    for (int i = lane; i < a.S; i += 32) {
      size_t m = (size_t)n * a.S + i;
      float4 g = gp[m], v = gv[m]; float z = recs[m].z;
      so[0] += g.x; so[1] += g.y; so[2] += g.z;
      sd[0] += z * g.x; sd[1] += z * g.y; sd[2] += z * g.z;
      sv[0] += v.x; sv[1] += v.y; sv[2] += v.z;
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) { so[c] = warp_sum(so[c]); sd[c] = warp_sum(sd[c]); sv[c] = warp_sum(sv[c]); }
    if (lane == 0) {
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
  }
}

// warp k sums rayred[.][k] over the rays in a fixed order and adds the total to its gradient: one add per output and call, so within
// the call nothing can reorder.  The add is atomic so that other work (the reference-image stage on a forked stream) may add into the
// same buffers at the same time and the sum stays correct; it is reproducible bit for bit when that work is ordered after this call,
// as the Trainer does (model/training.py, _GraphStep.body_a: the stage's stream waits for the whole backward).
__global__ void ray_reduce(nnb_render_bwd_args b, const float* __restrict__ rayred) {
  const nnb_render_args& a = b.fwd;
  const int k = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float s = 0.f;
  for (int n = lane; n < a.N; n += 32) s += rayred[(size_t)n * 16 + k];
  s = warp_sum(s);
  if (lane == 0) {
    if (k < 9) atomicAdd(b.g_c2w + 4 * (k / 3) + (k % 3), s);
    else if (k < 12) atomicAdd(b.g_c2w + 4 * (k - 9) + 3, s);
    else if (k == 12) { if (b.g_cam) atomicAdd(b.g_cam + 0, s); }
    else if (k == 13) { if (b.g_cam) atomicAdd(b.g_cam + 5, s); }
    else if (b.g_scale_shift && !a.depth) atomicAdd(b.g_scale_shift + (k - 14), s);
  }
}

SimtPtrs make_ptrs(const WsLayout& L, void* ws) {
  char* base = static_cast<char*>(ws);
  SimtPtrs P{};
  P.rec = reinterpret_cast<SampleRec*>(base + L.rec);
  P.gs = reinterpret_cast<float4*>(base + L.gs); P.gp = reinterpret_cast<float4*>(base + L.gp); P.gv = reinterpret_cast<float4*>(base + L.gv);
  for (int l = 0; l < 8; ++l) { P.h[l] = reinterpret_cast<float*>(base + L.h[l]); P.dy[l] = reinterpret_cast<float*>(base + L.dy[l]); }
  P.feat = reinterpret_cast<float*>(base + L.feat); P.hr = reinterpret_cast<float*>(base + L.hr);
  P.enc = reinterpret_cast<float*>(base + L.enc); P.denc = reinterpret_cast<float*>(base + L.denc);
  P.dfeat = reinterpret_cast<float*>(base + L.dfeat); P.dyr = reinterpret_cast<float*>(base + L.dyr);
  P.dyc = reinterpret_cast<float4*>(base + L.dyc);
  P.rayred = reinterpret_cast<float*>(base + L.rayred); P.wpart = reinterpret_cast<float*>(base + L.wpart);
  return P;
}

template <int D> constexpr size_t fwd_smem() { return (2 * TM * ldb<D>() + 2 * KC * WS_LD) * sizeof(float); }
template <int D> constexpr size_t bwd_smem() { return fwd_smem<D>() + (TM * 64 + TM * 4) * sizeof(float); }

}  // namespace

// entry points used by nnb_api.cu ------------------------------------------------------
template <int D>
static cudaError_t simt_init_dim() {
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(simt_mlp_fwd<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fwd_smem<D>());
    if (e != cudaSuccess) return e;
    e = cudaFuncSetAttribute(simt_mlp_dgrad<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bwd_smem<D>());
    if (e != cudaSuccess) return e;
    e = cudaFuncSetAttribute(simt_field_tangent<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bwd_smem<D>());
    if (e != cudaSuccess) return e;
    e = cudaFuncSetAttribute(simt_mlp_fwd_n<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fwd_smem<D>());
    if (e == cudaSuccess) e = cudaFuncSetAttribute(simt_mlp_dgrad_n<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bwd_smem<D>());
    if (e == cudaSuccess) e = cudaFuncSetAttribute(simt_march<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fwd_smem<D>());
    if (e == cudaSuccess) e = cudaFuncSetAttribute(simt_secant<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fwd_smem<D>());
    if (e == cudaSuccess) e = cudaFuncSetAttribute(simt_frame<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fwd_smem<D>());
    if (e == cudaSuccess) e = cudaFuncSetAttribute(simt_frame_stash<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fwd_smem<D>());
    if (e == cudaSuccess) e = cudaFuncSetAttribute(simt_dgrad_chunk<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bwd_smem<D>());
    if (e == cudaSuccess) e = cudaFuncSetAttribute(simt_stash_pack<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fwd_smem<D>());
    if (e == cudaSuccess) e = cudaFuncSetAttribute(simt_dgrad_pack<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bwd_smem<D>());
    if (e != cudaSuccess) return e;
    attr = true;
  }
  return cudaSuccess;
}
static cudaError_t simt_init() {
  cudaError_t e = simt_init_dim<256>();
  if (e == cudaSuccess) e = simt_init_dim<128>();
  if (e == cudaSuccess) e = simt_init_dim<64>();
  return e;
}
// the MLP kernels of width L.D (the width was validated by nnb_api.cu)
static void launch_mlp_fwd(const nnb_render_args& a, const SimtPtrs& P, const WsLayout& L, int stash, cudaStream_t st) {
  const int tiles = (int)((L.M + TM - 1) / TM);
  if (L.D == 128) simt_mlp_fwd<128><<<tiles, 256, fwd_smem<128>(), st>>>(a, P, L.M, stash);
  else if (L.D == 64) simt_mlp_fwd<64><<<tiles, 256, fwd_smem<64>(), st>>>(a, P, L.M, stash);
  else simt_mlp_fwd<256><<<tiles, 256, fwd_smem<256>(), st>>>(a, P, L.M, stash);
}
static void launch_mlp_dgrad(const nnb_render_args& a, const SimtPtrs& P, const WsLayout& L, int write_dy, cudaStream_t st) {
  const int tiles = (int)((L.M + TM - 1) / TM);
  if (L.D == 128) simt_mlp_dgrad<128><<<tiles, 256, bwd_smem<128>(), st>>>(a, P, L.M, write_dy);
  else if (L.D == 64) simt_mlp_dgrad<64><<<tiles, 256, bwd_smem<64>(), st>>>(a, P, L.M, write_dy);
  else simt_mlp_dgrad<256><<<tiles, 256, bwd_smem<256>(), st>>>(a, P, L.M, write_dy);
}

cudaError_t simt_render_fwd(const nnb_render_args& a, const WsLayout& L, cudaStream_t st) {
  SimtPtrs P = make_ptrs(L, a.workspace);
  cudaError_t e0 = simt_init();
  if (e0 != cudaSuccess) return e0;
  nnb_prof_mark(st); nnb_prof_mark(st);
  launch_mlp_fwd(a, P, L, (a.flags & NNB_STASH) ? 1 : 0, st);
  nnb_prof_mark(st);
  composite_fwd<<<(a.N + 7) / 8, 256, 0, st>>>(a, P.rec);
  nnb_prof_mark(st);
  return cudaGetLastError();
}

__global__ void rec_to_rgba(const SampleRec* rec, float4* out, size_t M) {
  size_t m = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (m < M) out[m] = make_float4(rec[m].r, rec[m].g, rec[m].b, rec[m].a);
}

cudaError_t simt_field_fwd(const nnb_render_args& a, const WsLayout& L, float* out_rgba, cudaStream_t st) {
  SimtPtrs P = make_ptrs(L, a.workspace);
  cudaError_t e0 = simt_init();
  if (e0 != cudaSuccess) return e0;
  launch_mlp_fwd(a, P, L, (a.flags & NNB_STASH) ? 1 : 0, st);
  rec_to_rgba<<<(unsigned)((L.M + 255) / 256), 256, 0, st>>>(P.rec, reinterpret_cast<float4*>(out_rgba), L.M);
  return cudaGetLastError();
}

cudaError_t simt_wgrad_all(const SimtPtrs& P, const WsLayout& L, float* gw, cudaStream_t st, const int* mrows = nullptr);
cudaError_t run_simt_wgrad(WJobs& J, size_t M, int D, int msplit, float* part, cudaStream_t st, const int* mrows = nullptr);

// nnb_field_hvp: forward with stash, data-gradient chain for a cotangent 1 on the logit (dy stash), tangent chain + point term, then
// the weight-gradient jobs d s' / d W_l = sum_m dy_l[m] (x) x'_{l-1}[m] and d s' / d w_sigma = sum_m h'7[m] (no bias jobs).
// a.flags holds NNB_STASH | NNB_HVP | NNB_RAW_DENSITY (nnb_api.cu)
cudaError_t simt_field_hvp(const nnb_render_args& a, const WsLayout& L, const float* u, float* g_pts, float* g_weights, cudaStream_t st) {
  SimtPtrs P = make_ptrs(L, a.workspace);
  cudaError_t e = simt_init();
  if (e != cudaSuccess) return e;
  char* base = static_cast<char*>(a.workspace);
  TangentPtrs T{};
  for (int l = 0; l < 8; ++l) T.th[l] = reinterpret_cast<float*>(base + L.th[l]);
  T.tenc = reinterpret_cast<float*>(base + L.tenc);
  T.u = reinterpret_cast<const float4*>(u); T.gp = reinterpret_cast<float4*>(g_pts);
  launch_mlp_fwd(a, P, L, 1, st);
  logit_seed<<<(unsigned)((L.M + 255) / 256), 256, 0, st>>>(P.gs, L.M);
  launch_mlp_dgrad(a, P, L, 1, st);
  const int tiles = (int)((L.M + TM - 1) / TM);
  if (L.D == 128) simt_field_tangent<128><<<tiles, 256, bwd_smem<128>(), st>>>(a, P, T, L.M);
  else if (L.D == 64) simt_field_tangent<64><<<tiles, 256, bwd_smem<64>(), st>>>(a, P, T, L.M);
  else simt_field_tangent<256><<<tiles, 256, bwd_smem<256>(), st>>>(a, P, T, L.M);
  e = cudaGetLastError();
  if (e != cudaSuccess || !g_weights) return e;
  WJobs J{}; int nj = 0;
  auto add = [&](const float* dY, int ldy, int Nn, const float* X, int ldx, int Kk, float* dW, int ldw) {
    WJob& j = J.j[nj++];
    j.dY = dY; j.ldy = ldy; j.Nn = Nn; j.X = X; j.ldx = ldx; j.Kk = Kk; j.dW = dW; j.ldw = ldw; j.db = nullptr;
  };
  const int D = L.D;
  add(P.dy[0], D, D, T.tenc, 64, 63, g_weights + nnb::w_off(D, 0), 63);
  for (int l = 1; l < 8; ++l) {
    add(P.dy[l], D, D, T.th[l - 1], D, D, g_weights + nnb::w_off(D, l), nnb::w_ld(D, l));
    if (l == 4) add(P.dy[4], D, D, T.tenc, 64, 63, g_weights + nnb::w_off(D, 4) + D, D + 63);
  }
  add(reinterpret_cast<const float*>(P.dyc) + 3, 4, 1, T.th[7], D, D, g_weights + nnb::W_SIG(D), D);   // the logit's cotangent, 1
  J.njobs = nj;
  return run_simt_wgrad(J, L.M, D, simt_wgrad_msplit(L.M), P.wpart, st);
}

cudaError_t simt_field_bwd(const nnb_render_args& a, const WsLayout& L, const float* g_rgba, float* g_pts, float* g_dirs, float* g_weights,
                           cudaStream_t st) {
  SimtPtrs P = make_ptrs(L, a.workspace);
  cudaError_t e = simt_init();
  if (e != cudaSuccess) return e;
  e = cudaMemcpyAsync(P.gs, g_rgba, L.M * 16, cudaMemcpyDeviceToDevice, st);
  if (e != cudaSuccess) return e;
  launch_mlp_dgrad(a, P, L, g_weights ? 1 : 0, st);
  if (g_weights) { e = simt_wgrad_all(P, L, g_weights, st); if (e != cudaSuccess) return e; }
  if (g_pts) { e = cudaMemcpyAsync(g_pts, P.gp, L.M * 16, cudaMemcpyDeviceToDevice, st); if (e != cudaSuccess) return e; }
  if (g_dirs) { e = cudaMemcpyAsync(g_dirs, P.gv, L.M * 16, cudaMemcpyDeviceToDevice, st); if (e != cudaSuccess) return e; }
  return cudaGetLastError();
}

// ---- nnb_ray_march and nnb_geometry_frame on this engine (NNB_ENGINE_SIMT) -----------------------------------------------------------
// The march: run_ray_march (nnb_march.cuh) with simt_march rounds and simt_secant passes, persistent grids of every CTA the SMs hold.
// A point's occupancy is the exact forward's (simt_mlp_fwd's arithmetic, which does not depend on the tile or row that evaluates it), so
// depth, first and bracket are the bits of Renderer.ray_marching / secant over nnb_field_fwd on this engine.
size_t simt_ray_march_workspace(int N, int n_steps) { return march_layout_bytes(N, n_steps, 0).total; }

template <int D>
static cudaError_t simt_ray_march_dim(const nnb_ray_march_args& r, cudaStream_t st) {
  cudaError_t e = simt_init();
  if (e != cudaSuccess) return e;
  static int slots = 0;   // CTAs of simt_march resident on the device at once
  if (!slots) {
    int dev = 0, n_sm = 0, per_sm = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, simt_march<D>, 256, fwd_smem<D>());
    if (e != cudaSuccess) return e;
    slots = n_sm * (per_sm > 0 ? per_sm : 1);
  }
  const MarchWs w = march_layout_bytes(r.N, r.n_steps, 0);
  const int grid = r.N < slots ? r.N : slots, tiles = (r.N + TM - 1) / TM;
  return run_ray_march(
      r, w, D, st, [&](const nnb_render_args& a, const MarchPtrs& q) { simt_march<D><<<grid, 256, fwd_smem<D>(), st>>>(a, q, r.N); },
      [&](const nnb_render_args& a, const MarchPtrs& q) { simt_secant<D><<<tiles < slots ? tiles : slots, 256, fwd_smem<D>(), st>>>(a, q); });
}
cudaError_t simt_ray_march(const nnb_ray_march_args& r, int D, cudaStream_t st) {
  return D == 128 ? simt_ray_march_dim<128>(r, st) : (D == 64 ? simt_ray_march_dim<64>(r, st) : simt_ray_march_dim<256>(r, st));
}

// rgba[m] = the (r, g, b, a) of record m for the n = min(*count - off, cap) rows of simt_mlp_fwd_n
__global__ void rec_to_rgba_n(const SampleRec* __restrict__ rec, float4* __restrict__ out, const int* __restrict__ count, int off, int cap) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m < min(*count - off, cap)) out[m] = make_float4(rec[m].r, rec[m].g, rec[m].b, rec[m].a);
}

// Workspace of nnb_geometry_frame on this engine, every section 256-byte aligned: hit count | ray0, dir [N][3], far, depth [N] | compacted
// rows: surface points, view directions [N][3], pixel indices [N], normal cotangents [N], d logit / d p [Npad], colours [N] float4 | the
// march's workspace (N rays) | the fp32 stash of one pass of at most GEO_PASS compacted rows: records, h0..h7, feat, hr, enc, denc, the
// direction adjoint.  Npad = N rounded up to 64: the chain writes whole 64-row tiles of d logit / d p.
constexpr int GEO_PASS = 32768;
struct SimtGeoWs { size_t count, ray0, dir, far, depth, pts, vdir, pix, gs, gp, rgba, march, rec, h[8], feat, hr, enc, denc, gv, total; int cap; };
static SimtGeoWs simt_geo_layout(int N, int n_steps, int D) {
  SimtGeoWs w{};
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t o = off; off += align_up(bytes, 256); return o; };
  const size_t n = (size_t)N, npad = align_up(n, TM);
  w.cap = (int)(npad < (size_t)GEO_PASS ? npad : (size_t)GEO_PASS);
  const size_t c = (size_t)w.cap, d = (size_t)D;
  w.count = take(4);
  w.ray0 = take(n * 12); w.dir = take(n * 12); w.far = take(n * 4); w.depth = take(n * 4);
  w.pts = take(n * 12); w.vdir = take(n * 12); w.pix = take(n * 4); w.gs = take(n * 16); w.gp = take(npad * 16); w.rgba = take(n * 16);
  w.march = take(march_layout_bytes(N, n_steps, 0).total);
  w.rec = take(c * sizeof(SampleRec));
  for (int l = 0; l < 8; ++l) w.h[l] = take(c * d * 4);
  w.feat = take(c * d * 4); w.hr = take(c * d / 2 * 4); w.enc = take(c * 64 * 4); w.denc = take(c * 32 * 4); w.gv = take(c * 16);
  w.total = off;
  return w;
}
size_t simt_geometry_frame_workspace(int N, int n_steps, int D) { return simt_geo_layout(N, n_steps, D).total; }

// nnb_geometry_frame on this engine: geo_rays, the exact march, geo_compact, then per pass of at most GEO_PASS compacted rows the normals
// (simt_mlp_fwd_n with the stash and simt_mlp_dgrad_n: OfficialStaticNerf.gradient's nnb_field_fwd + nnb_field_bwd with NNB_RAW_DENSITY,
// no view directions, cotangent (0, 0, 0, 1)) and the surface colour (simt_mlp_fwd_n at (p, -dir): OfficialStaticNerf.forward's
// nnb_field_fwd), with the row count read on the device, and geo_shade.  Passes past the hit count exit at once.  Nothing is read back.
template <int D>
static cudaError_t simt_geometry_frame_dim(const nnb_geometry_args& g, cudaStream_t st) {
  cudaError_t e = simt_init();
  if (e != cudaSuccess) return e;
  const SimtGeoWs w = simt_geo_layout(g.N, g.n_steps, D);
  char* base = static_cast<char*>(g.workspace);
  auto F = [&](size_t off) { return reinterpret_cast<float*>(base + off); };
  auto F4 = [&](size_t off) { return reinterpret_cast<float4*>(base + off); };
  int* count = reinterpret_cast<int*>(base + w.count);
  e = cudaMemsetAsync(count, 0, 4, st);
  if (e != cudaSuccess) return e;
  const int blocks = (g.N + 255) / 256;
  geo_rays<<<blocks, 256, 0, st>>>(g.T, g.pixels, g.N, g.radius, F(w.ray0), F(w.dir), F(w.far), g.ray0, g.ray_dir, g.far_);
  nnb_ray_march_args r{};
  r.weights = g.weights; r.ray0 = F(w.ray0); r.ray_dir = F(w.dir); r.far_ = F(w.far); r.frac = g.frac;
  r.N = g.N; r.n_steps = g.n_steps; r.n_secant = g.n_secant; r.hidden_dim = D; r.near_ = g.near_; r.tau = g.tau;
  r.flags = g.flags; r.engine = NNB_ENGINE_SIMT; r.depth = F(w.depth);
  r.workspace = base + w.march; r.workspace_bytes = w.rec - w.march;
  e = simt_ray_march_dim<D>(r, st);
  if (e != cudaSuccess) return e;
  int* pix = reinterpret_cast<int*>(base + w.pix);
  geo_compact<<<blocks, 256, 0, st>>>(g.N, F(w.ray0), F(w.dir), F(w.depth), count, F(w.pts), F(w.vdir), pix, F4(w.gs), g.rgb, g.rgb_surf,
                                      g.depth, reinterpret_cast<float4*>(g.grad));
  SimtPtrs P{};
  P.rec = reinterpret_cast<SampleRec*>(base + w.rec);
  for (int l = 0; l < 8; ++l) P.h[l] = F(w.h[l]);
  P.feat = F(w.feat); P.hr = F(w.hr); P.enc = F(w.enc); P.denc = F(w.denc); P.gv = F4(w.gv);
  nnb_render_args a{};
  a.weights = g.weights; a.N = g.N; a.S = 1; a.hidden_dim = D; a.engine = NNB_ENGINE_SIMT;
  const uint32_t occ_flags = g.flags & (NNB_DIST_ALPHA | NNB_SOFTPLUS);
  const int grid = w.cap / TM;
  for (int off = 0; off < g.N; off += w.cap) {
    a.pts = F(w.pts) + 3 * (size_t)off; a.dirs = nullptr; a.flags = occ_flags | NNB_RAW_DENSITY | NNB_STASH;
    P.gs = F4(w.gs) + off; P.gp = F4(w.gp) + off;
    simt_mlp_fwd_n<D><<<grid, 256, fwd_smem<D>(), st>>>(a, P, count, off, w.cap, 1);
    simt_mlp_dgrad_n<D><<<grid, 256, bwd_smem<D>(), st>>>(a, P, count, off, w.cap);   // d logit / d p
    a.dirs = F(w.vdir) + 3 * (size_t)off; a.flags = occ_flags;
    simt_mlp_fwd_n<D><<<grid, 256, fwd_smem<D>(), st>>>(a, P, count, off, w.cap, 0);   // surface colour
    rec_to_rgba_n<<<(w.cap + 255) / 256, 256, 0, st>>>(P.rec, F4(w.rgba) + off, count, off, w.cap);
  }
  geo_shade<<<blocks, 256, 0, st>>>(g.T, count, pix, F4(w.gp), F4(w.rgba), g.rgb, g.rgb_surf, reinterpret_cast<float4*>(g.grad));
  return cudaGetLastError();
}
cudaError_t simt_geometry_frame(const nnb_geometry_args& g, int D, cudaStream_t st) {
  return D == 128 ? simt_geometry_frame_dim<128>(g, st) : (D == 64 ? simt_geometry_frame_dim<64>(g, st) : simt_geometry_frame_dim<256>(g, st));
}

// ---- nnb_render_frame on this engine: run_render_frame (nnb_frame.cuh) with one simt_frame round per 32-sample chunk, a persistent grid
// of every CTA the SMs hold.  A sample's (r, g, b, a) is simt_mlp_fwd's (the exact forward does not depend on the tile or row that
// evaluates it) and frame_step sums the lane terms in composite_fwd's order, so at t_min = 0 the outputs are nnb_render_fwd's bits.
size_t simt_render_frame_workspace(int N) { return frame_layout_bytes(N, 0).total; }

// the persistent grid of simt_frame for a: every CTA the SMs hold, at most one per tile (0 on an error, in *e)
template <int D>
static int simt_frame_grid(const nnb_render_args& a, cudaError_t* e) {
  *e = simt_init();
  if (*e != cudaSuccess) return 0;
  static int slots = 0;   // CTAs of simt_frame resident on the device at once
  if (!slots) {
    int dev = 0, n_sm = 0, per_sm = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
    *e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, simt_frame<D>, 256, fwd_smem<D>());
    if (*e != cudaSuccess) return 0;
    slots = n_sm * (per_sm > 0 ? per_sm : 1);
  }
  const int per = TM / (a.S < 32 ? a.S : 32), tiles = (a.N + per - 1) / per;
  return tiles < slots ? tiles : slots;
}

template <int D>
static cudaError_t simt_render_frame_dim(const nnb_render_args& a, float t_min, int* n_eval, float* t_final, cudaStream_t st) {
  cudaError_t e;
  const int grid = simt_frame_grid<D>(a, &e);
  if (e != cudaSuccess) return e;
  return run_render_frame(a, frame_layout_bytes(a.N, 0), t_min, n_eval, t_final, st,
                          [&](const FramePtrs& f) { simt_frame<D><<<grid, 256, fwd_smem<D>(), st>>>(a, f); });
}
cudaError_t simt_render_frame(const nnb_render_args& a, float t_min, int* n_eval, float* t_final, int D, cudaStream_t st) {
  return D == 128 ? simt_render_frame_dim<128>(a, t_min, n_eval, t_final, st)
       : D == 64  ? simt_render_frame_dim<64>(a, t_min, n_eval, t_final, st) : simt_render_frame_dim<256>(a, t_min, n_eval, t_final, st);
}

// ---- nnb_render_frame_bwd on this engine (nnb_render_frame_bwd_engine, nnb_render_frame_train_fwd_engine / _bwd_engine): the rounds of
// nnb_frame.cuh with the exact kernels.  The chunk stash packs R = min(S, 32) rows per ray (frame_chunk_adjoint<true>), so at S <= 32 it
// holds nnb_render_fwd's rows in nnb_render_fwd's order, and its weight-gradient stage has the stash path's M and split count.  Workspace:
// frame_bwd_layout_bytes without weight images, the chunk stash make_layout(N, R, NNB_STASH, NNB_ENGINE_SIMT, D).
static FrameBwdWs simt_frame_bwd_layout(int N, int S, int D) {
  return frame_bwd_layout_bytes(N, S, 0, make_layout(N, S < 32 ? S : 32, NNB_STASH, NNB_ENGINE_SIMT, D).total, 0);
}
size_t simt_render_frame_bwd_workspace(int N, int S, int D) { return simt_frame_bwd_layout(N, S, D).total; }

// The forward half: run_render_frame with simt_frame at t_min = 0 (every ray runs every round), the carry after each chunk but the last
// copied to the checkpoints.  It leaves the checkpoints in the workspace for the reverse half.
template <int D>
static cudaError_t simt_frame_train_fwd_dim(const nnb_render_args& a, cudaStream_t st) {
  cudaError_t e;
  const int grid = simt_frame_grid<D>(a, &e);
  if (e != cudaSuccess) return e;
  const int N = a.N, C = (a.S + 31) / 32;
  const FrameBwdWs w = simt_frame_bwd_layout(N, a.S, D);
  float* ckpt = reinterpret_cast<float*>(static_cast<char*>(a.workspace) + w.ckpt);
  cudaError_t ec = cudaSuccess;
  e = run_render_frame(a, w.f, 0.f, nullptr, nullptr, st, [&](const FramePtrs& f) {
    simt_frame<D><<<grid, 256, fwd_smem<D>(), st>>>(a, f);
    if (f.k + 1 < C && ec == cudaSuccess) ec = cudaMemcpyAsync(ckpt + (size_t)f.k * N, f.carry, (size_t)N * 4, cudaMemcpyDeviceToDevice, st);
  });
  return e == cudaSuccess ? ec : e;
}

// The reverse half: rounds k = C - 1 .. 0, each on the chunk stash: simt_frame_stash, frame_chunk_adjoint, simt_dgrad_chunk, (g_weights)
// simt_wgrad_all, whose reduce adds the round's dW into g_weights, and frame_ray_acc; then frame_ray_finish and ray_reduce.  Of what the
// forward half wrote it reads the checkpoints only (data, no index or counter), so a workspace the forward half did not fill gives wrong
// numbers, never an access outside the workspace.
template <int D>
static cudaError_t simt_frame_train_bwd_dim(const nnb_render_bwd_args& b, cudaStream_t st) {
  const nnb_render_args& a = b.fwd;
  cudaError_t e = simt_init();
  if (e != cudaSuccess) return e;
  const int N = a.N, C = (a.S + 31) / 32, R = a.S < 32 ? a.S : 32;
  const FrameBwdWs w = simt_frame_bwd_layout(N, a.S, D);
  char* base = static_cast<char*>(a.workspace);
  auto F = [&](size_t off) { return reinterpret_cast<float*>(base + off); };
  const WsLayout L = make_layout(N, R, NNB_STASH, NNB_ENGINE_SIMT, D);   // offsets from the chunk stash's own base
  const SimtPtrs P = make_ptrs(L, base + w.chunk);
  FrameBwdPtrs fb{};
  fb.rounds = C; fb.ckpt = F(w.ckpt); fb.suffix = F(w.suffix); fb.rec = P.rec;
  fb.gs = P.gs; fb.gp = P.gp; fb.gv = P.gv; fb.raypart = F(w.raypart);
  const int write_dy = b.g_weights ? 1 : 0, warps = (N + 7) / 8, tiles = (int)((L.M + TM - 1) / TM);
  for (int k = C - 1; k >= 0; --k) {
    FramePtrs f{};
    f.k = k;
    fb.k = k;
    simt_frame_stash<D><<<tiles, 256, fwd_smem<D>(), st>>>(a, P, f);
    frame_chunk_adjoint<true><<<warps, 256, 0, st>>>(b, fb);
    simt_dgrad_chunk<D><<<tiles, 256, bwd_smem<D>(), st>>>(a, P, L.M, write_dy, k);
    e = cudaGetLastError();
    if (e == cudaSuccess && b.g_weights) e = simt_wgrad_all(P, L, b.g_weights, st);
    if (e != cudaSuccess) return e;
    frame_ray_acc<true><<<warps, 256, 0, st>>>(a, fb);
  }
  frame_ray_finish<<<warps, 256, 0, st>>>(b, F(w.raypart), P.rayred);
  ray_reduce<<<1, 512, 0, st>>>(b, P.rayred);
  return cudaGetLastError();
}

cudaError_t simt_render_frame_train_fwd(const nnb_render_args& a, int D, cudaStream_t st) {
  return D == 128 ? simt_frame_train_fwd_dim<128>(a, st) : (D == 64 ? simt_frame_train_fwd_dim<64>(a, st) : simt_frame_train_fwd_dim<256>(a, st));
}
cudaError_t simt_render_frame_train_bwd(const nnb_render_bwd_args& b, int D, cudaStream_t st) {
  return D == 128 ? simt_frame_train_bwd_dim<128>(b, st) : (D == 64 ? simt_frame_train_bwd_dim<64>(b, st) : simt_frame_train_bwd_dim<256>(b, st));
}
// nnb_render_frame_bwd_engine on this engine: the two halves in sequence
cudaError_t simt_render_frame_bwd(const nnb_render_bwd_args& b, int D, cudaStream_t st) {
  const cudaError_t e = simt_render_frame_train_fwd(b.fwd, D, st);
  return e != cudaSuccess ? e : simt_render_frame_train_bwd(b, D, st);
}

// ---- nnb_render_fwd_tmin_engine / nnb_render_bwd_tmin_engine on this engine: the tensor-core pair's rounds (tc_render_tmin_fwd_dim /
// _bwd_dim) with the exact kernels, on the packed stash of pack_round_base.  Workspace, every section 256-byte aligned: the packed stash
// make_layout(C 64 ceil(R N / 64), 1, NNB_STASH, NNB_ENGINE_SIMT, D) at offset 0 (every ray in every round) | carry, chunk counts [N] |
// lane partials [N][5][32] | checkpoints [C - 1][N] | lists [C][N] | counts [C + 1] | ray lane partials [N][9][32].  No weight images:
// the exact kernels read the fp32 weights.
struct PackWs { WsLayout L; size_t carry, chunks, part, ckpt, lists, counts, raypart, total; };
static PackWs simt_pack_layout(int N, int S, int D) {
  PackWs w{};
  const int C = (S + 31) / 32, R = S < 32 ? S : 32;
  const size_t n = (size_t)N;
  w.L = make_layout((int)((size_t)C * TM * (((size_t)R * n + TM - 1) / TM)), 1, NNB_STASH, NNB_ENGINE_SIMT, D);
  size_t off = w.L.total;
  auto take = [&](size_t bytes) { const size_t o = off; off += align_up(bytes, 256); return o; };
  w.carry = take(n * 4); w.chunks = take(n * 4); w.part = take(n * 640); w.ckpt = take((size_t)(C - 1) * n * 4);
  w.lists = take((size_t)C * n * 4); w.counts = take((size_t)(C + 1) * 4); w.raypart = take(n * 288 * 4);
  w.total = off;
  return w;
}
size_t simt_render_tmin_workspace(int N, int S, int D) { return simt_pack_layout(N, S, D).total; }

// the forward: rounds k = 0 .. C - 1 of frame_live_list (round k's list from the chunk counts), simt_stash_pack (chunk k of the listed rays
// with the training stash) and simt_pack_step (frame_step's compositing and stop rule); then frame_finish.  Every launch after the first
// sizes itself from device counts; nothing is read back.
template <int D>
static cudaError_t simt_tmin_fwd_dim(const nnb_frame_args& fa, cudaStream_t st) {
  const nnb_render_args& a = fa.fwd;
  cudaError_t e = simt_init();
  if (e != cudaSuccess) return e;
  const int N = a.N, C = (a.S + 31) / 32, R = a.S < 32 ? a.S : 32;
  const PackWs w = simt_pack_layout(N, a.S, D);
  char* base = static_cast<char*>(a.workspace);
  auto I = [&](size_t off) { return reinterpret_cast<int*>(base + off); };
  const SimtPtrs P = make_ptrs(w.L, base);
  int *lists = I(w.lists), *counts = I(w.counts);
  FramePtrs f{};
  f.t_min = fa.t_min;
  f.carry = reinterpret_cast<float*>(base + w.carry); f.chunks = I(w.chunks); f.part = reinterpret_cast<float*>(base + w.part);
  float* ckpt = reinterpret_cast<float*>(base + w.ckpt);
  const int tiles = (R * N + TM - 1) / TM, warps = (N + 7) / 8;
  for (int k = 0; k < C; ++k) {
    f.k = k; f.list = lists + (size_t)k * N; f.count = counts + k;
    frame_live_list<<<1, 1024, 0, st>>>(f.chunks, N, k, C, lists + (size_t)k * N, counts + k);
    simt_stash_pack<D><<<tiles, 256, fwd_smem<D>(), st>>>(a, P, f);
    simt_pack_step<<<warps, 256, 0, st>>>(a, f, P.rec, ckpt, C);
  }
  frame_finish<<<warps, 256, 0, st>>>(a, f, fa.n_eval, fa.t_final);
  return cudaGetLastError();
}

// the backward: the C lists again from the chunk counts (clamped to 1..C); simt_pack_adjoint (every ray's compositing adjoint, padding
// cotangents, the row count); simt_dgrad_pack on those rows; with g_weights, one weight-gradient stage on them (simt_wgrad_live, the
// jobs of simt_wgrad_all); simt_pack_ray_acc, frame_ray_finish and ray_reduce.  Of what the forward wrote it reads the chunk counts, the
// checkpoints and the stash, so a backward without its forward gives wrong numbers, never an access outside the workspace.
template <int D>
static cudaError_t simt_tmin_bwd_dim(const nnb_render_bwd_args& b, cudaStream_t st) {
  const nnb_render_args& a = b.fwd;
  cudaError_t e = simt_init();
  if (e != cudaSuccess) return e;
  const int N = a.N, C = (a.S + 31) / 32;
  const PackWs w = simt_pack_layout(N, a.S, D);
  const WsLayout& L = w.L;
  char* base = static_cast<char*>(a.workspace);
  auto F = [&](size_t off) { return reinterpret_cast<float*>(base + off); };
  auto I = [&](size_t off) { return reinterpret_cast<int*>(base + off); };
  const SimtPtrs P = make_ptrs(L, base);
  const int* chunks = I(w.chunks);
  int *lists = I(w.lists), *counts = I(w.counts);
  for (int k = 0; k < C; ++k) frame_live_list<<<1, 1024, 0, st>>>(chunks, N, k, C, lists + (size_t)k * N, counts + k);
  FrameBwdPtrs fb{};
  fb.rounds = C; fb.ckpt = F(w.ckpt); fb.rec = P.rec; fb.gs = P.gs; fb.gp = P.gp; fb.gv = P.gv; fb.raypart = F(w.raypart);
  const int warps = (N + 7) / 8;
  simt_pack_adjoint<<<(N + 2 * C + 7) / 8, 256, 0, st>>>(b, fb, chunks, lists, counts);
  simt_dgrad_pack<D><<<(unsigned)(L.M / TM), 256, bwd_smem<D>(), st>>>(a, P, L.M, b.g_weights ? 1 : 0, C, counts, lists);
  e = cudaGetLastError();
  if (e == cudaSuccess && b.g_weights) e = simt_wgrad_all(P, L, b.g_weights, st, counts + C);
  if (e != cudaSuccess) return e;
  simt_pack_ray_acc<<<warps, 256, 0, st>>>(a, fb, chunks, lists, counts);
  frame_ray_finish<<<warps, 256, 0, st>>>(b, F(w.raypart), P.rayred);
  ray_reduce<<<1, 512, 0, st>>>(b, P.rayred);
  return cudaGetLastError();
}
cudaError_t simt_render_fwd_tmin(const nnb_frame_args& f, int D, cudaStream_t st) {
  return D == 128 ? simt_tmin_fwd_dim<128>(f, st) : (D == 64 ? simt_tmin_fwd_dim<64>(f, st) : simt_tmin_fwd_dim<256>(f, st));
}
cudaError_t simt_render_bwd_tmin(const nnb_render_bwd_args& b, int D, cudaStream_t st) {
  return D == 128 ? simt_tmin_bwd_dim<128>(b, st) : (D == 64 ? simt_tmin_bwd_dim<64>(b, st) : simt_tmin_bwd_dim<256>(b, st));
}

// jobs -> simt_wgrad into part[off ..]; R[i] receives job i's reduction (launch_wgrad_reduce).  chained: programmatic dependent
// launch behind the previous grid on the stream (see tc_wgrad_all).  mrows (not NULL): simt_wgrad_live on the first *mrows of M rows
cudaError_t launch_simt_wgrad(WJobs& J, size_t M, int D, int msplit, float* part, size_t off, RedJob* R, bool chained, cudaStream_t st,
                              const int* mrows = nullptr) {
  int tiles = 0;
  for (int i = 0; i < J.njobs; ++i) {
    WJob& j = J.j[i];
    j.tiles_k = (j.Kk + 63) / 64; j.ntiles = ((j.Nn + 63) / 64) * j.tiles_k; j.tile_start = tiles; tiles += j.ntiles;
    const size_t stride = (size_t)j.Nn * j.Kk + j.Nn;
    R[i] = RedJob{j.dW, j.db, j.Nn, j.Kk, j.ldw, msplit, j.db ? 1 : 0, off, stride};
    j.part_off = off;
    off += stride * msplit;
  }
  if (off > wpart_floats(M, D)) return cudaErrorInvalidValue;
  cudaLaunchAttribute at{};
  at.id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at.val.programmaticStreamSerializationAllowed = 1;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(tiles, msplit); cfg.blockDim = dim3(256); cfg.stream = st;
  cfg.attrs = &at; cfg.numAttrs = chained ? 1 : 0;
  cudaError_t e = mrows ? cudaLaunchKernelEx(&cfg, simt_wgrad_live, J, M, part, mrows)
                        : cudaLaunchKernelEx(&cfg, simt_wgrad, J, M, msplit, part);
  return e != cudaSuccess ? e : cudaGetLastError();
}

// jobs -> simt_wgrad into the partial buffer, then wgrad_reduce into dW / db
cudaError_t run_simt_wgrad(WJobs& J, size_t M, int D, int msplit, float* part, cudaStream_t st, const int* mrows) {
  RedJob R[16];
  cudaError_t e = launch_simt_wgrad(J, M, D, msplit, part, 0, R, false, st, mrows);
  if (e != cudaSuccess) return e;
  return launch_wgrad_reduce(R, J.njobs, part, st);
}

// the head jobs of tc_wgrad_all -> head_wgrad at jobs_wgrad_msplit(M) splits, launched chained into part[off ..] (njobs <= 4); the
// caller reduces them through R.  mcount (not NULL): head_wgrad_live on min(32 *mcount, M) rows
cudaError_t launch_head_wgrad(const SmallJob* jobs, int njobs, size_t M, int D, float* part, size_t off, RedJob* R, cudaStream_t st,
                              const int* mcount) {
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(head_wgrad, cudaFuncAttributeMaxDynamicSharedMemorySize, HW_SMEM);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(head_wgrad_live, cudaFuncAttributeMaxDynamicSharedMemorySize, HW_SMEM);
    if (e != cudaSuccess) return e;
    attr = true;
  }
  if (njobs > 4) return cudaErrorInvalidValue;
  const int msplit = jobs_wgrad_msplit(M);
  HJobs J{};
  for (int i = 0; i < njobs; ++i) {
    const SmallJob& s = jobs[i];
    // rows are staged whole by bulk copies: 16-byte aligned rows of 16-byte multiples (dY from its aligned row start)
    const int yoff = (int)((reinterpret_cast<uintptr_t>(s.dY) % 16) / 4);
    int kw = 32, rn = 1;
    while (kw < s.Kk) kw *= 2;
    while (rn * (256 / (kw < 256 ? kw : 256)) < s.Nn) rn *= 2;
    if (kw > 256 || rn > 16 || s.ldx > HW_MAX_LDX || s.ldx % 4 || reinterpret_cast<uintptr_t>(s.X) % 16 || s.ldy > HW_MAX_LDY ||
        s.ldy % 4 || yoff + s.Nn > s.ldy || (rn >= 4 && yoff != 0))
      return cudaErrorInvalidValue;
    J.j[i] = HJob{s.dY, s.X, s.ldy, yoff, s.Nn, s.ldx, s.Kk, kw, rn, off};
    const size_t stride = (size_t)s.Nn * s.Kk + s.Nn;
    R[i] = RedJob{s.dW, s.db, s.Nn, s.Kk, s.ldw, msplit, s.db ? 1 : 0, off, stride};
    off += stride * msplit;
  }
  if (off > wpart_floats(M, D)) return cudaErrorInvalidValue;
  J.njobs = njobs;
  cudaLaunchAttribute at{};
  at.id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at.val.programmaticStreamSerializationAllowed = 1;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(msplit, njobs); cfg.blockDim = dim3(256); cfg.dynamicSmemBytes = HW_SMEM; cfg.stream = st;
  cfg.attrs = &at; cfg.numAttrs = 1;
  cudaError_t e = mcount ? cudaLaunchKernelEx(&cfg, head_wgrad_live, J, M, msplit, part, mcount)
                         : cudaLaunchKernelEx(&cfg, head_wgrad, J, M, msplit, part);
  return e != cudaSuccess ? e : cudaGetLastError();
}

cudaError_t launch_composite_fwd(const nnb_render_args& a, const SampleRec* recs, cudaStream_t st) {
  composite_fwd<<<(a.N + 7) / 8, 256, 0, st>>>(a, recs);
  return cudaGetLastError();
}

// mrows (not NULL): every job on the first *mrows of L.M rows, read on the device (simt_wgrad_live)
cudaError_t simt_wgrad_all(const SimtPtrs& P, const WsLayout& L, float* gw, cudaStream_t st, const int* mrows) {
  {
    WJobs J{}; int nj = 0;
    auto add = [&](const float* dY, int ldy, int Nn, const float* X, int ldx, int Kk, float* dW, int ldw, float* db) {
      WJob& j = J.j[nj++];
      j.dY = dY; j.ldy = ldy; j.Nn = Nn; j.X = X; j.ldx = ldx; j.Kk = Kk; j.dW = dW; j.ldw = ldw; j.db = db;
    };
    const int D = L.D, DR = D / 2;
    add(P.dy[0], D, D, P.enc, 64, 63, gw + nnb::w_off(D, 0), 63, gw + nnb::b_off(D, 0));
    for (int l = 1; l < 8; ++l) {
      add(P.dy[l], D, D, P.h[l - 1], D, D, gw + nnb::w_off(D, l), nnb::w_ld(D, l), gw + nnb::b_off(D, l));
      if (l == 4) add(P.dy[4], D, D, P.enc, 64, 63, gw + nnb::w_off(D, 4) + D, D + 63, nullptr);
    }
    add(reinterpret_cast<const float*>(P.dyc) + 3, 4, 1, P.h[7], D, D, gw + nnb::W_SIG(D), D, gw + nnb::B_SIG(D));
    add(P.dfeat, D, D, P.h[7], D, D, gw + nnb::W_FEAT(D), D, gw + nnb::B_FEAT(D));
    add(P.dyr, DR, DR, P.feat, D, D, gw + nnb::W_RGBH(D), D + 27, gw + nnb::B_RGBH(D));
    add(P.dyr, DR, DR, P.denc, 32, 27, gw + nnb::W_RGBH(D) + D, D + 27, nullptr);
    add(reinterpret_cast<const float*>(P.dyc), 4, 3, P.hr, DR, DR, gw + nnb::W_RGB(D), DR, gw + nnb::B_RGB(D));
    J.njobs = nj;
    return run_simt_wgrad(J, L.M, D, simt_wgrad_msplit(L.M), P.wpart, st, mrows);
  }
}

// the weight-gradient stage of simt_render_bwd alone, on whatever the stash holds (nnb_debug_wgrad)
cudaError_t simt_wgrad_stage(const nnb_render_args& a, const WsLayout& L, float* gw, cudaStream_t st) {
  return simt_wgrad_all(make_ptrs(L, a.workspace), L, gw, st);
}

// ray_reduce of rayred [N][16] into b's pose, camera and scale / shift gradients (nnb_render_frame_bwd)
cudaError_t launch_ray_reduce(const nnb_render_bwd_args& b, const float* rayred, cudaStream_t st) {
  ray_reduce<<<1, 512, 0, st>>>(b, rayred);
  return cudaGetLastError();
}

cudaError_t launch_wgrad_reduce(const RedJob* jobs, int njobs, const float* part, cudaStream_t st) {
  RedJobs J{};
  J.njobs = njobs < 16 ? njobs : 16;
  J.e0[0] = 0;
  for (int i = 0; i < J.njobs; ++i) { J.j[i] = jobs[i]; J.e0[i + 1] = J.e0[i] + jobs[i].Nn * jobs[i].Kk + (jobs[i].db ? jobs[i].Nn : 0); }
  wgrad_reduce<<<(J.e0[J.njobs] + 255) / 256, 256, 0, st>>>(J, part);
  return cudaGetLastError();
}

cudaError_t simt_render_bwd_with(const nnb_render_bwd_args& b, const WsLayout& L, cudaStream_t st, DgradFn dgrad, WgradFn wgrad);
cudaError_t simt_render_bwd(const nnb_render_bwd_args& b, const WsLayout& L, cudaStream_t st) { return simt_render_bwd_with(b, L, st, nullptr, nullptr); }

// dgrad / wgrad: the data- / weight-gradient stages (nullptr: the fp32 SIMT kernels)
cudaError_t simt_render_bwd_with(const nnb_render_bwd_args& b, const WsLayout& L, cudaStream_t st, DgradFn dgrad, WgradFn wgrad) {
  const nnb_render_args& a = b.fwd;
  SimtPtrs P = make_ptrs(L, a.workspace);
  cudaError_t e0 = simt_init();
  if (e0 != cudaSuccess) return e0;
  nnb_prof_mark(st);
  composite_bwd<<<(a.N + 7) / 8, 256, 0, st>>>(b, P.rec, P.gs);
  nnb_prof_mark(st);
  const int write_dy = b.g_weights ? 1 : 0;
  if (dgrad) { cudaError_t ed = dgrad(b, L, write_dy, st); if (ed != cudaSuccess) return ed; }
  else launch_mlp_dgrad(a, P, L, write_dy, st);
  nnb_prof_mark(st);
  if (b.g_weights) {
    cudaError_t ew = wgrad ? wgrad(a, L, b.g_weights, st) : simt_wgrad_all(P, L, b.g_weights, st);
    if (ew != cudaSuccess) return ew;
  }
  nnb_prof_mark(st);
  ray_bwd<<<(a.N + 7) / 8, 256, 0, st>>>(b, P.rec, P.gp, P.gv, P.rayred);
  ray_reduce<<<1, 512, 0, st>>>(b, P.rayred);
  nnb_prof_mark(st);
  return cudaGetLastError();
}
