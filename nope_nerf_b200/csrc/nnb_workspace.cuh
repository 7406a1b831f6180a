// Workspace carving shared by both engines (caller-provided scratch, see nnb_workspace_bytes).
#pragma once
#include "nnb_common.cuh"

struct WsLayout {
  size_t M, Mpad;
  int D;        // hidden width of the field (64 | 128 | 256)
  // per-sample records
  size_t rec;   // SampleRec[Mpad]            (forward -> compositing / backward)
  size_t gs;    // float4[Mpad]  d/d(rgb_i, a_i) from compositing adjoint
  size_t gp;    // float4[Mpad]  d/d p_i
  size_t gv;    // float4[Mpad]  d/d viewdir_i
  // fixed-order reductions (no float atomics: a step's gradients are the same bits on every run)
  size_t rayred;   // float[N][16]  per-ray pose / intrinsics / scale-shift adjoints, summed over rays by ray_reduce
  size_t wpart;    // float[]       per-sample-split partial weight gradients, summed over the splits by wgrad_reduce
  // SIMT engine activation stash (fp32, [sample][feature]; D features per trunk layer, D / 2 of the rgb hidden layer)
  size_t h[8], feat, hr, enc, denc;
  size_t dy[8], dfeat, dyr, dyc;
  // second-order field backward (NNB_HVP, SIMT engine only): tangent stash of nnb_field_hvp, [sample][feature] like h / enc
  size_t th[8], tenc;
  // TC engine: ReLU gate bits (h > 0) of h0..h7 and the rgb hidden layer, written by tc_field_fwd, read by tc_dgrad (see gate_bits_off)
  size_t gates;
  size_t total;  // bytes
};

// weight-gradient stage of a backward that consumes the fp32 stash: accumulates every MLP parameter gradient into gw
typedef cudaError_t (*WgradFn)(const nnb_render_args& a, const WsLayout& L, float* gw, cudaStream_t st);
// data-gradient stage of such a backward: head adjoints, the chain through the MLP (dY stash when write_dy), d p and d viewdir
typedef cudaError_t (*DgradFn)(const nnb_render_bwd_args& b, const WsLayout& L, int write_dy, cudaStream_t st);

// job of the fp32 SIMT weight-gradient kernel: dW[n][k] += sum_m dY[m*ldy+n] X[m*ldx+k]
struct SmallJob { const float* dY; const float* X; float* dW; float* db; int ldy, Nn, ldx, Kk, ldw; };

__host__ __device__ inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// sample splits of the weight-gradient kernels (each split writes its own partial dW, see wgrad_reduce)
inline int simt_wgrad_msplit(size_t M) { int m = (int)((M + 4095) / 4096); return m < 1 ? 1 : (m > 16 ? 16 : m); }
inline int jobs_wgrad_msplit(size_t M) { int m = (int)((M + 2047) / 2048); return m < 1 ? 1 : (m > 64 ? 64 : m); }
// floats of the partial buffer that the small SIMT jobs use (one bias slot per row, jobs_wgrad_msplit splits)
inline size_t small_jobs_part_floats(const SmallJob* jobs, int njobs, size_t M) {
  size_t f = 0;
  for (int i = 0; i < njobs; ++i) f += (size_t)jobs[i].Nn * jobs[i].Kk + jobs[i].Nn;
  return f * jobs_wgrad_msplit(M);
}
// sample splits of tc_wgrad's D-wide jobs: 8 at D = 256, more at smaller widths (fewer row slices per job) to fill the SMs
inline int tc_wgrad_msplit_big(int D) { return 2048 / D; }
constexpr size_t WPART_PAD = 16 * 512;   // bias slots of every job (up to two per output row)
inline size_t wpart_floats(size_t M, int D) {
  const size_t np = (size_t)nnb::num_params(D);
  const size_t a = (size_t)simt_wgrad_msplit(M) * (np + WPART_PAD);
  const size_t b = (size_t)tc_wgrad_msplit_big(D) * (np + WPART_PAD);   // tc_wgrad: <= 2048 / D splits of the D-wide jobs, 32 of the encoding jobs
  const size_t c = (size_t)jobs_wgrad_msplit(M) * 8192;                 // small SIMT jobs
  return a > b ? (a > c ? a : c) : (b > c ? b : c);
}

// one weight-gradient job's partials: split y writes part[off + y * stride + e], e < Nn * Kk the dW element (n * Kk + k),
// then `dbslots` x Nn bias partials; wgrad_reduce adds sum_y (and sum over the slots) to dW[n * ldw + k] / db[n] in a fixed order
struct RedJob { float* dW; float* db; int Nn, Kk, ldw, nsplit, dbslots; size_t off, stride; };
cudaError_t launch_wgrad_reduce(const RedJob* jobs, int njobs, const float* part, cudaStream_t st);

// Programmatic dependent launch (PDL) of the TC engine's weight-gradient stage (see tc_wgrad_all).
// launch_dependents: once every CTA of this grid has issued it (or exited), the next grid on the stream may start, if that grid is
// launched with cudaLaunchAttributeProgrammaticStreamSerialization; otherwise it has no effect.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
// wait: blocks until the grid this one was launched behind has completed and its stores are visible; a no-op in a grid launched
// without that attribute.  A CTA blocked here keeps its SM, so the weight-gradient kernels let only their last CTA wait, after its
// partials are stored: that is enough to make the grid complete only after its predecessor has.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ReLU gate bits of the TC engine, in the order of the wgmma accumulator fragment, so that each consumer thread (0..255) of a
// 128-sample tile writes its bits with one vector store in tc_field_fwd and reads them with one vector load in tc_dgrad.
// Region `gates`: [layer 0..8][tile][thread][D/2 bits of a trunk layer (layers 0..7 = h0..h7) | D/4 bits of the rgb hidden layer
// (layer 8)].  Thread t (warp w = t / 32, lane) holds tile rows r0 = 64 (w / 4) + 16 (w % 4) + lane / 4 and r0 + 8, columns
// 8j + c0 + {0, 1} with c0 = 2 (lane % 4); its bit b = 4j + 2r + e is (h[row r0 + 8r][column 8j + c0 + e] > 0), stored most significant
// first: bit W - 1 - b % W of its little-endian W-bit word b / W, W = 32 (W = 16 for the 16 bits of the rgb hidden layer at D = 64).
__host__ __device__ inline size_t gate_bits_bytes(size_t Mpad, int D) { return Mpad * (size_t)D + Mpad * (size_t)D / 16; }
__host__ __device__ inline size_t gate_bits_off(int layer, size_t tile, int thread, size_t Mpad, int D) {
  return layer < 8 ? ((size_t)layer * (Mpad / 128) + tile) * (16 * (size_t)D) + (size_t)thread * (D / 16)
                   : Mpad * (size_t)D + tile * (8 * (size_t)D) + (size_t)thread * (D / 32);
}

inline WsLayout make_layout(int N, int S, uint32_t flags, int engine, int D = 256) {
  WsLayout L{};
  L.D = D;
  L.M = (size_t)N * S;
  L.Mpad = align_up(L.M, 128);
  size_t o = 0;
  auto take = [&](size_t bytes) { size_t r = o; o = align_up(o + bytes, 256); return r; };
  L.rec = take(L.Mpad * sizeof(SampleRec));
  if (flags & NNB_STASH) {
    L.gs = take(L.Mpad * 16); L.gp = take(L.Mpad * 16); L.gv = take(L.Mpad * 16);
    L.rayred = take((size_t)N * 16 * 4); L.wpart = take(wpart_floats(L.M, D) * 4);
    // fp32 [sample][feature] stash, written by the forward of either engine and read by the backward
    const size_t d = (size_t)D, dr = (size_t)(D / 2);
    for (int l = 0; l < 8; ++l) L.h[l] = take(L.Mpad * d * 4);
    L.feat = take(L.Mpad * d * 4); L.hr = take(L.Mpad * dr * 4);
    L.enc = take(L.Mpad * 64 * 4); L.denc = take(L.Mpad * 32 * 4);
    for (int l = 0; l < 8; ++l) L.dy[l] = take(L.Mpad * d * 4);
    L.dfeat = take(L.Mpad * d * 4); L.dyr = take(L.Mpad * dr * 4); L.dyc = take(L.Mpad * 16);
    if (engine == NNB_ENGINE_TC) L.gates = take(gate_bits_bytes(L.Mpad, D));
    if (engine == NNB_ENGINE_SIMT && (flags & NNB_HVP)) {   // Mpad rows: the SIMT kernels process whole 64-row tiles
      for (int l = 0; l < 8; ++l) L.th[l] = take(L.Mpad * d * 4);
      L.tenc = take(L.Mpad * 64 * 4);
    }
  }
  L.total = o;
  return L;
}
