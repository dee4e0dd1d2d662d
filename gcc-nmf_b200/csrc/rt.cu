// The real-time block path as ONE stream-ordered unit with no host synchronisation inside, capturable in a CUDA graph:
//   reference  gccNMF/realtime/gccNMFProcessor.py:201-231 (GCCNMFProcessor.processFrames), :245-270 (the Theano graph it runs),
//              gccNMF/realtime/utils.py:99-116 (OverlapAddProcessor.processFrames: 8-block input / output rings around it),
//              notebooks/onlineSpeechEnhancement.ipynb:433-438 (per-frame coefficient inference, the numInferenceIterations > 0 branch).
//
// One audio block = five small kernels (+ two per inference iteration), every intermediate in the caller-owned state buffer:
//   A  rt_analysis    per frame: window . samples (from the input ring, or from the caller's windowed frames) -> one complex FFT for
//                     the stereo pair (left + i right, Hermitian split) -> X (2, F, nT) complex64, PHAT coherence, realGCC
//                     G[t][d][f] = Re(coh[f] E[f][d]) (float32, as the Theano float32 graph), gccPHAT[d][t] = nanmean_f G, |X|
//   I  rt_inf_ratio / rt_inf_update   (inference_iterations > 0)  H-only KL updates with the fixed dictionary, all 2 nT columns
//   B  rt_atoms       gccNMF[d][k] = sum_f G[t][d][f] W[f][k] (float32) -> argmax over TDOA per atom -> atom mask (boxcar / window, float64)
//   C  rt_filter      tfMask[f][t] = (W . mask) / rowsum(W)   (or (W . (H mask)) / (W . H) per channel with inference); Y = tfMask X
//   D  rt_synthesis   per frame: Hermitian rebuild, inverse FFT of the stereo pair, x synthesis window
//   E  rt_ola_emit    overlap-add of the nT frames into the output ring in frame order, emits block [-3B, -2B), pushes the block into
//                     the input ring; one extra CTA keeps the GCC-PHAT history ring and the sliding-window localisation
//                     (argmax of the nanmean over the last `localization_window` columns -> target TDOA index of the NEXT block).
// The rings are circular in place (the reference shifts 8 blocks of memory per call); positions derive from a device-side block
// counter, so a captured graph replays unchanged block after block.
//
// Streams (slots).  One state buffer serves S independent audio streams that share the configuration, W, E, the windows and H0:
//   [ shared region: twiddles, windows, W, W^T, row / column sums, E^T, H0 ]  [ slot 0 ] [ slot 1 ] ... [ slot S-1 ]
// Each slot region (fixed stride) holds its RtDev (parameters, block counter, history index, target, `active`), its rings, its
// GCC-PHAT history and its per-block intermediates.  Every kernel of a block covers all S slots in one launch (a slot dimension in
// the grid, or several slots per warp where the dictionary is the operand to share), so the kernel count per block does not depend
// on S.  The single-stream entry points (gccnmf_rt_*) are the S = 1 case of the same carve and kernels.
// Equivalence: slot s of an S-slot state computes bit for bit what a single-stream state fed the same blocks computes.  Every
// reduction below has a fixed order that does not depend on the other slots or on the tile shape: rt_atoms is one fmaf chain per
// output over f = 0 .. F-1 from 0.f (zero padding appends fmaf(0, 0, acc) = acc), the argmax is a maximum under a strict total
// order (numpy's: NaN first, then value, then the lower index), and the inference / filter kernels sum lane-strided over the
// contracted index and then through the same xor butterfly for every slot.
// An inactive slot costs no work: its output slice is written as zeros, its input slice is ignored, its state is left as it was.
//
// Sources (gccnmf_rtsep_*, P >= 2 target TDOAs per slot, the reference's TARGET_MODE_MULTIPLE).  rt_atoms also keeps the P target
// rows gccNMF[tau_s][k] of its accumulators and gives every atom to the source whose value wins under rt_better: P one-hot masks.
// Each slot then carries P copies of the mask, Y, synthesis frames and output ring, one source region of fixed stride after
// another; filter, synthesis and emit run once per source (a source dimension in the grid), each source through the same code
// and order a single-target slot runs.  Analysis, inference, the input ring and the localisation run once per slot; with
// localisation on, the P largest peaks of the windowed GCC-PHAT mean become the targets of the next block.
//
// Bank (gccnmf_rtbank_*, the reference's per-processor dictionary size / type and microphone spacing, gccNMFProcessor.py:131-157).
// The shared region holds Qd dictionary entries (W, W^T, recV, colsumW, H0, each sized at K_max = cfg.num_atoms, entry i with its
// own K_i <= K_max) and Qe steering entries (E^T) at fixed strides, the K_i table and the slots sorted by dictionary (stable).
// Every slot region ends with the slot's (dictionary, steering) pair.  Each kernel reads the entries of its slot through one
// by-value RtBank argument; the empty bank (gccnmf_rt_*, rtm, rtsep) puts every slot on the layout's one dictionary and table.
// Slot s on (i, j) computes bit for bit what a single-stream state built with (W_i, E_j) computes: every per-output order
// depends only on the contracted index.  The inference and filter kernels run one slot per warp with a bank; rt_atoms takes its
// (slot, frame) pairs in dictionary order, so a CTA spans more than one entry only where the sorted order changes entry, and
// then runs its f loop once per entry.
#include <cmath>
#include <vector>

#include "common.cuh"
#include "fft.cuh"
#include "records.cuh"
#include "streams.cuh"

namespace {

constexpr int kRtMaxN = 2048;
constexpr int kRtMaxFrames = 8;          // frames per block the filter kernel keeps in registers
constexpr int kRtMaxD = 128;
constexpr int kRtRingBlocks = 8;         // utils.py:85 numBlocksPerBuffer
constexpr int kRtMaxStreams = 4096;      // slots per state buffer
constexpr int kRtAtomsFc = 32;           // f values per shared-memory stage of the atoms contraction
constexpr int kRtMaxSources = GCCNMF_RTSEP_MAX_SOURCES;
constexpr int kRtMaxBank = GCCNMF_RTBANK_MAX_ENTRIES;   // dictionary entries and steering entries, each

struct RtDev {                           // device-resident parameters + loop-carried state (first bytes of a slot region)
  float target, eps, beta, noise_floor;  // gccNMFProcessor.py:196-199 (Theano shared scalars)
  int mode, separation, localization, loc_window;
  int block_counter;                     // blocks completed (incremented by the synthesis kernel)
  int hist_index;                        // write position of the GCC-PHAT history ring (utils.py:45-59)
  int active;                            // 0: the slot is skipped by every kernel of a block
};

// Pointer of slot s given the pointer of slot 0 and the slot stride in bytes.
template <typename T>
__host__ __device__ __forceinline__ T* rt_slot(T* p0, int s, size_t stride) {
  return (T*)((const char*)p0 + (size_t)s * stride);
}

// Where the kernels find a slot's dictionary and steering entries.  All zero (the empty bank): every slot on entry 0 of K atoms.
struct RtBank {
  int32_t* assign;                       // slot 0's (dictionary, steering, K_i of the last block computed), slot-strided
  const int32_t* K;                      // K_i of every dictionary entry
  const int32_t* order;                  // the S slots sorted by dictionary index (stable)
  size_t dict_stride, steer_stride;      // bytes from one entry to the next (W, W^T, recV, colsumW, H0 / E^T)
};
__device__ __forceinline__ int2 rt_entry(const RtBank& b, int s, size_t stride) {
  return b.assign ? *reinterpret_cast<const int2*>(rt_slot(b.assign, s, stride)) : int2{0, 0};
}
__device__ __forceinline__ int rt_sorted_slot(const RtBank& b, int i) { return b.order ? b.order[i] : i; }
__device__ __forceinline__ int rt_atoms_of(const RtBank& b, int dict, int K) { return b.K ? b.K[dict] : K; }

struct RtLayout {                        // carve of the caller-owned state buffer (pure function of the configuration and S)
  // shared by every slot
  float *win_a, *win_s, *W, *WT, *recV, *colsumW, *H0, *tw32;
  double* tw64;
  float2* ET;
  // slot 0 (slot s: rt_slot(p, s, stride))
  RtDev* dev;
  float *in_ring, *out_ring, *G, *gccphat, *Vabs, *H, *R, *frames;
  double *hist, *hmask;
  float2 *X, *Y;
  int32_t* argmax;
  // what filter, synthesis and emit read and write per source: source q of slot s at rt_slot(rt_slot(p, s, stride), q, src_stride).
  // P = 0: the slot's own hmask, Y, frames and out_ring with src_stride 0.  P > 0: P source regions appended to the slot (the
  // slot's own four are then unused), plus the targets, the status word and the target rows gccNMF[tau_q] (P, K, nT).
  double* smask;
  float2* sY;
  float *sframes, *sout, *tval;
  int32_t *targets, *status;
  size_t src_stride;
  // Qd, Qe > 0: W .. H0 and ET above are entry 0 of the bank (entry i at rt_slot(p, i, bank.dict_stride) / bank.steer_stride),
  // bank_K (Qd), order (S) in the shared region, assign (2 per slot) at the end of every slot region.
  RtBank bank;
  int32_t *bank_K, *order, *assign;
  int Qd, Qe;
  int F, Fp, L, S, P, D;
  size_t stride, bytes;
  bool ok;
};

RtLayout rt_carve(const gccnmf_rt_config& c, int S, int P, void* state, size_t state_bytes, int Qd = 0, int Qe = 0) {
  RtLayout l{};
  const int N = c.window_size, nT = c.windows_per_block, K = c.num_atoms, D = c.num_tdoas;
  l.F = N / 2 + 1;
  l.Fp = (l.F + 3) & ~3;
  l.L = kRtRingBlocks * c.block_size;
  l.S = S;
  l.P = P;
  l.D = D;
  l.Qd = Qd;
  l.Qe = Qe;
  char* base = state ? static_cast<char*>(state) : reinterpret_cast<char*>(256);
  WorkspaceCarver w(base, ~size_t(0) >> 1);
  l.tw64 = w.take<double>(N);
  l.tw32 = w.take<float>(N);
  l.win_a = w.take<float>(N);
  l.win_s = w.take<float>(N);
  {                                      // the one dictionary, or entry 0 of Qd (each carved alike from a 256-aligned base)
    WorkspaceCarver u(w.take<char>(0), ~size_t(0) >> 1);
    l.W = u.take<float>((size_t)l.F * K);
    l.WT = u.take<float>((size_t)K * l.Fp);
    l.recV = u.take<float>(l.F);
    l.colsumW = u.take<float>(K);
    l.H0 = u.take<float>((size_t)K * 2);
    l.bank.dict_stride = Qd > 0 ? align_up(u.used, 256) : 0;
    w.take<char>(Qd > 0 ? Qd * l.bank.dict_stride : u.used);
  }
  l.ET = w.take<float2>((size_t)D * l.Fp);
  if (Qe > 0) {
    l.bank.steer_stride = align_up((size_t)D * l.Fp * sizeof(float2), 256);
    w.take<char>((size_t)(Qe - 1) * l.bank.steer_stride);
  }
  if (Qd > 0) {
    l.bank_K = w.take<int32_t>(kRtMaxBank);
    l.order = w.take<int32_t>(S);
  }
  const size_t shared = align_up(w.used, 256);
  WorkspaceCarver v(base + shared, ~size_t(0) >> 1);
  l.dev = v.take<RtDev>(1);
  l.hist = v.take<double>((size_t)D * c.history_length);
  l.hmask = v.take<double>((size_t)K * nT);
  l.in_ring = v.take<float>((size_t)2 * l.L);
  l.out_ring = v.take<float>((size_t)2 * l.L);
  l.G = v.take<float>((size_t)nT * D * l.Fp);
  l.gccphat = v.take<float>((size_t)D * nT);
  l.Vabs = v.take<float>((size_t)l.F * 2 * nT);
  l.H = v.take<float>((size_t)K * 2 * nT);
  l.R = v.take<float>((size_t)l.F * 2 * nT);
  l.frames = v.take<float>((size_t)2 * nT * N);
  l.X = v.take<float2>((size_t)2 * l.F * nT);
  l.Y = v.take<float2>((size_t)2 * l.F * nT);
  l.argmax = v.take<int32_t>((size_t)K * nT);
  l.smask = l.hmask;
  l.sY = l.Y;
  l.sframes = l.frames;
  l.sout = l.out_ring;
  if (P > 0) {
    l.targets = v.take<int32_t>(kRtMaxSources);
    l.status = v.take<int32_t>(1);
    l.tval = v.take<float>((size_t)P * K * nT);
    char* src0 = v.take<char>(0);
    WorkspaceCarver u(src0, ~size_t(0) >> 1);
    l.smask = u.take<double>((size_t)K * nT);
    l.sY = u.take<float2>((size_t)2 * l.F * nT);
    l.sframes = u.take<float>((size_t)2 * nT * N);
    l.sout = u.take<float>((size_t)2 * l.L);
    l.src_stride = align_up(u.used, 256);
    v.take<char>((size_t)P * l.src_stride);
  }
  if (Qd > 0) {
    l.assign = v.take<int32_t>(3);       // zeroed by init and reset_slots: entries (0, 0), no block computed yet
    l.bank.assign = l.assign;
    l.bank.K = l.bank_K;
    l.bank.order = l.order;
  }
  l.stride = align_up(v.used, 256);
  l.bytes = shared + (size_t)S * l.stride;
  l.ok = state != nullptr && S >= 1 && l.bytes <= state_bytes;
  return l;
}

int rt_check(gccnmf_handle* h, const gccnmf_rt_config* c, int S = 1, int P = 0) {
  GCCNMF_REQUIRE(h, c != nullptr, "rt: NULL configuration");
  GCCNMF_REQUIRE(h, S >= 1 && S <= kRtMaxStreams, "rt: num_streams must be in [1, %d] (got %d)", kRtMaxStreams, S);
  GCCNMF_REQUIRE(h, P == 0 || (P >= 2 && P <= kRtMaxSources), "rt: num_sources must be in [2, %d] (got %d)", kRtMaxSources, P);
  const int N = c->window_size;
  GCCNMF_REQUIRE(h, N >= 64 && N <= kRtMaxN && (N & (N - 1)) == 0, "rt: window_size must be a power of two in [64, %d] (got %d)", kRtMaxN, N);
  GCCNMF_REQUIRE(h, c->hop_size >= 1 && c->block_size >= 1, "rt: hop_size and block_size must be positive");
  GCCNMF_REQUIRE(h, c->windows_per_block >= 1 && c->windows_per_block <= kRtMaxFrames, "rt: windows_per_block must be in [1, %d] (got %d)", kRtMaxFrames,
                 c->windows_per_block);
  GCCNMF_REQUIRE(h, c->num_atoms >= 1 && c->num_tdoas >= 1, "rt: num_atoms and num_tdoas must be positive");
  if (c->num_tdoas > kRtMaxD) return gccnmf_fail(h, GCCNMF_ERR_UNSUPPORTED, "rt: num_tdoas %d > %d", c->num_tdoas, kRtMaxD);
  GCCNMF_REQUIRE(h, c->history_length >= 1 && c->inference_iterations >= 0, "rt: history_length must be positive, inference_iterations >= 0");
  // the windows of one block must lie inside the 8-block rings (utils.py:107)
  GCCNMF_REQUIRE(h, N + (c->windows_per_block - 1) * c->hop_size <= kRtRingBlocks * c->block_size && 3 * c->block_size <= kRtRingBlocks * c->block_size,
                 "rt: window_size + (windows_per_block - 1) hop_size exceeds the 8-block ring");
  return 0;
}

// A bank needs entries of both kinds (the empty bank is the rtm / rtsep layout).
int rt_check_bank(gccnmf_handle* h, int Qd, int Qe) {
  GCCNMF_REQUIRE(h, Qd >= 1 && Qd <= kRtMaxBank && Qe >= 1 && Qe <= kRtMaxBank,
                 "rtbank: num_dictionaries and num_steerings must be in [1, %d] (got %d, %d)", kRtMaxBank, Qd, Qe);
  return 0;
}

// ---------------------------------------------------------------------------------------------- init-time kernels
// K_out (bank entries): the entry's atom count, written for the kernels of the next blocks.
__global__ void rt_init_dictionary_kernel(const float* __restrict__ W, int F, int Fp, int K, float* __restrict__ WT, float* __restrict__ recV,
                                          float* __restrict__ colsumW, int32_t* __restrict__ K_out) {
  // one thread per atom: column sum in row order (numpy.sum(W, axis=0)) + transposed copy; one thread per bin: row sum
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (K_out && i == 0) *K_out = K;
  if (i < K) {
    float s = 0.f;
    for (int f = 0; f < Fp; ++f) {
      const float w = f < F ? W[(int64_t)f * K + i] : 0.f;
      WT[(int64_t)i * Fp + f] = w;
      if (f < F) s += w;
    }
    colsumW[i] = s;
  }
  if (i < F) {
    double s = 0.0;
    for (int k = 0; k < K; ++k) s += (double)W[(int64_t)i * K + k];
    recV[i] = (float)s;                  // tensor.sum(W, axis=-1) in float32 (gccNMFProcessor.py:268)
  }
}

__global__ void rt_init_steering_kernel(const float2* __restrict__ E, int F, int Fp, int D, float2* __restrict__ ET) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= D * Fp) return;
  const int d = i / Fp, f = i - d * Fp;
  ET[i] = f < F ? E[(int64_t)f * D + d] : float2{0.f, 0.f};
}

// Parameters of up to kRtParamsPerLaunch slots, passed by value (the host array is consumed when the launch is enqueued).
constexpr int kRtParamsPerLaunch = 64;
struct RtParamsBatch {
  gccnmf_rtm_slot_params p[kRtParamsPerLaunch];
};

// set_active = 0 leaves the slot's `active` flag alone (the single-stream entry point has no such parameter).
__global__ void rt_set_params_kernel(RtDev* dev0, size_t stride, int first, int count, RtParamsBatch b, int set_active) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  RtDev* dev = rt_slot(dev0, first + i, stride);
  const gccnmf_rtm_slot_params& q = b.p[i];
  if (q.set_target) dev->target = q.target_index;
  dev->eps = q.epsilon; dev->beta = q.beta; dev->noise_floor = q.noise_floor;
  dev->mode = q.mode; dev->separation = q.separation_enabled ? 1 : 0; dev->localization = q.localization_enabled ? 1 : 0;
  dev->loc_window = q.localization_window;
  if (set_active) dev->active = q.active ? 1 : 0;
}

// Defaults of gccNMFProcessor.py:190-199 and `active` for slots [first, first + count) (after their regions were zeroed); with P
// sources, targets spread evenly over the D TDOAs: floor((2 q + 1) D / (2 P)).
__global__ void rt_default_params_kernel(RtDev* dev0, size_t stride, int first, int count, int32_t* targets0, int P, int D) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  RtDev* dev = rt_slot(dev0, first + i, stride);
  dev->target = 10.0f; dev->eps = 2.0f; dev->beta = 1.0f; dev->noise_floor = 0.0f;
  dev->mode = 1; dev->separation = 1; dev->localization = 0; dev->loc_window = 6;
  dev->active = 1;
  for (int q = 0; q < P; ++q) rt_slot(targets0, first + i, stride)[q] = (2 * q + 1) * D / (2 * P);
}

// ---------------------------------------------------------------------------------------------- numerics shared with gcc.cu
// numpy / Theano complex64 arithmetic of  X0 * conj(X1) / |X0| / |X1|  (gccNMFProcessor.py:253; runGCCNMF.py:44)
__device__ __forceinline__ float2 rt_coherence(float2 a, float2 b) {
  float re = __fadd_rn(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y));
  float im = __fsub_rn(__fmul_rn(a.y, b.x), __fmul_rn(a.x, b.y));
  const float ma = (float)sqrt((double)a.x * a.x + (double)a.y * a.y);
  const float mb = (float)sqrt((double)b.x * b.x + (double)b.y * b.y);
  const float ia = 1.0f / ma, ib = 1.0f / mb;
  re = __fmul_rn(re, ia); im = __fmul_rn(im, ia);
  re = __fmul_rn(re, ib); im = __fmul_rn(im, ib);
  return float2{re, im};
}
// numpy.argmax ordering: NaN is a maximum, the first occurrence wins.  A strict total order on (value, index) pairs, so the
// argmax is the same whatever order the candidates are compared in.
__device__ __forceinline__ bool rt_better(float v, int i, float bv, int bi) {
  const bool vn = v != v, bn = bv != bv;
  if (vn || bn) return vn && (!bn || i < bi);
  return v > bv || (v == bv && i < bi);
}
__device__ __forceinline__ bool rt_better64(double v, int i, double bv, int bi) {
  const bool vn = v != v, bn = bv != bv;
  if (vn || bn) return vn && (!bn || i < bi);
  return v > bv || (v == bv && i < bi);
}

// Logical ring position p of the reference's 8-block buffers (0 = oldest sample, L - 1 = newest) AFTER the shift of call number
// `call` (1-based) -> physical index: the sample stream position is call * B - L + p.
__device__ __forceinline__ int rt_ring_index(int p, int call, int B, int L) {
  long long a = (long long)call * B - L + p;
  a %= L;
  return (int)(a < 0 ? a + L : a);
}

// ---------------------------------------------------------------------------------------------- A: analysis (one CTA per frame and slot)
__global__ void __launch_bounds__(kFftThreads)
rt_analysis_kernel(const RtDev* __restrict__ dev0, size_t stride, const float* __restrict__ windowed,   // (S, 2, N, nT) or NULL: ring + new block
                   const float* __restrict__ in_blocks, const float* __restrict__ in_ring0, int B, int L, int hop, int nT,
                   const float* __restrict__ win_a, const double2* __restrict__ tw, int N, int log2n, const float2* __restrict__ ET, int D, int Fp,
                   float2* __restrict__ X0, float* __restrict__ G0, float* __restrict__ gccphat0, float* __restrict__ Vabs0,
                   const float* __restrict__ H0, float* __restrict__ Hs0, int K, int inference, RtBank bank) {
  __shared__ double2 fft[kRtMaxN];
  __shared__ float2 coh[kRtMaxN / 2 + 1];
  const int t = blockIdx.x, s = blockIdx.y, F = N / 2 + 1;
  const RtDev* dev = rt_slot(dev0, s, stride);
  if (!dev->active) return;
  const int2 entry = rt_entry(bank, s, stride);      // the slot's steering table and inference seed
  ET = rt_slot(ET, entry.y, bank.steer_stride);
  H0 = rt_slot(H0, entry.x, bank.dict_stride);
  K = rt_atoms_of(bank, entry.x, K);
  if (bank.assign && t == 0 && threadIdx.x == 0) rt_slot(bank.assign, s, stride)[2] = K;    // the shape of this block's K-shaped items
  const float* in_ring = rt_slot(in_ring0, s, stride);
  const float* in_block = in_blocks ? in_blocks + (int64_t)s * 2 * B : nullptr;
  if (windowed) windowed += (int64_t)s * 2 * N * nT;
  float2* X = rt_slot(X0, s, stride);
  float* G = rt_slot(G0, s, stride);
  float* gccphat = rt_slot(gccphat0, s, stride);
  float* Vabs = rt_slot(Vabs0, s, stride);
  float* H = rt_slot(Hs0, s, stride);
  const int call = dev->block_counter + 1;
  const int w0 = L - N - (nT - 1 - t) * hop;         // utils.py:107 windowIndexes[t]
  for (int i = threadIdx.x; i < N; i += blockDim.x) {
    float l, r;
    if (windowed) {
      l = windowed[((int64_t)0 * N + i) * nT + t];
      r = windowed[((int64_t)1 * N + i) * nT + t];
    } else {
      const int p = w0 + i;
      if (p >= L - B) {                               // the block being pushed in by this call
        l = in_block[p - (L - B)];
        r = in_block[B + p - (L - B)];
      } else {
        const int q = rt_ring_index(p, call, B, L);
        l = in_ring[q];
        r = in_ring[L + q];
      }
    }
    const float w = win_a[i];
    fft[bitrev(i, log2n)] = double2{(double)__fmul_rn(l, w), (double)__fmul_rn(r, w)};   // float32 product (:202), double transform
  }
  __syncthreads();
  fft_inplace<double2, double>(fft, tw, N, log2n, false);
  for (int k = threadIdx.x; k < F; k += blockDim.x) {
    const double2 a = fft[k], b = fft[(N - k) & (N - 1)];
    const float2 xl = float2{(float)(0.5 * (a.x + b.x)), (float)(0.5 * (a.y - b.y))};
    const float2 xr = float2{(float)(0.5 * (a.y + b.y)), (float)(0.5 * (b.x - a.x))};
    X[((int64_t)0 * F + k) * nT + t] = xl;
    X[((int64_t)1 * F + k) * nT + t] = xr;
    coh[k] = rt_coherence(xl, xr);
    if (inference) {                                  // abs(stereoSTFTFrame).T (onlineSpeechEnhancement.ipynb:433): column 2 t + channel
      Vabs[(int64_t)k * (2 * nT) + 2 * t] = (float)sqrt((double)xl.x * xl.x + (double)xl.y * xl.y);
      Vabs[(int64_t)k * (2 * nT) + 2 * t + 1] = (float)sqrt((double)xr.x * xr.x + (double)xr.y * xr.y);
    }
  }
  if (inference)                                      // every frame starts from the same seeded H0 (the notebook re-seeds per call)
    for (int k = threadIdx.x; k < K; k += blockDim.x) {
      H[(int64_t)k * (2 * nT) + 2 * t] = H0[2 * k];
      H[(int64_t)k * (2 * nT) + 2 * t + 1] = H0[2 * k + 1];
    }
  __syncthreads();
  // realGCC[f][t][d] = Re(coh[f] * E[f][d]) in complex64 arithmetic (:254), stored [t][d][f]
  float* Gt = G + (int64_t)t * D * Fp;
  for (int i = threadIdx.x; i < D * Fp; i += blockDim.x) {
    const int d = i / Fp, f = i - d * Fp;
    float v = 0.f;
    if (f < F) {
      const float2 c = coh[f], e = ET[i];
      v = __fsub_rn(__fmul_rn(c.x, e.x), __fmul_rn(c.y, e.y));
    }
    Gt[i] = v;
  }
  __syncthreads();
  // gccPHAT[d] = nanmean over f (:214)
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int d = warp; d < D; d += kFftThreads / 32) {
    double sum = 0.0;
    int n = 0;
    for (int f = lane; f < F; f += 32) {
      const float v = Gt[(int64_t)d * Fp + f];
      if (v == v) { sum += (double)v; ++n; }
    }
    for (int o = 16; o > 0; o >>= 1) { sum += __shfl_xor_sync(0xffffffffu, sum, o); n += __shfl_xor_sync(0xffffffffu, n, o); }
    if (lane == 0) gccphat[(int64_t)d * nT + t] = n > 0 ? (float)(sum / (double)n) : __int_as_float(0x7fc00000);
  }
}

// ---------------------------------------------------------------------------------------------- I: coefficient inference
// Slots per warp of the inference and filter kernels: the dictionary row a warp streams is used for all of them.  The register
// budget is 16 float (inference) or 32 double (filter) accumulators per lane.
constexpr int rt_inf_slots(int J) { return J >= 16 ? 1 : 16 / J; }
constexpr int rt_filter_slots(int NT) { return NT >= 8 ? 1 : 8 / NT; }

// R[f][j] = V[f][j] / sum_k W[f][k] H[k][j]   (gccNMFFunctions.py:76, V / dot(W, H)); one warp per bin and SG slots, J = 2 nT
// columns.  Per slot and column: lane-strided fmaf over k from 0.f, then the xor butterfly.  With a bank, one slot per warp (SG = 1)
// and the W, W^T and colsumW of the slot's dictionary entry: the order over k does not depend on the entry.
template <int J, int SG>
__global__ void __launch_bounds__(256)
rt_inf_ratio_kernel(const RtDev* __restrict__ dev0, size_t stride, int S, const float* __restrict__ W, const float* __restrict__ H0,
                    const float* __restrict__ V0, int F, int K, float* __restrict__ R0, RtBank bank) {
  const int f = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31, s0 = blockIdx.y * SG;
  if (f >= F) return;
  if constexpr (SG == 1) {                           // the slot's dictionary entry (grouped warps run without a bank only)
    const int dict = rt_entry(bank, s0, stride).x;
    W = rt_slot(W, dict, bank.dict_stride);
    K = rt_atoms_of(bank, dict, K);
  }
  bool on[SG];
  bool any = false;
#pragma unroll
  for (int g = 0; g < SG; ++g) {
    on[g] = s0 + g < S && rt_slot(dev0, s0 + g, stride)->active;
    any |= on[g];
  }
  if (!any) return;
  float acc[SG][J];
#pragma unroll
  for (int g = 0; g < SG; ++g)
#pragma unroll
    for (int j = 0; j < J; ++j) acc[g][j] = 0.f;
  for (int k = lane; k < K; k += 32) {
    const float w = W[(int64_t)f * K + k];
#pragma unroll
    for (int g = 0; g < SG; ++g) {
      if (!on[g]) continue;
      const float* H = rt_slot(H0, s0 + g, stride);
#pragma unroll
      for (int j = 0; j < J; ++j) acc[g][j] = fmaf(w, H[(int64_t)k * J + j], acc[g][j]);
    }
  }
#pragma unroll
  for (int g = 0; g < SG; ++g) {
    if (!on[g]) continue;
    const float* V = rt_slot(V0, s0 + g, stride);
    float* R = rt_slot(R0, s0 + g, stride);
#pragma unroll
    for (int j = 0; j < J; ++j) {
      float s = acc[g][j];
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      if (lane == 0) R[(int64_t)f * J + j] = V[(int64_t)f * J + j] / s;
    }
  }
}
// H[k][j] *= (sum_f W[f][k] R[f][j]) / (colsum(W)[k] + alpha + eps)   (:76); one warp per atom and SG slots over the transposed
// dictionary, lane-strided over f, then the xor butterfly.
template <int J, int SG>
__global__ void __launch_bounds__(256)
rt_inf_update_kernel(const RtDev* __restrict__ dev0, size_t stride, int S, const float* __restrict__ WT, int Fp, const float* __restrict__ R0, int F,
                     int K, const float* __restrict__ colsumW, float alpha, float eps, float* __restrict__ H0, RtBank bank) {
  const int k = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31, s0 = blockIdx.y * SG;
  if (k >= K) return;                                // the grid is rounded up to whole CTAs of 8 warps
  if constexpr (SG == 1) {                           // the slot's dictionary entry (grouped warps run without a bank only)
    const int dict = rt_entry(bank, s0, stride).x;
    if (k >= rt_atoms_of(bank, dict, K)) return;    // the grid covers K_max atoms
    WT = rt_slot(WT, dict, bank.dict_stride);
    colsumW = rt_slot(colsumW, dict, bank.dict_stride);
  }
  bool on[SG];
  bool any = false;
#pragma unroll
  for (int g = 0; g < SG; ++g) {
    on[g] = s0 + g < S && rt_slot(dev0, s0 + g, stride)->active;
    any |= on[g];
  }
  if (!any) return;
  float acc[SG][J];
#pragma unroll
  for (int g = 0; g < SG; ++g)
#pragma unroll
    for (int j = 0; j < J; ++j) acc[g][j] = 0.f;
  for (int f = lane; f < F; f += 32) {
    const float w = WT[(int64_t)k * Fp + f];
#pragma unroll
    for (int g = 0; g < SG; ++g) {
      if (!on[g]) continue;
      const float* R = rt_slot(R0, s0 + g, stride);
#pragma unroll
      for (int j = 0; j < J; ++j) acc[g][j] = fmaf(w, R[(int64_t)f * J + j], acc[g][j]);
    }
  }
  const float denom = (colsumW[k] + alpha) + eps;
#pragma unroll
  for (int g = 0; g < SG; ++g) {
    if (!on[g]) continue;
    float* H = rt_slot(H0, s0 + g, stride);
#pragma unroll
    for (int j = 0; j < J; ++j) {
      float s = acc[g][j];
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      if (lane == 0) H[(int64_t)k * J + j] = H[(int64_t)k * J + j] * (s / denom);
    }
  }
}

// ---------------------------------------------------------------------------------------------- B: per-atom TDOA argmax + atom mask
// One register-blocked SIMT tile over rows = (slot, frame, d) and columns = atoms: C[row][k] = sum_f G[row][f] W[f][k].
// 256 threads = 16 row groups x 16 atom groups; a thread owns TM consecutive rows and TN atoms.  A CTA covers RB = 16 TM rows =
// RB / Dp whole (slot, frame) pairs (Dp = D rounded up to 32, 64 or 128; rows d >= D are zero and never win) and KB = 16 TN atoms,
// so the argmax over d of every (pair, atom) it owns is inside the CTA.  Per f stage the W tile is staged in shared memory once
// and used by every pair of the CTA.  Each output is ONE fmaf chain over f = 0 .. F-1 starting from 0.f, in f order, whatever
// TM / TN: the float32 values, and so the decisions, do not depend on the tile shape or on the other slots.
//   TM = Dp / 16 (2, 4, 8), TN = 1: one pair x 16 atoms per CTA (K / 16 x pairs CTAs: latency for few streams)
//   TM = 8, TN = 8:                 128 rows x 128 atoms per CTA (64 accumulators per thread: throughput for many streams)
// P > 0 sources: the P target rows of every (pair, atom) go through shared memory to one pass that writes the P one-hot masks
// (source q of slot s at rt_slot(rt_slot(hmask0, s, stride), q, src_stride)) and the values (tval, (P, K, nT) per slot); the
// single-target mask is not written.
template <int TM, int TN>
__global__ void __launch_bounds__(256)
rt_atoms_kernel(const RtDev* __restrict__ dev0, size_t stride, int pairs, int nT, const float* __restrict__ G0, const float* __restrict__ W, int F,
                int Fp, int K, int D, int Dp, int32_t* __restrict__ argmax0, double* __restrict__ hmask0, const int32_t* __restrict__ targets0, int P,
                size_t src_stride, float* __restrict__ tval0, RtBank bank) {
  constexpr int RB = 16 * TM, KB = 16 * TN, GS = RB + 4, FC = kRtAtomsFc;
  static_assert(RB % 32 == 0 && (TM <= 2 || TM % 4 == 0) && (TN < 4 || TN % 4 == 0), "tile shape");
  static_assert(32 * KB + (RB / 32) * kRtMaxSources * KB <= FC * GS + FC * KB, "target rows must fit beside the argmax partials");
  __shared__ __align__(16) float sm[FC * GS + FC * KB];
  __shared__ int act[RB / 32], slot_of[RB / 32], dict_of[RB / 32], atoms_of[RB / 32];
  __shared__ int tgt[RB / 32][kRtMaxSources];
  float* Gs = sm;                         // [f][row]
  float* Ws = sm + FC * GS;               // [f][atom]
  // pairs per CTA: the narrow tile is launched with Dp = 16 TM, one pair, which lets the compiler drop the per-entry pass loop
  const int ppc = TN == 1 ? 1 : RB / Dp, k0 = blockIdx.x * KB, gp0 = blockIdx.y * ppc;
  const int ag = threadIdx.x & 15, rg = threadIdx.x >> 4;
  if (threadIdx.x < ppc) {                // pair gp: frame gp % nT of the slot at sorted position gp / nT
    const int gp = gp0 + threadIdx.x;
    const int s = gp < pairs ? rt_sorted_slot(bank, gp / nT) : 0;
    const int e = rt_entry(bank, s, stride).x;
    slot_of[threadIdx.x] = s;
    dict_of[threadIdx.x] = e;
    atoms_of[threadIdx.x] = rt_atoms_of(bank, e, K);
    act[threadIdx.x] = gp < pairs && rt_slot(dev0, s, stride)->active && k0 < atoms_of[threadIdx.x];
    for (int q = 0; q < P; ++q) tgt[threadIdx.x][q] = act[threadIdx.x] ? rt_slot(targets0, s, stride)[q] : -1;
  }
  __syncthreads();
  bool any = false;
  for (int p = 0; p < ppc; ++p) any |= act[p] != 0;
  if (!any) return;

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;
  auto atom_of = [&](int j) { return TN >= 4 ? (j >> 2) * 64 + ag * 4 + (j & 3) : j * 16 + ag; };
  const int mine = (rg * TM) / Dp;        // the pair of this thread's rows (a warp's rows lie in one pair)

  // One f loop per distinct dictionary entry of the CTA's active pairs (one pass unless the pairs straddle entries); a thread
  // accumulates only in its own pair's pass, so every output is still one fmaf chain over f.
  for (int pass = 0; pass < ppc; ++pass) {
    bool first = act[pass] != 0;
    for (int p = 0; p < pass; ++p) first &= !(act[p] && dict_of[p] == dict_of[pass]);
    if (!first) continue;
    const int e = dict_of[pass], Ke = atoms_of[pass];
    const float* We = rt_slot(W, e, bank.dict_stride);
    const bool accumulate = TN == 1 || (act[mine] && dict_of[mine] == e);     // the narrow tile's one pair is active here
    for (int f0 = 0; f0 < F; f0 += FC) {
      // G stage: float4 along f (Fp % 4 == 0, G zero on [F, Fp)), transposed into Gs[f][row]
      for (int i = threadIdx.x; i < RB * (FC / 4); i += 256) {
        const int row = i / (FC / 4), fq = i - row * (FC / 4), p = row / Dp, d = row - p * Dp, gp = gp0 + p, f = f0 + 4 * fq;
        float4 v = float4{0.f, 0.f, 0.f, 0.f};
        if (d < D && act[p] && (TN == 1 || dict_of[p] == e) && f < Fp) {
          const int t = gp % nT;
          v = *reinterpret_cast<const float4*>(rt_slot(G0, slot_of[p], stride) + ((int64_t)t * D + d) * Fp + f);
        }
        Gs[(4 * fq + 0) * GS + row] = v.x;
        Gs[(4 * fq + 1) * GS + row] = v.y;
        Gs[(4 * fq + 2) * GS + row] = v.z;
        Gs[(4 * fq + 3) * GS + row] = v.w;
      }
      for (int i = threadIdx.x; i < FC * KB; i += 256) {
        const int ff = i / KB, a = i - ff * KB;
        Ws[i] = (f0 + ff < F && k0 + a < Ke) ? We[(int64_t)(f0 + ff) * Ke + k0 + a] : 0.f;
      }
      __syncthreads();
      if (accumulate) {
#pragma unroll 4
        for (int ff = 0; ff < FC; ++ff) {
          float a[TM], b[TN];
          const float* gr = Gs + ff * GS + rg * TM;
          if constexpr (TM % 4 == 0) {
#pragma unroll
            for (int i = 0; i < TM; i += 4) {
              const float4 q = *reinterpret_cast<const float4*>(gr + i);
              a[i] = q.x; a[i + 1] = q.y; a[i + 2] = q.z; a[i + 3] = q.w;
            }
          } else {
#pragma unroll
            for (int i = 0; i < TM; ++i) a[i] = gr[i];
          }
          if constexpr (TN % 4 == 0) {
#pragma unroll
            for (int j = 0; j < TN; j += 4) {
              const float4 q = *reinterpret_cast<const float4*>(Ws + ff * KB + atom_of(j));
              b[j] = q.x; b[j + 1] = q.y; b[j + 2] = q.z; b[j + 3] = q.w;
            }
          } else {
#pragma unroll
            for (int j = 0; j < TN; ++j) b[j] = Ws[ff * KB + atom_of(j)];
          }
#pragma unroll
          for (int i = 0; i < TM; ++i)
#pragma unroll
            for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);     // tensor.dot(realGCC.T, W) in float32 (:259)
        }
      }
      __syncthreads();
    }
  }
  // argmax over d: first over the thread's TM rows, then over the row groups of the pair (partials alias the stage buffers)
  float* part_v = sm;
  int* part_i = reinterpret_cast<int*>(sm + 16 * KB);
  {
    const int r0 = rg * TM, d0 = r0 - (r0 / Dp) * Dp;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      float bv = 0.f;
      int bi = -1;
#pragma unroll
      for (int i = 0; i < TM; ++i)
        if (d0 + i < D && (bi < 0 || rt_better(acc[i][j], d0 + i, bv, bi))) { bv = acc[i][j]; bi = d0 + i; }
      part_v[rg * KB + atom_of(j)] = bv;
      part_i[rg * KB + atom_of(j)] = bi;
    }
  }
  float* tv = sm + 32 * KB;               // target rows [pair][source][atom], after the argmax partials
  if (P > 0) {
    const int r0 = rg * TM, p = r0 / Dp, d0 = r0 - p * Dp;
    for (int q = 0; q < P; ++q) {
      const int i = tgt[p][q] - d0;       // a duplicate target is a second copy of the same row
      if (i < 0 || i >= TM) continue;
#pragma unroll
      for (int ii = 0; ii < TM; ++ii)     // register selection (no dynamically indexed local array)
        if (ii == i)
#pragma unroll
          for (int j = 0; j < TN; ++j) tv[(p * kRtMaxSources + q) * KB + atom_of(j)] = acc[ii][j];
    }
  }
  __syncthreads();
  const int groups = Dp / TM;
  for (int idx = threadIdx.x; idx < ppc * KB; idx += 256) {
    const int p = idx / KB, a = idx - p * KB, gp = gp0 + p, k = k0 + a, Kp = atoms_of[p];
    if (!act[p] || k >= Kp) continue;
    float bv = 0.f;
    int bi = -1;
    for (int r = p * groups; r < (p + 1) * groups; ++r) {
      const int ci = part_i[r * KB + a];
      if (ci < 0) continue;
      const float cv = part_v[r * KB + a];
      if (bi < 0 || rt_better(cv, ci, bv, bi)) { bv = cv; bi = ci; }
    }
    const int s = slot_of[p], t = gp % nT;
    const RtDev* dev = rt_slot(dev0, s, stride);
    const int64_t o = (int64_t)k * nT + t;
    rt_slot(argmax0, s, stride)[o] = bi;
    if (P > 0) {                          // gccNMFFunctions.py:137-143 per block: the winning source takes the atom
      const float* v = tv + p * kRtMaxSources * KB + a;
      float wv = v[0];
      int wi = 0;
      for (int q = 1; q < P; ++q)
        if (rt_better(v[q * KB], q, wv, wi)) { wv = v[q * KB]; wi = q; }
      double* m0 = rt_slot(hmask0, s, stride);
      float* tval = rt_slot(tval0, s, stride);
      for (int q = 0; q < P; ++q) {
        rt_slot(m0, q, src_stride)[o] = q == wi ? 1.0 : 0.0;
        tval[((int64_t)q * Kp + k) * nT + t] = v[q * KB];          // (P, K_i, nT)
      }
      continue;
    }
    // int64 - float32 promotes to float64 in Theano and numpy alike: the mask arithmetic is float64 (:263, :265)
    const double dist = fabs((double)bi - (double)dev->target);
    double m;
    if (dev->mode == 0) m = dist < (double)dev->eps ? 1.0 : 0.0;
    else m = exp(-pow(dist / (double)dev->eps, (double)dev->beta)) / (double)(1.0f + dev->noise_floor) + (double)dev->noise_floor;
    rt_slot(hmask0, s, stride)[o] = m;
  }
}

// ---------------------------------------------------------------------------------------------- C: time-frequency mask, one warp per bin and SG slots
// Per slot, frame and channel: lane-strided float64 sums over k, then the xor butterfly.  blockIdx.z: the source (mask and Y at
// src_stride per source).  With a bank, one slot per warp and the W, recV and K_i of the slot's dictionary entry.
template <int NT, int SG, bool inference>
__global__ void __launch_bounds__(256)
rt_filter_kernel(const RtDev* __restrict__ dev0, size_t stride, int S, const float* __restrict__ W, const double* __restrict__ hmask0,
                 const float* __restrict__ recV, const float* __restrict__ H0, const float2* __restrict__ X0, int F, int K, float2* __restrict__ Y0,
                 size_t src_stride, RtBank bank) {
  const int f = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31, s0 = blockIdx.y * SG;
  if (f >= F) return;
  if constexpr (SG == 1) {                           // the slot's dictionary entry (grouped warps run without a bank only)
    const int dict = rt_entry(bank, s0, stride).x;
    W = rt_slot(W, dict, bank.dict_stride);
    recV = rt_slot(recV, dict, bank.dict_stride);
    K = rt_atoms_of(bank, dict, K);
  }
  hmask0 = rt_slot(hmask0, blockIdx.z, src_stride);
  Y0 = rt_slot(Y0, blockIdx.z, src_stride);
  bool on[SG];
  bool any = false;
#pragma unroll
  for (int g = 0; g < SG; ++g) {
    on[g] = false;
    if (s0 + g >= S) continue;
    const RtDev* dev = rt_slot(dev0, s0 + g, stride);
    if (!dev->active) continue;
    if (!dev->separation) {                          // :211 outputSpectrogram = complexMixtureSpectrogram.copy()
      const float2* X = rt_slot(X0, s0 + g, stride);
      float2* Y = rt_slot(Y0, s0 + g, stride);
      for (int i = lane; i < 2 * NT; i += 32) {
        const int c = i / NT, t = i - c * NT;
        Y[((int64_t)c * F + f) * NT + t] = X[((int64_t)c * F + f) * NT + t];
      }
      continue;
    }
    on[g] = true;
    any = true;
  }
  if (!any) return;
  double num[SG][2][NT], den[SG][2][NT];
#pragma unroll
  for (int g = 0; g < SG; ++g)
#pragma unroll
    for (int t = 0; t < NT; ++t) { num[g][0][t] = num[g][1][t] = den[g][0][t] = den[g][1][t] = 0.0; }
  for (int k = lane; k < K; k += 32) {
    const double w = (double)W[(int64_t)f * K + k];
#pragma unroll
    for (int g = 0; g < SG; ++g) {
      if (!on[g]) continue;
      const double* hmask = rt_slot(hmask0, s0 + g, stride);
      const float* H = rt_slot(H0, s0 + g, stride);
#pragma unroll
      for (int t = 0; t < NT; ++t) {
        const double m = hmask[(int64_t)k * NT + t];
        if constexpr (inference) {                   // sourceEstimate = W . (H * mask), recV = W . H  (ipynb:435-437)
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            const double hv = (double)H[(int64_t)k * (2 * NT) + 2 * t + c];
            num[g][c][t] += w * (hv * m);
            den[g][c][t] += w * hv;
          }
        } else {
          num[g][0][t] += w * m;                     // tensor.dot(W, HMask) (:267)
        }
      }
    }
  }
#pragma unroll
  for (int g = 0; g < SG; ++g) {
    if (!on[g]) continue;
#pragma unroll
    for (int t = 0; t < NT; ++t) {
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        if (c == 1 && !inference) continue;
        double a = num[g][c][t], b = den[g][c][t];
        for (int o = 16; o > 0; o >>= 1) { a += __shfl_xor_sync(0xffffffffu, a, o); b += __shfl_xor_sync(0xffffffffu, b, o); }
        num[g][c][t] = a; den[g][c][t] = b;
      }
    }
    if (lane < 2 * NT) {
      const float2* X = rt_slot(X0, s0 + g, stride);
      float2* Y = rt_slot(Y0, s0 + g, stride);
      const int c = lane / NT, t = lane - c * NT;
      double tf = 0.0;
#pragma unroll
      for (int tt = 0; tt < NT; ++tt)                // register selection (no dynamically indexed local array)
        if (tt == t) tf = inference ? (c ? num[g][1][tt] / den[g][1][tt] : num[g][0][tt] / den[g][0][tt]) : num[g][0][tt] / (double)recV[f];
      const float2 x = X[((int64_t)c * F + f) * NT + t];
      Y[((int64_t)c * F + f) * NT + t] = float2{(float)(tf * (double)x.x), (float)(tf * (double)x.y)};   // inputMask * spectrogram (:209)
    }
  }
}

// ---------------------------------------------------------------------------------------------- D: synthesis (one CTA per frame, slot and source)
__global__ void __launch_bounds__(kFftThreads)
rt_synthesis_kernel(RtDev* __restrict__ dev0, size_t stride, const float2* __restrict__ Y0, const float2* __restrict__ tw, int N, int log2n, int nT,
                    const float* __restrict__ win_s, float* __restrict__ frames0, float* __restrict__ out_windowed, int advance, size_t src_stride) {
  __shared__ float2 fft[kRtMaxN];
  const int t = blockIdx.x, s = blockIdx.y, F = N / 2 + 1;
  RtDev* dev = rt_slot(dev0, s, stride);
  Y0 = rt_slot(Y0, blockIdx.z, src_stride);
  frames0 = rt_slot(frames0, blockIdx.z, src_stride);
  if (out_windowed) out_windowed += ((int64_t)s * gridDim.z + blockIdx.z) * 2 * N * nT;      // (S, P, 2, N, nT)
  advance = advance && blockIdx.z == 0;
  if (!dev->active) {                                            // an inactive slot's output frames are zeros
    if (out_windowed)
      for (int i = threadIdx.x; i < N; i += blockDim.x) {
        out_windowed[((int64_t)0 * N + i) * nT + t] = 0.f;
        out_windowed[((int64_t)1 * N + i) * nT + t] = 0.f;
      }
    return;
  }
  const float2* Y = rt_slot(Y0, s, stride);
  float* frames = rt_slot(frames0, s, stride);
  for (int k = threadIdx.x; k < F; k += blockDim.x) {
    float2 a = Y[((int64_t)0 * F + k) * nT + t], b = Y[((int64_t)1 * F + k) * nT + t];
    if (k == 0 || k == N / 2) { a.y = 0.f; b.y = 0.f; }          // numpy.fft.irfft ignores them
    fft[bitrev(k, log2n)] = float2{a.x - b.y, a.y + b.x};
    if (k != 0 && k != N / 2) fft[bitrev(N - k, log2n)] = float2{a.x + b.y, b.x - a.y};
  }
  __syncthreads();
  fft_inplace<float2, float>(fft, tw, N, log2n, true);
  const float inv_n = 1.0f / (float)N;
  for (int i = threadIdx.x; i < N; i += blockDim.x) {
    const float2 z = fft[i];
    const float w = win_s[i];
    const float l = z.x * inv_n * w, r = z.y * inv_n * w;        // irfft(...) * synthesisWindowFunction (:231)
    frames[((int64_t)0 * nT + t) * N + i] = l;
    frames[((int64_t)1 * nT + t) * N + i] = r;
    if (out_windowed) {
      out_windowed[((int64_t)0 * N + i) * nT + t] = l;
      out_windowed[((int64_t)1 * N + i) * nT + t] = r;
    }
  }
  if (advance && t == 0 && threadIdx.x == 0) atomicAdd(&dev->block_counter, 1);     // the ring kernel that follows uses counter (= this call's number)
}

// ---------------------------------------------------------------------------------------------- localisation (one CTA per slot, D <= 128 threads used)
// P > 0: the P largest peaks of the mean (select_peaks) replace `targets`; with fewer peaks the targets stay and status bit 0 is set.
__device__ void rt_localize(RtDev* dev, const float* __restrict__ gccphat, int D, int nT, double* __restrict__ hist, int hist_len,
                            int32_t* __restrict__ targets, int32_t* __restrict__ status, int P) {
  __shared__ double mean_s[kRtMaxD];
  __shared__ unsigned char peak_s[kRtMaxD], chosen_s[kRtMaxD];
  __shared__ int num_peaks_s;
  __shared__ int32_t pick_s[kRtMaxSources];
  const int d = threadIdx.x;
  int idx = dev->hist_index;
  // gccPHATHistory.set(nanmean(realGCC, axis=0).T)   (:214 -> utils.py:45-59)
  if (d < D)
    for (int t = 0; t < nT; ++t) hist[(int64_t)d * hist_len + (idx + t) % hist_len] = (double)gccphat[(int64_t)d * nT + t];
  idx = (idx + nT) % hist_len;
  __syncthreads();
  if (d < D) {
    // nanmean over the last loc_window columns of the unravelled history (:221-222)
    const int w = min(max(dev->loc_window, 1), hist_len);
    double s = 0.0;
    int n = 0;
    for (int j = 0; j < w; ++j) {
      const double v = hist[(int64_t)d * hist_len + (idx - 1 - j + 2 * hist_len) % hist_len];
      if (v == v) { s += v; ++n; }
    }
    mean_s[d] = n > 0 ? s / (double)n : __longlong_as_double(0x7ff8000000000000LL);
  }
  __syncthreads();
  if (P > 0) {
    if (dev->localization) {            // estimateTargetTDOAIndexesFromAngularSpectrum, numSources branch (gccNMFFunctions.py:94-116)
      const int peaks = select_peaks(mean_s, D, P, peak_s, chosen_s, &num_peaks_s, pick_s);
      if (d == 0) {
        if (peaks >= P)
          for (int q = 0; q < P; ++q) targets[q] = pick_s[q];
        else
          *status |= GCCNMF_RTSEP_STATUS_FEW_PEAKS;
      }
    }
    if (d == 0) dev->hist_index = idx;
    return;
  }
  if (d == 0) {
    if (dev->localization) {
      double bv = mean_s[0];
      int bi = 0;
      for (int j = 1; j < D; ++j)
        if (rt_better64(mean_s[j], j, bv, bi)) { bv = mean_s[j]; bi = j; }
      dev->target = (float)bi;                       // targetTDOAIndex.set_value(tdoaIndex)
    }
    dev->hist_index = idx;
  }
}

__global__ void __launch_bounds__(128)
rt_localize_kernel(RtDev* dev0, size_t stride, const float* __restrict__ gccphat0, int D, int nT, double* __restrict__ hist0, int hist_len,
                   int32_t* __restrict__ targets0, int32_t* __restrict__ status0, int P) {
  const int s = blockIdx.x;
  RtDev* dev = rt_slot(dev0, s, stride);
  if (!dev->active) return;
  rt_localize(dev, rt_slot(gccphat0, s, stride), D, nT, rt_slot(hist0, s, stride), hist_len, rt_slot(targets0, s, stride), rt_slot(status0, s, stride), P);
}

// ---------------------------------------------------------------------------------------------- E: overlap-add ring, block emit, input push
// grid (ring CTAs + 1, S, sources).  CTAs [0, gridDim.x - 1): one thread per logical ring position of the range that changes or is
// emitted, into the source's own output ring; last CTA of source 0: localisation.  Source 0 pushes the input block.
__global__ void __launch_bounds__(128)
rt_ola_emit_kernel(RtDev* dev0, size_t stride, const float* __restrict__ frames0, int N, int hop, int nT, int B, int L, int p_first,
                   float* __restrict__ out_ring0, float* __restrict__ out_blocks, const float* __restrict__ in_blocks, float* __restrict__ in_ring0,
                   const float* __restrict__ gccphat0, int D, double* __restrict__ hist0, int hist_len, int32_t* __restrict__ targets0,
                   int32_t* __restrict__ status0, int P, size_t src_stride) {
  const int s = blockIdx.y, z = blockIdx.z;
  RtDev* dev = rt_slot(dev0, s, stride);
  const bool active = dev->active != 0;
  if (blockIdx.x == gridDim.x - 1) {
    if (active && z == 0)
      rt_localize(dev, rt_slot(gccphat0, s, stride), D, nT, rt_slot(hist0, s, stride), hist_len, rt_slot(targets0, s, stride),
                  rt_slot(status0, s, stride), P);
    return;
  }
  frames0 = rt_slot(frames0, z, src_stride);
  out_ring0 = rt_slot(out_ring0, z, src_stride);
  float* out_block = out_blocks + ((int64_t)s * gridDim.z + z) * 2 * B;       // (S, P, 2, B)
  const int p = p_first + blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= L) return;
  if (!active) {                                     // an inactive slot emits a block of zeros
    if (p >= L - 3 * B && p < L - 2 * B)
      for (int c = 0; c < 2; ++c) out_block[c * B + (p - (L - 3 * B))] = 0.f;
    return;
  }
  const float* frames = rt_slot(frames0, s, stride);
  float* out_ring = rt_slot(out_ring0, s, stride);
  float* in_ring = rt_slot(in_ring0, s, stride);
  const float* in_block = in_blocks + (int64_t)s * 2 * B;
  const int call = dev->block_counter;               // already advanced by the synthesis kernel
  const int q = rt_ring_index(p, call, B, L);
  const int w_first = L - N - (nT - 1) * hop;
#pragma unroll
  for (int c = 0; c < 2; ++c) {
    float acc = p >= L - B ? 0.f : out_ring[c * L + q];          // outputBuffer[:, -B:] = 0 (utils.py:105)
    if (p >= w_first) {
      for (int i = 0; i < nT; ++i) {                              // frame order, float32 buffer += float64 frame (utils.py:113-114)
        const int r = p - (w_first + i * hop);
        if (r >= 0 && r < N) acc = (float)((double)acc + (double)frames[((int64_t)c * nT + i) * N + r]);
      }
    }
    out_ring[c * L + q] = acc;
    if (p >= L - 3 * B && p < L - 2 * B) out_block[c * B + (p - (L - 3 * B))] = acc;   // outputFrames = outputBuffer[:, -3B:-2B] (:115)
    if (p >= L - B && z == 0) in_ring[c * L + q] = in_block[c * B + (p - (L - B))];    // inputBuffer[:, -B:] = inputFrames (:102)
  }
}

int ilog2_of(int n) {
  int l = 0;
  while ((1 << l) < n) ++l;
  return l;
}

#define RT_CARVE_OR_FAIL_B(l, S, P, Qd, Qe)                                                                                        \
  if (int st__ = rt_check(h, cfg, (S), (P))) return st__;                                                                          \
  RtLayout l = rt_carve(*cfg, (S), (P), state, state_bytes, (Qd), (Qe));                                                           \
  if (!l.ok) return gccnmf_fail(h, GCCNMF_ERR_WORKSPACE, "rt state buffer missing or too small: need %zu bytes", l.bytes)
#define RT_CARVE_OR_FAIL_P(l, S, P) RT_CARVE_OR_FAIL_B(l, S, P, 0, 0)
#define RT_CARVE_OR_FAIL(l, S) RT_CARVE_OR_FAIL_P(l, S, 0)

inline int rt_sources_grid(const RtLayout& l) { return l.P > 0 ? l.P : 1; }

// Several slots per warp (the dictionary row read once for all of them) only while the grid still has kRtWavesForSlotGroups waves
// of CTAs; with fewer streams one slot per warp keeps the device busy.  A bank runs one slot per warp (each on its own entry).
constexpr int kRtWavesForSlotGroups = 4;
inline bool rt_group_slots(const gccnmf_handle* h, const RtLayout& l, int ctas_x, int SG) {
  return SG > 1 && l.S > 1 && l.Qd == 0 && (int64_t)ctas_x * ((l.S + SG - 1) / SG) >= (int64_t)kRtWavesForSlotGroups * h->sm_count;
}

template <int J, int SG>
int rt_enqueue_inference_as(gccnmf_handle* h, const gccnmf_rt_config* cfg, const RtLayout& l, bool ratio, void* stream) {
  const int F = l.F, K = cfg->num_atoms, S = l.S, gy = (S + SG - 1) / SG;
  if (ratio)
    GCCNMF_LAUNCH(h, (rt_inf_ratio_kernel<J, SG>), dim3((F + 7) / 8, gy), 256, 0, stream, l.dev, l.stride, S, l.W, l.H, l.Vabs, F, K, l.R, l.bank);
  else
    GCCNMF_LAUNCH(h, (rt_inf_update_kernel<J, SG>), dim3((K + 7) / 8, gy), 256, 0, stream, l.dev, l.stride, S, l.WT, l.Fp, l.R, F, K, l.colsumW,
                  cfg->sparsity_alpha, cfg->epsilon, l.H, l.bank);
  return 0;
}
template <int J>
int rt_enqueue_inference(gccnmf_handle* h, const gccnmf_rt_config* cfg, const RtLayout& l, void* stream) {
  constexpr int SG = rt_inf_slots(J);
  const int F = l.F, K = cfg->num_atoms;
  const int st = rt_group_slots(h, l, (F + 7) / 8, SG) ? rt_enqueue_inference_as<J, SG>(h, cfg, l, true, stream)
                                                       : rt_enqueue_inference_as<J, 1>(h, cfg, l, true, stream);
  if (st) return st;
  return rt_group_slots(h, l, (K + 7) / 8, SG) ? rt_enqueue_inference_as<J, SG>(h, cfg, l, false, stream)
                                               : rt_enqueue_inference_as<J, 1>(h, cfg, l, false, stream);
}

template <int NT, int SG, bool INF>
int rt_enqueue_filter_as(gccnmf_handle* h, const gccnmf_rt_config* cfg, const RtLayout& l, void* stream) {
  const int F = l.F, K = cfg->num_atoms, S = l.S;
  GCCNMF_LAUNCH(h, (rt_filter_kernel<NT, SG, INF>), dim3((F + 7) / 8, (S + SG - 1) / SG, rt_sources_grid(l)), 256, 0, stream, l.dev, l.stride, S, l.W,
                l.smask, l.recV, l.H, l.X, F, K, l.sY, l.src_stride, l.bank);
  return 0;
}
template <int NT>
int rt_enqueue_filter(gccnmf_handle* h, const gccnmf_rt_config* cfg, const RtLayout& l, void* stream) {
  constexpr int SG = rt_filter_slots(NT);
  const bool inf = cfg->inference_iterations > 0;
  if (!rt_group_slots(h, l, (l.F + 7) / 8, SG))
    return inf ? rt_enqueue_filter_as<NT, 1, true>(h, cfg, l, stream) : rt_enqueue_filter_as<NT, 1, false>(h, cfg, l, stream);
  return inf ? rt_enqueue_filter_as<NT, SG, true>(h, cfg, l, stream) : rt_enqueue_filter_as<NT, SG, false>(h, cfg, l, stream);
}

// The atoms tile: 128 x 128 once it fills the device with at least one CTA per SM, else one (slot, frame) pair x 16 atoms.
template <int DJ>
int rt_enqueue_atoms(gccnmf_handle* h, const gccnmf_rt_config* cfg, const RtLayout& l, void* stream) {
  const int nT = cfg->windows_per_block, K = cfg->num_atoms, D = cfg->num_tdoas, pairs = l.S * nT, Dp = 16 * DJ;
  const int big_ctas = ((K + 127) / 128) * ((pairs + 128 / Dp - 1) / (128 / Dp));
  if (big_ctas >= h->sm_count)
    GCCNMF_LAUNCH(h, (rt_atoms_kernel<8, 8>), dim3((K + 127) / 128, (pairs + 128 / Dp - 1) / (128 / Dp)), 256, 0, stream, l.dev, l.stride, pairs, nT,
                  l.G, l.W, l.F, l.Fp, K, D, Dp, l.argmax, l.smask, l.targets, l.P, l.src_stride, l.tval, l.bank);
  else
    GCCNMF_LAUNCH(h, (rt_atoms_kernel<DJ, 1>), dim3((K + 15) / 16, pairs), 256, 0, stream, l.dev, l.stride, pairs, nT, l.G, l.W, l.F, l.Fp, K, D, Dp,
                  l.argmax, l.smask, l.targets, l.P, l.src_stride, l.tval, l.bank);
  return 0;
}

// Kernels A .. D (+ inference) of one block for every slot; `windowed` != NULL: frames given by the caller (processFrames, (S, 2, N, nT)),
// else cut from the rings and `in_blocks` (S, 2, B).
int rt_enqueue_core(gccnmf_handle* h, const gccnmf_rt_config* cfg, const RtLayout& l, const float* windowed, const float* in_blocks, float* out_windowed,
                    const double* forced_mask, int advance, void* stream) {
  const int N = cfg->window_size, nT = cfg->windows_per_block, K = cfg->num_atoms, D = cfg->num_tdoas, log2n = ilog2_of(N), S = l.S;
  const int inf = cfg->inference_iterations;
  GCCNMF_LAUNCH(h, rt_analysis_kernel, dim3(nT, S), kFftThreads, 0, stream, l.dev, l.stride, windowed, in_blocks, l.in_ring, cfg->block_size, l.L,
                cfg->hop_size, nT, l.win_a, reinterpret_cast<const double2*>(l.tw64), N, log2n, l.ET, D, l.Fp, l.X, l.G, l.gccphat, l.Vabs, l.H0, l.H, K,
                inf > 0 ? 1 : 0, l.bank);
  for (int it = 0; it < inf; ++it) {
    int st = 0;
    switch (nT) {
      case 1: st = rt_enqueue_inference<2>(h, cfg, l, stream); break;
      case 2: st = rt_enqueue_inference<4>(h, cfg, l, stream); break;
      case 3: st = rt_enqueue_inference<6>(h, cfg, l, stream); break;
      case 4: st = rt_enqueue_inference<8>(h, cfg, l, stream); break;
      case 5: st = rt_enqueue_inference<10>(h, cfg, l, stream); break;
      case 6: st = rt_enqueue_inference<12>(h, cfg, l, stream); break;
      case 7: st = rt_enqueue_inference<14>(h, cfg, l, stream); break;
      default: st = rt_enqueue_inference<16>(h, cfg, l, stream); break;
    }
    if (st) return st;
  }
  int st = 0;
  if (forced_mask) {     // teacher forcing / externally decided masks: the filter uses the caller's (S, K, nT) float64 atom masks
    const size_t row = (size_t)K * nT * sizeof(double);
    GCCNMF_CHECK_CUDA(h, cudaMemcpy2DAsync(l.hmask, l.stride, forced_mask, row, row, S, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  } else if (D <= 32) st = rt_enqueue_atoms<2>(h, cfg, l, stream);
  else if (D <= 64) st = rt_enqueue_atoms<4>(h, cfg, l, stream);
  else st = rt_enqueue_atoms<8>(h, cfg, l, stream);
  if (st) return st;
  switch (nT) {
    case 1: st = rt_enqueue_filter<1>(h, cfg, l, stream); break;
    case 2: st = rt_enqueue_filter<2>(h, cfg, l, stream); break;
    case 3: st = rt_enqueue_filter<3>(h, cfg, l, stream); break;
    case 4: st = rt_enqueue_filter<4>(h, cfg, l, stream); break;
    case 5: st = rt_enqueue_filter<5>(h, cfg, l, stream); break;
    case 6: st = rt_enqueue_filter<6>(h, cfg, l, stream); break;
    case 7: st = rt_enqueue_filter<7>(h, cfg, l, stream); break;
    default: st = rt_enqueue_filter<8>(h, cfg, l, stream); break;
  }
  if (st) return st;
  GCCNMF_LAUNCH(h, rt_synthesis_kernel, dim3(nT, S, rt_sources_grid(l)), kFftThreads, 0, stream, l.dev, l.stride, l.sY,
                reinterpret_cast<const float2*>(l.tw32), N, log2n, nT, l.win_s, l.sframes, out_windowed, advance, l.src_stride);
  return 0;
}

int rt_enqueue_params(gccnmf_handle* h, const RtLayout& l, int first, int count, const gccnmf_rtm_slot_params* params, int set_active, void* stream) {
  for (int i0 = 0; i0 < count; i0 += kRtParamsPerLaunch) {
    const int n = count - i0 < kRtParamsPerLaunch ? count - i0 : kRtParamsPerLaunch;
    RtParamsBatch b{};
    for (int i = 0; i < n; ++i) b.p[i] = params[i0 + i];
    GCCNMF_LAUNCH(h, rt_set_params_kernel, 1, kRtParamsPerLaunch, 0, stream, l.dev, l.stride, first + i0, n, b, set_active);
  }
  return 0;
}

// A bank's slots in dictionary order, after every change of an assignment (stream-ordered, like the changes themselves).
int rt_enqueue_sort(gccnmf_handle* h, const RtLayout& l, void* stream) {
  if (l.Qd > 0) GCCNMF_LAUNCH(h, sort_by_entry_kernel, 1, 32, 0, stream, l.assign, l.stride, l.S, l.Qd, l.order, nullptr);
  return 0;
}

// Zeroes the regions of slots [first, first + count) and gives them the defaults of gccNMFProcessor.py:190-199, active (and bank
// entries (0, 0)).
int rt_enqueue_reset(gccnmf_handle* h, const RtLayout& l, int first, int count, void* stream) {
  GCCNMF_CHECK_CUDA(h, cudaMemsetAsync(rt_slot(reinterpret_cast<char*>(l.dev), first, l.stride), 0, (size_t)count * l.stride, (cudaStream_t)stream));
  GCCNMF_LAUNCH(h, rt_default_params_kernel, (count + 127) / 128, 128, 0, stream, l.dev, l.stride, first, count, l.targets, l.P, l.D);
  return rt_enqueue_sort(h, l, stream);
}

// Dictionary entry i (the layout's one dictionary without a bank): W (F, Ki) and H0 (Ki, 2) or NULL, device pointers.
int rt_enqueue_dictionary(gccnmf_handle* h, const RtLayout& l, int i, const float* W, int Ki, const float* H0, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  const size_t st = l.bank.dict_stride;
  float* We = rt_slot(l.W, i, st);
  GCCNMF_CHECK_CUDA(h, cudaMemcpyAsync(We, W, (size_t)l.F * Ki * sizeof(float), cudaMemcpyDeviceToDevice, s));
  if (H0) GCCNMF_CHECK_CUDA(h, cudaMemcpyAsync(rt_slot(l.H0, i, st), H0, (size_t)Ki * 2 * sizeof(float), cudaMemcpyDeviceToDevice, s));
  const int n = Ki > l.F ? Ki : l.F;
  GCCNMF_LAUNCH(h, rt_init_dictionary_kernel, (n + 127) / 128, 128, 0, stream, We, l.F, l.Fp, Ki, rt_slot(l.WT, i, st), rt_slot(l.recV, i, st),
                rt_slot(l.colsumW, i, st), l.bank_K ? l.bank_K + i : nullptr);
  return 0;
}

// Steering entry j (the layout's one table without a bank): E (F, D) complex64, a device pointer.
int rt_enqueue_steering(gccnmf_handle* h, const RtLayout& l, int j, const float* E, void* stream) {
  GCCNMF_LAUNCH(h, rt_init_steering_kernel, (l.D * l.Fp + 255) / 256, 256, 0, stream, reinterpret_cast<const float2*>(E), l.F, l.Fp, l.D,
                rt_slot(l.ET, j, l.bank.steer_stride));
  return 0;
}

// Qd dictionaries W[i] (F, K[i]) with H0[i] (K[i], 2) (H0 or H0[i] NULL without inference) and Qe steering tables E[j]; the
// single-stream, rtm and rtsep entries pass one of each with Qd = Qe = 0 (no bank).
int rt_init(gccnmf_handle* h, const gccnmf_rt_config* cfg, int S, int P, int Qd, int Qe, const float* const* W, const int* K,
            const float* const* H0, const float* const* E, const float* analysis_window, const float* synthesis_window, void* state,
            size_t state_bytes, void* stream) {
  RT_CARVE_OR_FAIL_B(l, S, P, Qd, Qe);
  const int nd = Qd > 0 ? Qd : 1, ne = Qe > 0 ? Qe : 1;
  GCCNMF_REQUIRE(h, W && K && E && analysis_window && synthesis_window, "rt_init: NULL pointer");
  for (int i = 0; i < nd; ++i) {
    GCCNMF_REQUIRE(h, W[i] != nullptr, "rt_init: NULL pointer");
    GCCNMF_REQUIRE(h, K[i] >= 1 && K[i] <= cfg->num_atoms, "rt_init: dictionary %d: %d atoms outside [1, num_atoms = %d]", i, K[i], cfg->num_atoms);
    GCCNMF_REQUIRE(h, cfg->inference_iterations == 0 || (H0 && H0[i]), "rt_init: coefficient inference needs the initial H0 (K, 2)");
  }
  for (int j = 0; j < ne; ++j) GCCNMF_REQUIRE(h, E[j] != nullptr, "rt_init: NULL pointer");
  cudaStream_t s = (cudaStream_t)stream;
  const int N = cfg->window_size;
  const double* tw64 = nullptr;
  const float* tw32 = nullptr;
  if (int st = gccnmf_get_twiddles(h, N, &tw64, &tw32)) return st;
  GCCNMF_CHECK_CUDA(h, cudaMemsetAsync(state, 0, l.bytes, s));                 // rings, history (initValue = 0), counters, entries (0, 0)
  GCCNMF_CHECK_CUDA(h, cudaMemcpyAsync(l.tw64, tw64, (size_t)N * sizeof(double), cudaMemcpyDeviceToDevice, s));
  GCCNMF_CHECK_CUDA(h, cudaMemcpyAsync(l.tw32, tw32, (size_t)N * sizeof(float), cudaMemcpyDeviceToDevice, s));
  GCCNMF_CHECK_CUDA(h, cudaMemcpyAsync(l.win_a, analysis_window, (size_t)N * sizeof(float), cudaMemcpyDeviceToDevice, s));
  GCCNMF_CHECK_CUDA(h, cudaMemcpyAsync(l.win_s, synthesis_window, (size_t)N * sizeof(float), cudaMemcpyDeviceToDevice, s));
  for (int i = 0; i < nd; ++i)
    if (int st = rt_enqueue_dictionary(h, l, i, W[i], K[i], H0 ? H0[i] : nullptr, stream)) return st;
  for (int j = 0; j < ne; ++j)
    if (int st = rt_enqueue_steering(h, l, j, E[j], stream)) return st;
  GCCNMF_LAUNCH(h, rt_default_params_kernel, (S + 127) / 128, 128, 0, stream, l.dev, l.stride, 0, S, l.targets, l.P, l.D);
  return rt_enqueue_sort(h, l, stream);
}

// The single-stream, rtm and rtsep form: one dictionary of cfg.num_atoms atoms, one steering table.
int rt_init(gccnmf_handle* h, const gccnmf_rt_config* cfg, int S, int P, const float* W, const float* E, const float* analysis_window,
            const float* synthesis_window, const float* H0, void* state, size_t state_bytes, void* stream) {
  const float* Ws[1] = {W};
  const float* Es[1] = {E};
  const float* H0s[1] = {H0};
  const int Ks[1] = {cfg ? cfg->num_atoms : 0};
  return rt_init(h, cfg, S, P, 0, 0, Ws, Ks, H0 ? H0s : nullptr, Es, analysis_window, synthesis_window, state, state_bytes, stream);
}

int rt_process_block(gccnmf_handle* h, const gccnmf_rt_config* cfg, int S, int P, void* state, size_t state_bytes, const float* in_blocks,
                     float* out_blocks, const double* forced_atom_mask, void* stream, int Qd = 0, int Qe = 0) {
  RT_CARVE_OR_FAIL_B(l, S, P, Qd, Qe);
  GCCNMF_REQUIRE(h, in_blocks && out_blocks, "rt_process_block: NULL pointer");
  if (int st = rt_enqueue_core(h, cfg, l, nullptr, in_blocks, nullptr, forced_atom_mask, 1, stream)) return st;
  const int N = cfg->window_size, nT = cfg->windows_per_block, B = cfg->block_size;
  const int w_first = l.L - N - (nT - 1) * cfg->hop_size;
  const int p_first = w_first < l.L - 3 * B ? w_first : l.L - 3 * B;
  const int ctas = (l.L - p_first + 127) / 128;
  GCCNMF_LAUNCH(h, rt_ola_emit_kernel, dim3(ctas + 1, S, rt_sources_grid(l)), 128, 0, stream, l.dev, l.stride, l.sframes, N, cfg->hop_size, nT, B, l.L,
                p_first, l.sout, out_blocks, in_blocks, l.in_ring, l.gccphat, cfg->num_tdoas, l.hist, cfg->history_length, l.targets, l.status, l.P,
                l.src_stride);
  return GCCNMF_OK;
}

int rt_process_frames(gccnmf_handle* h, const gccnmf_rt_config* cfg, int S, int P, void* state, size_t state_bytes, const float* windowed, float* out,
                      const double* forced_atom_mask, void* stream, int Qd = 0, int Qe = 0) {
  RT_CARVE_OR_FAIL_B(l, S, P, Qd, Qe);
  GCCNMF_REQUIRE(h, windowed && out, "rt_process_frames: NULL pointer");
  if (int st = rt_enqueue_core(h, cfg, l, windowed, nullptr, out, forced_atom_mask, 0, stream)) return st;
  GCCNMF_LAUNCH(h, rt_localize_kernel, S, 128, 0, stream, l.dev, l.stride, l.gccphat, cfg->num_tdoas, cfg->windows_per_block, l.hist, cfg->history_length,
                l.targets, l.status, l.P);
  return GCCNMF_OK;
}

int rt_graph_create(gccnmf_handle* h, const gccnmf_rt_config* cfg, int S, int P, void* state, size_t state_bytes, float* in_blocks, float* out_blocks,
                    const float* in_host, float* out_host, void** graph_exec, void* stream, int Qd = 0, int Qe = 0) {
  GCCNMF_REQUIRE(h, graph_exec != nullptr && stream != nullptr, "rt_graph_create: needs a non-default stream and an output slot");
  *graph_exec = nullptr;
  RT_CARVE_OR_FAIL_B(l, S, P, Qd, Qe);
  GCCNMF_REQUIRE(h, in_blocks && out_blocks, "rt_graph_create: NULL pointer");
  const size_t block_bytes = (size_t)S * 2 * cfg->block_size * sizeof(float);
  auto enqueue = [&] { return rt_process_block(h, cfg, S, P, state, state_bytes, in_blocks, out_blocks, nullptr, stream, Qd, Qe); };
  return capture_graph(h, "rt_graph_create", stream, in_blocks, in_host, block_bytes, out_blocks, out_host, block_bytes * rt_sources_grid(l), enqueue,
                       graph_exec);
}

// Items 2 and 4 are source 0's with P > 0; items 9 .. 13 exist only with P > 0, item 14 only with a bank.  With a bank the
// K-shaped items (2, 5, 6, 10, 11) have the K_i of the block they were computed in (of the slot's current dictionary before its
// first block), read from the device after the work queued before.
int rt_export(gccnmf_handle* h, const gccnmf_rt_config* cfg, int S, int P, void* state, size_t state_bytes, int slot, int what, void* dst, void* stream,
              int Qd = 0, int Qe = 0) {
  RT_CARVE_OR_FAIL_B(l, S, P, Qd, Qe);
  GCCNMF_REQUIRE(h, dst != nullptr, "rt_export: NULL destination");
  GCCNMF_REQUIRE(h, slot >= 0 && slot < S, "rt_export: slot %d outside [0, %d)", slot, S);
  const size_t nT = cfg->windows_per_block, D = cfg->num_tdoas, F = l.F, st = l.stride;
  size_t K = cfg->num_atoms;
  const bool known = what >= 0 && (what < 9 || (P > 0 && what < 14) || (Qd > 0 && what == 14));
  if (known && Qd > 0 && (what == 2 || what == 5 || what == 6 || what == 10 || what == 11)) {
    int32_t entry[3] = {0, 0, 0}, Ki = 0;                // dictionary, steering, K_i of the last block computed (0: none yet)
    GCCNMF_CHECK_CUDA(h, cudaMemcpyAsync(entry, rt_slot(l.assign, slot, st), sizeof(entry), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
    GCCNMF_CHECK_CUDA(h, cudaStreamSynchronize((cudaStream_t)stream));
    Ki = entry[2];
    if (Ki == 0) {
      GCCNMF_CHECK_CUDA(h, cudaMemcpyAsync(&Ki, l.bank_K + entry[0], sizeof(Ki), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
      GCCNMF_CHECK_CUDA(h, cudaStreamSynchronize((cudaStream_t)stream));
    }
    K = (size_t)Ki;
  }
  const void* src = nullptr;
  size_t bytes = 0, rows = 1;            // rows > 1: one row of `bytes` per source, src_stride apart in the state
  switch (known ? what : -1) {
    case 0: src = rt_slot(l.gccphat, slot, st); bytes = D * nT * sizeof(float); break;
    case 1: src = &rt_slot(l.dev, slot, st)->target; bytes = sizeof(float); break;
    case 2: src = rt_slot(l.smask, slot, st); bytes = K * nT * sizeof(double); break;
    case 3: src = rt_slot(l.X, slot, st); bytes = 2 * F * nT * sizeof(float2); break;
    case 4: src = rt_slot(l.sY, slot, st); bytes = 2 * F * nT * sizeof(float2); break;
    case 5: src = rt_slot(l.argmax, slot, st); bytes = K * nT * sizeof(int32_t); break;
    case 6: src = rt_slot(l.H, slot, st); bytes = K * 2 * nT * sizeof(float); break;
    case 7: src = rt_slot(l.hist, slot, st); bytes = D * (size_t)cfg->history_length * sizeof(double); break;
    case 8: src = &rt_slot(l.dev, slot, st)->hist_index; bytes = sizeof(int); break;
    case 9: src = rt_slot(l.targets, slot, st); bytes = (size_t)P * sizeof(int32_t); break;
    case 10: src = rt_slot(l.smask, slot, st); bytes = K * nT * sizeof(double); rows = P; break;
    case 11: src = rt_slot(l.tval, slot, st); bytes = (size_t)P * K * nT * sizeof(float); break;
    case 12: src = rt_slot(l.sY, slot, st); bytes = 2 * F * nT * sizeof(float2); rows = P; break;
    case 13: src = rt_slot(l.status, slot, st); bytes = sizeof(int32_t); break;
    case 14: src = rt_slot(l.assign, slot, st); bytes = 2 * sizeof(int32_t); break;
    default: return gccnmf_fail(h, GCCNMF_ERR_INVALID_ARGUMENT, "rt_export: unknown item %d", what);
  }
  if (rows > 1)
    GCCNMF_CHECK_CUDA(h, cudaMemcpy2DAsync(dst, bytes, src, l.src_stride, bytes, rows, cudaMemcpyDefault, (cudaStream_t)stream));
  else
    GCCNMF_CHECK_CUDA(h, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDefault, (cudaStream_t)stream));
  return GCCNMF_OK;
}

// Per-slot parameters of slots [first_slot, first_slot + count): as given without sources; with P sources mode, target_index and
// set_target are ignored (the masks are one-hot, the targets come from set_targets or the localisation).
int rt_slot_params(gccnmf_handle* h, const gccnmf_rt_config* cfg, const RtLayout& l, int first_slot, int count, const gccnmf_rtm_slot_params* params,
                   void* stream) {
  const char* name = l.P > 0 ? "rtsep_set_params" : "rtm_set_params";
  if (int st = stream_range_check(h, name, l.S, first_slot, count)) return st;
  GCCNMF_REQUIRE(h, params != nullptr, "%s: NULL parameters", name);
  for (int i = 0; i < count; ++i) {
    GCCNMF_REQUIRE(h, l.P > 0 || params[i].mode == 0 || params[i].mode == 1, "%s: slot %d: mode must be 0 (boxcar) or 1 (window)", name, first_slot + i);
    GCCNMF_REQUIRE(h, params[i].localization_window >= 1, "%s: slot %d: localization_window must be >= 1 (got %d)", name, first_slot + i,
                   params[i].localization_window);
    // a strict local maximum needs both neighbours (argrelmax never returns the end points)
    GCCNMF_REQUIRE(h, l.P == 0 || !params[i].localization_enabled || cfg->num_tdoas >= 3, "%s: slot %d: localisation needs num_tdoas >= 3 (got %d)",
                   name, first_slot + i, cfg->num_tdoas);
  }
  if (l.P == 0) return rt_enqueue_params(h, l, first_slot, count, params, 1, stream);
  for (int i0 = 0; i0 < count; i0 += kRtParamsPerLaunch) {
    const int n = count - i0 < kRtParamsPerLaunch ? count - i0 : kRtParamsPerLaunch;
    gccnmf_rtm_slot_params p[kRtParamsPerLaunch];
    for (int i = 0; i < n; ++i) {
      p[i] = params[i0 + i];
      p[i].set_target = 0;
      p[i].mode = 1;
    }
    if (int st = rt_enqueue_params(h, l, first_slot + i0, n, p, 1, stream)) return st;
  }
  return GCCNMF_OK;
}

int rt_set_targets(gccnmf_handle* h, const gccnmf_rt_config* cfg, const RtLayout& l, int first_slot, int count, const int32_t* targets_host,
                   void* stream) {
  if (int st = stream_range_check(h, "rtsep_set_targets", l.S, first_slot, count)) return st;
  GCCNMF_REQUIRE(h, targets_host != nullptr, "rtsep_set_targets: NULL targets");
  const int P = l.P;
  for (int i = 0; i < count * P; ++i)
    GCCNMF_REQUIRE(h, targets_host[i] >= -1 && targets_host[i] < cfg->num_tdoas, "rtsep_set_targets: slot %d source %d: target %d outside [0, %d) (or -1)",
                   first_slot + i / P, i % P, targets_host[i], cfg->num_tdoas);
  return enqueue_stream_rows(h, l.targets, l.stride, 0, first_slot, count, P, targets_host, true, stream);
}

// ---------------------------------------------------------------------------------------------- stream records
// The persistent state of slot s is every byte a later block reads that an earlier block or a setting wrote:
//   dev[s]            parameters, block_counter (ring positions), hist_index, target, active   (set_params / defaults, synthesis, rt_localize)
//   hist[s]           the GCC-PHAT history ring, D x history_length f64                         (rt_localize)
//   in_ring[s]        the 8-block input ring of both channels                                   (rt_ola_emit -> rt_analysis)
//   out_ring[s]       the 8-block output ring of both channels; P > 0: sout of every source     (rt_ola_emit)
//   targets[s], status[s]   (P > 0)                                                             (rt_localize, set_targets -> rt_atoms)
// Everything else is shared by the slots (windows, dictionary and steering entries, what init derives from them, H0), rewritten
// by every block before it is read (G ... argmax, the masks, tval, the source Y and frames), or the slot's bank assignment, which
// a load writes from the entries it maps by content.  assign[2] (K_i of the last block computed) describes the destination's
// scratch and stays.  Region g of slot s is [offset + s stride, + bytes) from slot 0's region; it goes to [rec_offset, + bytes)
// of the record's payload, and [rec_offset + bytes, + span) of the record is zero.
static_assert(sizeof(RtDev) == 44, "RtDev");
constexpr size_t kRtRecordHeaderBytes = GCCNMF_RECORD_HEADER_BYTES;
static_assert(sizeof(gccnmf_rtrec_header) <= kRtRecordHeaderBytes, "record header");

// The state offsets follow the destination's carve (they depend on K_max through the scratch between the regions); the record
// offsets depend only on the configuration without num_atoms and on P.
RecordMap rt_record_map(const gccnmf_rt_config& c, int P, int Qd = 0, int Qe = 0) {
  const RtLayout l = rt_carve(c, 1, P, nullptr, 0, Qd, Qe);
  RecordMapBuilder b{l.dev, l.stride};
  b.add(l.dev, sizeof(RtDev));
  b.add(l.hist, (size_t)c.num_tdoas * c.history_length * sizeof(double));
  b.add(l.in_ring, (size_t)2 * l.L * sizeof(float));
  for (int q = 0; q < (P > 0 ? P : 1); ++q) b.add(rt_slot(l.sout, q, l.src_stride), (size_t)2 * l.L * sizeof(float));
  if (P > 0) {
    b.add(l.targets, kRtMaxSources * sizeof(int32_t));
    b.add(l.status, sizeof(int32_t));
  }
  return b.m;
}

size_t rt_record_bytes(const gccnmf_rt_config& c, int P) { return kRtRecordHeaderBytes + align_up(rt_record_map(c, P).payload, 256); }

// Grid (count, regions + 1).  CTA (i, g < regions) copies region g of slot first + i between the state and record i of the staging.
// CTA (i, regions), the header: a save writes the header (the host part `head`, the digests and K_i of the slot's entries, found
// through its assignment) and zeroes the header's tail and the payload's; a load maps the record's dictionary (digest and K_i) and
// steering digest to the lowest matching entry of this state, as the host did, and writes the slot's assignment (bank only).  The
// digests are item 0 the windows, items 1 .. nd the dictionaries and nd + 1 .. nd + ne the steering entries.
__global__ void __launch_bounds__(256)
rt_record_copy_kernel(char* __restrict__ slot0, size_t stride, int first, RecordMap m, char* __restrict__ staging, size_t rec_bytes, int to_staging,
                      gccnmf_rtrec_header head, const uint64_t* __restrict__ digest, const int32_t* __restrict__ atoms, int nd, int ne,
                      int32_t* __restrict__ assign0) {
  const int s = first + blockIdx.x;
  char* rec = staging + (size_t)blockIdx.x * rec_bytes;
  if (blockIdx.y < m.n) {
    record_copy_region(slot0, s, m.r[blockIdx.y], rec + kRtRecordHeaderBytes, to_staging);
    return;
  }
  int32_t* assign = assign0 ? rt_slot(assign0, s, stride) : nullptr;
  if (to_staging) {
    for (size_t i = sizeof(head) / 4 + threadIdx.x; i < kRtRecordHeaderBytes / 4; i += blockDim.x) reinterpret_cast<uint32_t*>(rec)[i] = 0;
    for (size_t i = (kRtRecordHeaderBytes + m.payload) / 4 + threadIdx.x; i < rec_bytes / 4; i += blockDim.x) reinterpret_cast<uint32_t*>(rec)[i] = 0;
    if (threadIdx.x == 0) {
      const int di = assign ? assign[0] : 0, ej = assign ? assign[1] : 0;
      head.windows_digest = digest[0];
      head.dictionary_digest = digest[1 + di];
      head.steering_digest = digest[1 + nd + ej];
      head.dictionary_atoms = atoms[1 + di];
      *reinterpret_cast<gccnmf_rtrec_header*>(rec) = head;
    }
  } else if (threadIdx.x == 0 && assign) {
    const gccnmf_rtrec_header got = *reinterpret_cast<const gccnmf_rtrec_header*>(rec);
    const int di = record_find_entry(digest + 1, atoms + 1, nd, got.dictionary_digest, got.dictionary_atoms);
    const int ej = record_find_entry(digest + 1 + nd, nullptr, ne, got.steering_digest, 0);
    if (di >= 0 && ej >= 0) assign[0] = di, assign[1] = ej;
  }
}

// What a record must agree on from the host arguments alone: magic, ABI version, kind, P, payload size and the configuration
// without num_atoms.  The digests and K_i are the device's.
gccnmf_rtrec_header rt_record_header(const gccnmf_rt_config& cfg, int P) {
  gccnmf_rtrec_header r{};
  r.magic = GCCNMF_RECORD_MAGIC;
  r.abi_version = GCCNMF_ABI_VERSION;
  r.kind = GCCNMF_RECORD_KIND_RT;
  r.num_sources = P;
  r.payload_bytes = rt_record_map(cfg, P).payload;
  gccnmf_rt_config c = cfg;
  c.num_atoms = 0;
  static_assert(sizeof(c) <= sizeof(r.config), "record config");
  memcpy(r.config, &c, sizeof(c));
  return r;
}

// The digest items of a state: the windows, its nd dictionaries (nd = ne = 1 without a bank) and its ne steering entries, each with
// chunk slots for K_max atoms.  The workspace: count whole records, then the chunk digests, the item digests and the items' K_i.
struct RtRecordWork {
  DigestItems d;
  int nd, ne;
  size_t chunks, digests, atoms, bytes;
};
RtRecordWork rt_record_work(const gccnmf_rt_config& c, const RtLayout& l, int count) {
  RtRecordWork w{};
  const size_t N = c.window_size, F = l.F, K = c.num_atoms, inf = c.inference_iterations > 0 ? 1 : 0, et_words = (size_t)2 * l.D * l.Fp;
  w.nd = l.Qd > 0 ? l.Qd : 1;
  w.ne = l.Qe > 0 ? l.Qe : 1;
  const int cd = digest_chunks(F * K + 2 * K * inf);
  w.d.g[0] = DigestGroup{l.win_a, l.win_s, 0, 0, N, N, nullptr, 0, 1, digest_chunks(2 * N)};
  w.d.g[1] = l.bank_K ? DigestGroup{l.W, l.H0, l.bank.dict_stride, l.bank.dict_stride, F, 2 * inf, l.bank_K, 0, w.nd, cd}
                      : DigestGroup{l.W, l.H0, 0, 0, F * K, 2 * K * inf, nullptr, (int)K, 1, cd};
  w.d.g[2] = DigestGroup{l.ET, nullptr, l.bank.steer_stride, 0, et_words, 0, nullptr, 0, w.ne, digest_chunks(et_words)};
  w.d.n = 3;
  int slots = 0;
  for (const DigestGroup& g : w.d.g) slots += g.count * g.chunks;
  const int items = 1 + w.nd + w.ne;
  w.chunks = align_up((size_t)count * rt_record_bytes(c, l.P), 256);
  w.digests = w.chunks + align_up((size_t)slots * sizeof(uint64_t), 256);
  w.atoms = w.digests + align_up((size_t)items * sizeof(uint64_t), 256);
  w.bytes = w.atoms + align_up((size_t)items * sizeof(int32_t), 256);
  return w;
}

int rt_enqueue_digests(gccnmf_handle* h, const RtRecordWork& w, char* workspace, void* stream) {
  return record_enqueue_digests(h, w.d, reinterpret_cast<uint64_t*>(workspace + w.chunks), reinterpret_cast<uint64_t*>(workspace + w.digests),
                                reinterpret_cast<int32_t*>(workspace + w.atoms), stream);
}

#define RT_RECORD_ARGS_OR_FAIL(what)                                                                                               \
  const bool empty__ = Qd == 0 && Qe == 0;                                                                                         \
  if (!empty__)                                                                                                                    \
    if (int st__ = rt_check_bank(h, Qd, Qe)) return st__;                                                                          \
  RT_CARVE_OR_FAIL_B(l, S, P, Qd, Qe);                                                                                             \
  if (int st__ = stream_range_check(h, what, S, first, count)) return st__;                                                      \
  const RecordMap m = rt_record_map(*cfg, P, Qd, Qe);                                                                              \
  const size_t rec_bytes = rt_record_bytes(*cfg, P);                                                                               \
  GCCNMF_REQUIRE(h, record != nullptr && record_bytes >= (size_t)count * rec_bytes, what ": record needs %zu bytes for %d slots",  \
                 (size_t)count * rec_bytes, count);                                                                                \
  const RtRecordWork w = rt_record_work(*cfg, l, count);                                                                           \
  if (workspace == nullptr || workspace_bytes < w.bytes || ((uintptr_t)workspace & 15) != 0)                                       \
    return gccnmf_fail(h, GCCNMF_ERR_WORKSPACE, what ": workspace needs %zu bytes, 16-byte aligned", w.bytes);                     \
  char* ws = static_cast<char*>(workspace)

int rt_save_slots(gccnmf_handle* h, const gccnmf_rt_config* cfg, int S, int P, int Qd, int Qe, void* state, size_t state_bytes, int first, int count,
                  void* record, size_t record_bytes, void* workspace, size_t workspace_bytes, void* stream) {
  GCCNMF_ENTER(h);
  RT_RECORD_ARGS_OR_FAIL("rtrec_save_slots");
  if (int st = rt_enqueue_digests(h, w, ws, stream)) return st;
  GCCNMF_LAUNCH(h, rt_record_copy_kernel, dim3(count, m.n + 1), 256, 0, stream, reinterpret_cast<char*>(l.dev), l.stride, first, m, ws, rec_bytes, 1,
                rt_record_header(*cfg, P), reinterpret_cast<const uint64_t*>(ws + w.digests), reinterpret_cast<const int32_t*>(ws + w.atoms), w.nd,
                w.ne, l.assign);
  GCCNMF_CHECK_CUDA(h, cudaMemcpyAsync(record, ws, (size_t)count * rec_bytes, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  return GCCNMF_OK;
}

int rt_load_slots(gccnmf_handle* h, const gccnmf_rt_config* cfg, int S, int P, int Qd, int Qe, void* state, size_t state_bytes, int first, int count,
                  const void* record, size_t record_bytes, void* workspace, size_t workspace_bytes, void* stream) {
  GCCNMF_ENTER(h);
  RT_RECORD_ARGS_OR_FAIL("rtrec_load_slots");
  const gccnmf_rtrec_header want = rt_record_header(*cfg, P);
  for (int i = 0; i < count; ++i) {      // the host fields, before the device is touched
    gccnmf_rtrec_header got;
    memcpy(&got, (const char*)record + (size_t)i * rec_bytes, sizeof(got));
    if (int st = record_check_header(h, "rtrec_load_slots", i, &got, &want, offsetof(gccnmf_rtrec_header, config))) return st;
    GCCNMF_REQUIRE(h, got.reserved == 0, "rtrec_load_slots: record %d: reserved word %d", i, got.reserved);
  }
  // the destination's digests and K_i, read back once
  if (int st = rt_enqueue_digests(h, w, ws, stream)) return st;
  const int nd = w.nd, ne = w.ne, items = 1 + nd + ne;
  uint64_t digest[1 + 2 * kRtMaxBank];
  int32_t atoms[1 + 2 * kRtMaxBank];
  cudaStream_t s = (cudaStream_t)stream;
  GCCNMF_CHECK_CUDA(h, cudaMemcpyAsync(digest, ws + w.digests, items * sizeof(uint64_t), cudaMemcpyDeviceToHost, s));
  GCCNMF_CHECK_CUDA(h, cudaMemcpyAsync(atoms, ws + w.atoms, items * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  GCCNMF_CHECK_CUDA(h, cudaStreamSynchronize(s));
  for (int r = 0; r < count; ++r) {
    gccnmf_rtrec_header got;
    memcpy(&got, (const char*)record + (size_t)r * rec_bytes, sizeof(got));
    GCCNMF_REQUIRE(h, got.windows_digest == digest[0], "rtrec_load_slots: record %d: other analysis / synthesis windows", r);
    GCCNMF_REQUIRE(h, record_find_entry(digest + 1, atoms + 1, nd, got.dictionary_digest, got.dictionary_atoms) >= 0,
                   "rtrec_load_slots: record %d: no dictionary entry of this engine holds its dictionary (%d atoms)", r, got.dictionary_atoms);
    GCCNMF_REQUIRE(h, record_find_entry(digest + 1 + nd, nullptr, ne, got.steering_digest, 0) >= 0,
                   "rtrec_load_slots: record %d: no steering entry of this engine holds its steering table", r);
  }
  GCCNMF_CHECK_CUDA(h, cudaMemcpyAsync(ws, record, (size_t)count * rec_bytes, cudaMemcpyHostToDevice, s));
  GCCNMF_LAUNCH(h, rt_record_copy_kernel, dim3(count, m.n + 1), 256, 0, stream, reinterpret_cast<char*>(l.dev), l.stride, first, m, ws, rec_bytes, 0,
                want, reinterpret_cast<const uint64_t*>(ws + w.digests), reinterpret_cast<const int32_t*>(ws + w.atoms), nd, ne, l.assign);
  return rt_enqueue_sort(h, l, stream);
}

}  // namespace

extern "C" {

// ---------------------------------------------------------------------------------------------- single stream (S = 1)
size_t gccnmf_rt_state_bytes(const gccnmf_rt_config* cfg) {
  if (!cfg || cfg->window_size < 2 || cfg->block_size < 1 || cfg->windows_per_block < 1 || cfg->num_atoms < 1 || cfg->num_tdoas < 1 ||
      cfg->history_length < 1)
    return 0;
  return rt_carve(*cfg, 1, 0, nullptr, 0).bytes;
}

// W (F, K) f32, E (F, D) complex64 (expJOmegaTau, gccNMFProcessor.py:248), windows (N) f32, H0 (K, 2) f32 or NULL (all device pointers).
int gccnmf_rt_init(gccnmf_handle* h, const gccnmf_rt_config* cfg, const float* W, const float* E, const float* analysis_window,
                   const float* synthesis_window, const float* H0, void* state, size_t state_bytes, void* stream) {
  GCCNMF_ENTER(h);
  return rt_init(h, cfg, 1, 0, W, E, analysis_window, synthesis_window, H0, state, state_bytes, stream);
}

// setTargetTDOARange (:272-276) + the settable attributes (:136-151).  set_target = 0 leaves the target TDOA index alone (it is
// loop-carried device state when localisation is on).
int gccnmf_rt_set_params(gccnmf_handle* h, const gccnmf_rt_config* cfg, void* state, size_t state_bytes, float target_index, int set_target,
                         float epsilon, float beta, float noise_floor, int mode, int separation_enabled, int localization_enabled,
                         int localization_window, void* stream) {
  GCCNMF_ENTER(h);
  RT_CARVE_OR_FAIL(l, 1);
  GCCNMF_REQUIRE(h, mode == 0 || mode == 1, "rt_set_params: mode must be 0 (boxcar) or 1 (window)");
  // gccPHATHistory[:, -w:] (:221) takes the last w columns only for w >= 1; w = 0 would take the whole history
  GCCNMF_REQUIRE(h, localization_window >= 1, "rt_set_params: localization_window must be >= 1 (got %d)", localization_window);
  const gccnmf_rtm_slot_params p{target_index, set_target, epsilon, beta, noise_floor, mode, separation_enabled, localization_enabled,
                                 localization_window, 1};
  return rt_enqueue_params(h, l, 0, 1, &p, 0, stream);
}

// GCCNMFProcessor.processFrames (:201-231): windowed (2, N, nT) f32 -> out (2, N, nT) f32, both on the device.
int gccnmf_rt_process_frames(gccnmf_handle* h, const gccnmf_rt_config* cfg, void* state, size_t state_bytes, const float* windowed, float* out,
                             const double* forced_atom_mask, void* stream) {
  GCCNMF_ENTER(h);
  return rt_process_frames(h, cfg, 1, 0, state, state_bytes, windowed, out, forced_atom_mask, stream);
}

// OverlapAddProcessor.processFrames(GCCNMFProcessor.processFrames) (utils.py:99-116 around gccNMFProcessor.py:201-231):
// in_block (2, B) f32 -> out_block (2, B) f32 (the block emitted is the one pushed in two calls earlier).
int gccnmf_rt_process_block(gccnmf_handle* h, const gccnmf_rt_config* cfg, void* state, size_t state_bytes, const float* in_block, float* out_block,
                            const double* forced_atom_mask, void* stream) {
  GCCNMF_ENTER(h);
  return rt_process_block(h, cfg, 1, 0, state, state_bytes, in_block, out_block, forced_atom_mask, stream);
}

// One block as a CUDA graph: [H2D of in_host ->] the kernels of gccnmf_rt_process_block [-> D2H to out_host].  in_block / out_block
// are device staging buffers (2, B); in_host / out_host pinned host buffers or NULL.  *graph_exec is a cudaGraphExec_t.
int gccnmf_rt_graph_create(gccnmf_handle* h, const gccnmf_rt_config* cfg, void* state, size_t state_bytes, float* in_block, float* out_block,
                           const float* in_host, float* out_host, void** graph_exec, void* stream) {
  GCCNMF_ENTER(h);
  return rt_graph_create(h, cfg, 1, 0, state, state_bytes, in_block, out_block, in_host, out_host, graph_exec, stream);
}

int gccnmf_rt_graph_launch(gccnmf_handle* h, void* graph_exec, void* stream) {
  GCCNMF_ENTER(h);
  GCCNMF_REQUIRE(h, graph_exec != nullptr, "rt_graph_launch: NULL graph");
  GCCNMF_CHECK_CUDA(h, cudaGraphLaunch((cudaGraphExec_t)graph_exec, (cudaStream_t)stream));
  h->launches++;
  return GCCNMF_OK;
}

int gccnmf_rt_graph_destroy(gccnmf_handle* h, void* graph_exec) {
  GCCNMF_ENTER(h);
  if (graph_exec) GCCNMF_CHECK_CUDA(h, cudaGraphExecDestroy((cudaGraphExec_t)graph_exec));
  return GCCNMF_OK;
}

// Copies one piece of the block state to dst (device or pinned host memory, cudaMemcpyDefault), stream-ordered:
//   0 gccPHAT (D, nT) f32   1 target TDOA index (1) f32   2 atom mask (K, nT) f64   3 input spectrogram X (2, F, nT) c64
//   4 output spectrogram (2, F, nT) c64   5 TDOA argmax per atom (K, nT) i32   6 inferred coefficients H (K, 2 nT) f32
//   7 GCC-PHAT history ring (D, history_length) f64 followed by nothing (its write index is item 8)   8 history write index (1) i32
int gccnmf_rt_export(gccnmf_handle* h, const gccnmf_rt_config* cfg, void* state, size_t state_bytes, int what, void* dst, void* stream) {
  GCCNMF_ENTER(h);
  return rt_export(h, cfg, 1, 0, state, state_bytes, 0, what, dst, stream);
}

// ---------------------------------------------------------------------------------------------- S streams (slots) in one state
size_t gccnmf_rtm_state_bytes(const gccnmf_rt_config* cfg, int num_streams) {
  if (rt_check(nullptr, cfg, num_streams) != 0) return 0;
  return rt_carve(*cfg, num_streams, 0, nullptr, 0).bytes;
}

int gccnmf_rtm_init(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, const float* W, const float* E, const float* analysis_window,
                    const float* synthesis_window, const float* H0, void* state, size_t state_bytes, void* stream) {
  GCCNMF_ENTER(h);
  return rt_init(h, cfg, num_streams, 0, W, E, analysis_window, synthesis_window, H0, state, state_bytes, stream);
}

int gccnmf_rtm_reset_slots(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, void* state, size_t state_bytes, int first_slot, int count,
                           void* stream) {
  GCCNMF_ENTER(h);
  RT_CARVE_OR_FAIL(l, num_streams);
  if (int st = stream_range_check(h, "rtm_reset_slots", num_streams, first_slot, count)) return st;
  return rt_enqueue_reset(h, l, first_slot, count, stream);
}

int gccnmf_rtm_set_params(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, void* state, size_t state_bytes, int first_slot, int count,
                          const gccnmf_rtm_slot_params* params, void* stream) {
  GCCNMF_ENTER(h);
  RT_CARVE_OR_FAIL(l, num_streams);
  return rt_slot_params(h, cfg, l, first_slot, count, params, stream);
}

int gccnmf_rtm_process_frames(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, void* state, size_t state_bytes, const float* windowed,
                              float* out, const double* forced_atom_mask, void* stream) {
  GCCNMF_ENTER(h);
  return rt_process_frames(h, cfg, num_streams, 0, state, state_bytes, windowed, out, forced_atom_mask, stream);
}

int gccnmf_rtm_process_block(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, void* state, size_t state_bytes, const float* in_blocks,
                             float* out_blocks, const double* forced_atom_mask, void* stream) {
  GCCNMF_ENTER(h);
  return rt_process_block(h, cfg, num_streams, 0, state, state_bytes, in_blocks, out_blocks, forced_atom_mask, stream);
}

int gccnmf_rtm_graph_create(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, void* state, size_t state_bytes, float* in_blocks,
                            float* out_blocks, const float* in_host, float* out_host, void** graph_exec, void* stream) {
  GCCNMF_ENTER(h);
  return rt_graph_create(h, cfg, num_streams, 0, state, state_bytes, in_blocks, out_blocks, in_host, out_host, graph_exec, stream);
}

int gccnmf_rtm_export(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, void* state, size_t state_bytes, int slot, int what, void* dst,
                      void* stream) {
  GCCNMF_ENTER(h);
  return rt_export(h, cfg, num_streams, 0, state, state_bytes, slot, what, dst, stream);
}

// ---------------------------------------------------------------------------------------------- S streams x P sources
size_t gccnmf_rtsep_state_bytes(const gccnmf_rt_config* cfg, int num_streams, int num_sources) {
  if (num_sources == 0 || rt_check(nullptr, cfg, num_streams, num_sources) != 0) return 0;
  return rt_carve(*cfg, num_streams, num_sources, nullptr, 0).bytes;
}

int gccnmf_rtsep_init(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, int num_sources, const float* W, const float* E,
                      const float* analysis_window, const float* synthesis_window, const float* H0, void* state, size_t state_bytes, void* stream) {
  GCCNMF_ENTER(h);
  GCCNMF_REQUIRE(h, num_sources != 0, "rtsep: num_sources must be in [2, %d] (got 0)", kRtMaxSources);
  return rt_init(h, cfg, num_streams, num_sources, W, E, analysis_window, synthesis_window, H0, state, state_bytes, stream);
}

int gccnmf_rtsep_reset_slots(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, int num_sources, void* state, size_t state_bytes,
                             int first_slot, int count, void* stream) {
  GCCNMF_ENTER(h);
  GCCNMF_REQUIRE(h, num_sources != 0, "rtsep: num_sources must be in [2, %d] (got 0)", kRtMaxSources);
  RT_CARVE_OR_FAIL_P(l, num_streams, num_sources);
  if (int st = stream_range_check(h, "rtsep_reset_slots", num_streams, first_slot, count)) return st;
  return rt_enqueue_reset(h, l, first_slot, count, stream);
}

// mode, target_index and set_target are ignored: the sources' masks are one-hot by construction and their targets come from
// gccnmf_rtsep_set_targets or the localisation.
int gccnmf_rtsep_set_params(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, int num_sources, void* state, size_t state_bytes,
                            int first_slot, int count, const gccnmf_rtm_slot_params* params, void* stream) {
  GCCNMF_ENTER(h);
  GCCNMF_REQUIRE(h, num_sources != 0, "rtsep: num_sources must be in [2, %d] (got 0)", kRtMaxSources);
  RT_CARVE_OR_FAIL_P(l, num_streams, num_sources);
  return rt_slot_params(h, cfg, l, first_slot, count, params, stream);
}

int gccnmf_rtsep_set_targets(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, int num_sources, void* state, size_t state_bytes,
                             int first_slot, int count, const int32_t* targets_host, void* stream) {
  GCCNMF_ENTER(h);
  GCCNMF_REQUIRE(h, num_sources != 0, "rtsep: num_sources must be in [2, %d] (got 0)", kRtMaxSources);
  RT_CARVE_OR_FAIL_P(l, num_streams, num_sources);
  return rt_set_targets(h, cfg, l, first_slot, count, targets_host, stream);
}

int gccnmf_rtsep_process_frames(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, int num_sources, void* state, size_t state_bytes,
                                const float* windowed, float* out, void* stream) {
  GCCNMF_ENTER(h);
  GCCNMF_REQUIRE(h, num_sources != 0, "rtsep: num_sources must be in [2, %d] (got 0)", kRtMaxSources);
  return rt_process_frames(h, cfg, num_streams, num_sources, state, state_bytes, windowed, out, nullptr, stream);
}

int gccnmf_rtsep_process_block(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, int num_sources, void* state, size_t state_bytes,
                               const float* in_blocks, float* out_blocks, void* stream) {
  GCCNMF_ENTER(h);
  GCCNMF_REQUIRE(h, num_sources != 0, "rtsep: num_sources must be in [2, %d] (got 0)", kRtMaxSources);
  return rt_process_block(h, cfg, num_streams, num_sources, state, state_bytes, in_blocks, out_blocks, nullptr, stream);
}

int gccnmf_rtsep_graph_create(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, int num_sources, void* state, size_t state_bytes,
                              float* in_blocks, float* out_blocks, const float* in_host, float* out_host, void** graph_exec, void* stream) {
  GCCNMF_ENTER(h);
  GCCNMF_REQUIRE(h, num_sources != 0, "rtsep: num_sources must be in [2, %d] (got 0)", kRtMaxSources);
  return rt_graph_create(h, cfg, num_streams, num_sources, state, state_bytes, in_blocks, out_blocks, in_host, out_host, graph_exec, stream);
}

int gccnmf_rtsep_export(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, int num_sources, void* state, size_t state_bytes, int slot,
                        int what, void* dst, void* stream) {
  GCCNMF_ENTER(h);
  GCCNMF_REQUIRE(h, num_sources != 0, "rtsep: num_sources must be in [2, %d] (got 0)", kRtMaxSources);
  return rt_export(h, cfg, num_streams, num_sources, state, state_bytes, slot, what, dst, stream);
}


// ---------------------------------------------------------------------------------------------- S streams x P sources over a bank
// of Qd dictionaries and Qe steering tables
#define RT_BANK_OR_FAIL(l)                                                                                                         \
  if (int st__ = rt_check_bank(h, num_dictionaries, num_steerings)) return st__;                                                  \
  RT_CARVE_OR_FAIL_B(l, num_streams, num_sources, num_dictionaries, num_steerings)

size_t gccnmf_rtbank_state_bytes(const gccnmf_rt_config* cfg, int num_streams, int num_sources, int num_dictionaries, int num_steerings) {
  const bool empty = num_dictionaries == 0 && num_steerings == 0;
  if (!empty && rt_check_bank(nullptr, num_dictionaries, num_steerings) != 0) return 0;
  if (rt_check(nullptr, cfg, num_streams, num_sources) != 0) return 0;
  return rt_carve(*cfg, num_streams, num_sources, nullptr, 0, num_dictionaries, num_steerings).bytes;
}

int gccnmf_rtbank_init(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, int num_sources, int num_dictionaries, int num_steerings,
                       void* state, size_t state_bytes, const float* const* W, const int* num_atoms, const float* const* H0, const float* const* E,
                       const float* analysis_window, const float* synthesis_window, void* stream) {
  GCCNMF_ENTER(h);
  if (int st = rt_check_bank(h, num_dictionaries, num_steerings)) return st;
  return rt_init(h, cfg, num_streams, num_sources, num_dictionaries, num_steerings, W, num_atoms, H0, E, analysis_window, synthesis_window, state,
                 state_bytes, stream);
}

int gccnmf_rtbank_load_dictionary(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, int num_sources, int num_dictionaries,
                                  int num_steerings, void* state, size_t state_bytes, int index, const float* W, int num_atoms, const float* H0,
                                  void* stream) {
  GCCNMF_ENTER(h);
  RT_BANK_OR_FAIL(l);
  GCCNMF_REQUIRE(h, index >= 0 && index < num_dictionaries, "rtbank_load_dictionary: entry %d outside [0, %d)", index, num_dictionaries);
  GCCNMF_REQUIRE(h, num_atoms >= 1 && num_atoms <= cfg->num_atoms, "rtbank_load_dictionary: %d atoms outside [1, num_atoms = %d]", num_atoms,
                 cfg->num_atoms);
  GCCNMF_REQUIRE(h, W != nullptr, "rtbank_load_dictionary: NULL dictionary");
  GCCNMF_REQUIRE(h, cfg->inference_iterations == 0 || H0 != nullptr, "rtbank_load_dictionary: coefficient inference needs the initial H0 (K, 2)");
  return rt_enqueue_dictionary(h, l, index, W, num_atoms, H0, stream);
}

int gccnmf_rtbank_load_steering(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, int num_sources, int num_dictionaries, int num_steerings,
                                void* state, size_t state_bytes, int index, const float* E, void* stream) {
  GCCNMF_ENTER(h);
  RT_BANK_OR_FAIL(l);
  GCCNMF_REQUIRE(h, index >= 0 && index < num_steerings, "rtbank_load_steering: entry %d outside [0, %d)", index, num_steerings);
  GCCNMF_REQUIRE(h, E != nullptr, "rtbank_load_steering: NULL steering table");
  return rt_enqueue_steering(h, l, index, E, stream);
}

int gccnmf_rtbank_assign(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, int num_sources, int num_dictionaries, int num_steerings,
                         void* state, size_t state_bytes, int first_slot, int count, const int32_t* dictionary, const int32_t* steering, void* stream) {
  GCCNMF_ENTER(h);
  RT_BANK_OR_FAIL(l);
  if (int st = stream_range_check(h, "rtbank_assign", num_streams, first_slot, count)) return st;
  for (int i = 0; i < count; ++i) {
    GCCNMF_REQUIRE(h, !dictionary || (dictionary[i] >= -1 && dictionary[i] < num_dictionaries),
                   "rtbank_assign: slot %d: dictionary %d outside [0, %d) (or -1)", first_slot + i, dictionary[i], num_dictionaries);
    GCCNMF_REQUIRE(h, !steering || (steering[i] >= -1 && steering[i] < num_steerings), "rtbank_assign: slot %d: steering %d outside [0, %d) (or -1)",
                   first_slot + i, steering[i], num_steerings);
  }
  std::vector<int32_t> rows(2 * (size_t)count);         // (dictionary, steering) per slot; a NULL array keeps
  for (int i = 0; i < count; ++i) {
    rows[2 * i] = dictionary ? dictionary[i] : -1;
    rows[2 * i + 1] = steering ? steering[i] : -1;
  }
  if (int st = enqueue_stream_rows(h, l.assign, l.stride, 0, first_slot, count, 2, rows.data(), true, stream)) return st;
  return rt_enqueue_sort(h, l, stream);
}

int gccnmf_rtbank_reset_slots(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, int num_sources, int num_dictionaries, int num_steerings,
                              void* state, size_t state_bytes, int first_slot, int count, void* stream) {
  GCCNMF_ENTER(h);
  RT_BANK_OR_FAIL(l);
  if (int st = stream_range_check(h, "rtbank_reset_slots", num_streams, first_slot, count)) return st;
  return rt_enqueue_reset(h, l, first_slot, count, stream);
}

int gccnmf_rtbank_set_params(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, int num_sources, int num_dictionaries, int num_steerings,
                             void* state, size_t state_bytes, int first_slot, int count, const gccnmf_rtm_slot_params* params, void* stream) {
  GCCNMF_ENTER(h);
  RT_BANK_OR_FAIL(l);
  return rt_slot_params(h, cfg, l, first_slot, count, params, stream);
}

int gccnmf_rtbank_set_targets(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, int num_sources, int num_dictionaries, int num_steerings,
                              void* state, size_t state_bytes, int first_slot, int count, const int32_t* targets_host, void* stream) {
  GCCNMF_ENTER(h);
  GCCNMF_REQUIRE(h, num_sources != 0, "rtbank_set_targets: needs num_sources in [2, %d] (got 0)", kRtMaxSources);
  RT_BANK_OR_FAIL(l);
  return rt_set_targets(h, cfg, l, first_slot, count, targets_host, stream);
}

int gccnmf_rtbank_process_frames(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, int num_sources, int num_dictionaries,
                                 int num_steerings, void* state, size_t state_bytes, const float* windowed, float* out, const double* forced_atom_mask,
                                 void* stream) {
  GCCNMF_ENTER(h);
  if (int st = rt_check_bank(h, num_dictionaries, num_steerings)) return st;
  GCCNMF_REQUIRE(h, num_sources == 0 || !forced_atom_mask, "rtbank_process_frames: forced atom masks need num_sources = 0");
  return rt_process_frames(h, cfg, num_streams, num_sources, state, state_bytes, windowed, out, forced_atom_mask, stream, num_dictionaries, num_steerings);
}

int gccnmf_rtbank_process_block(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, int num_sources, int num_dictionaries, int num_steerings,
                                void* state, size_t state_bytes, const float* in_blocks, float* out_blocks, const double* forced_atom_mask, void* stream) {
  GCCNMF_ENTER(h);
  if (int st = rt_check_bank(h, num_dictionaries, num_steerings)) return st;
  GCCNMF_REQUIRE(h, num_sources == 0 || !forced_atom_mask, "rtbank_process_block: forced atom masks need num_sources = 0");
  return rt_process_block(h, cfg, num_streams, num_sources, state, state_bytes, in_blocks, out_blocks, forced_atom_mask, stream, num_dictionaries,
                          num_steerings);
}

int gccnmf_rtbank_graph_create(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, int num_sources, int num_dictionaries, int num_steerings,
                               void* state, size_t state_bytes, float* in_blocks, float* out_blocks, const float* in_host, float* out_host,
                               void** graph_exec, void* stream) {
  GCCNMF_ENTER(h);
  if (int st = rt_check_bank(h, num_dictionaries, num_steerings)) return st;
  return rt_graph_create(h, cfg, num_streams, num_sources, state, state_bytes, in_blocks, out_blocks, in_host, out_host, graph_exec, stream,
                         num_dictionaries, num_steerings);
}

int gccnmf_rtbank_export(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, int num_sources, int num_dictionaries, int num_steerings,
                         void* state, size_t state_bytes, int slot, int what, void* dst, void* stream) {
  GCCNMF_ENTER(h);
  if (int st = rt_check_bank(h, num_dictionaries, num_steerings)) return st;
  return rt_export(h, cfg, num_streams, num_sources, state, state_bytes, slot, what, dst, stream, num_dictionaries, num_steerings);
}

// ---------------------------------------------------------------------------------------------- stream records of every form
// (num_streams, num_sources, num_dictionaries, num_steerings): (1, 0, 0, 0) gccnmf_rt_*, (S, 0, 0, 0) rtm, (S, P, 0, 0) rtsep, else a bank
size_t gccnmf_rtrec_record_bytes(const gccnmf_rt_config* cfg, int num_sources) {
  if (rt_check(nullptr, cfg, 1, num_sources) != 0) return 0;
  return rt_record_bytes(*cfg, num_sources);
}

size_t gccnmf_rtrec_workspace_bytes(const gccnmf_rt_config* cfg, int num_streams, int num_sources, int num_dictionaries, int num_steerings, int count) {
  const bool empty = num_dictionaries == 0 && num_steerings == 0;
  if ((!empty && rt_check_bank(nullptr, num_dictionaries, num_steerings) != 0) || rt_check(nullptr, cfg, num_streams, num_sources) != 0 || count < 1)
    return 0;
  const RtLayout l = rt_carve(*cfg, num_streams, num_sources, nullptr, 0, num_dictionaries, num_steerings);
  return rt_record_work(*cfg, l, count).bytes;
}

int gccnmf_rtrec_save_slots(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, int num_sources, int num_dictionaries, int num_steerings,
                            void* state, size_t state_bytes, int first, int count, void* record, size_t record_bytes, void* workspace,
                            size_t workspace_bytes, void* stream) {
  return rt_save_slots(h, cfg, num_streams, num_sources, num_dictionaries, num_steerings, state, state_bytes, first, count, record, record_bytes,
                       workspace, workspace_bytes, stream);
}

int gccnmf_rtrec_load_slots(gccnmf_handle* h, const gccnmf_rt_config* cfg, int num_streams, int num_sources, int num_dictionaries, int num_steerings,
                            void* state, size_t state_bytes, int first, int count, const void* record, size_t record_bytes, void* workspace,
                            size_t workspace_bytes, void* stream) {
  return rt_load_slots(h, cfg, num_streams, num_sources, num_dictionaries, num_steerings, state, state_bytes, first, count, record, record_bytes,
                       workspace, workspace_bytes, stream);
}

}  // extern "C"
