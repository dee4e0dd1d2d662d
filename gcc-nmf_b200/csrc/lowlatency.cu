// The online / low-latency notebook loop (onlineSpeechEnhancement.ipynb:406-447, lowLatencySpeechEnhancement.ipynb:511-584) for
// S independent streams, one hop at a time, computing what performOnlineSpeechEnhancement computes in batch (online.py).
//
// A call pushes `hops` hops per stream and runs, in stream order and without a host synchronisation:
//   ll_push        input ring (last N - hop samples) + new samples -> a linear staging row per stream and channel
//   stft           every frame of the call straight from the staging rows (stft.cu's per-frame float64 FFT, so a frame's bits do
//                  not depend on how many frames share the launch)                                  -> X (2, F, T), T = S hops
//   phat_angspec   coherence + angular spectrum (gcc.cu, per column)
//   ll_targets     running maximum from the carried one, target = argmax (gccnmf_online_targets' comparisons), carry stored
//   tdoa_argmax    all-TDOA GCC-NMF argmax per atom (gcc_tc.cu), then the gated float64 launch (gcc.cu) that redoes every decision
//                  when the refinement list overflowed -- the host fallback of online.py cannot run inside a graph
//   ll_mask        boxcar atom mask with the stream's epsilon (atom_mask_kernel mode 0's arithmetic)
//   ll_infer       (inference only) H-only KL updates of each frame's (K, 2) coefficients from H0, in a fixed order per column
//   wiener         wiener_apply / wiener_apply_h (gcc.cu, per column)
//   istft frames   the per-frame inverse FFT of istft_ola (stft.cu)
//   ll_ola_emit    acc = float32(fma(w[r], frame[r], acc)) into an N-sample output ring in frame order, emit gain x acc, zero the
//                  emitted positions, move the input ring on
// Every column is computed on its own in each stage, so the result of a stream does not depend on the other streams or on how its
// samples are split into calls.
//
// With P sources per stream (gccnmf_llsep_*) the stages after phat_angspec are instead:
//   ll_src_targets     running maximum as above, then per frame the P largest peaks of it (select_peaks) as the stream's targets,
//                      held when there are fewer (status bit 0); overrides replace them    -> column targets (T, P)
//   target_gccnmf      the float64 GCC-NMF values at each column's P targets (gcc.cu)      -> values (P, K, T)
//   coeff_mask         one-hot masks per source (gcc.cu); an all-NaN (k, t) goes to no source and sets bit 1 of the call's status
//   ll_infer           (inference only) once per column, H shared by the sources
//   wiener             per source, with its mask
//   istft frames       one launch over the (P, 2) spectra
//   ll_src_ola_emit    per (stream, source): ll_ola_emit_kernel's overlap-add and emit into the source's own ring
//   ll_src_advance     per stream, after every source has emitted: the input ring and the hop count move on
//
// With a history of Lh > 0 frames per stream (gccnmf_llhist_*) the targets stage is ll_hist_targets / ll_hist_src_targets instead:
// the running maximum as above, every valid frame's angular column into the stream's (D, Lh) ring, and for a stream on window
// w >= 1 the nanmean of its newest w columns in place of the running maximum (rt_localize's rule).  With Lh = 0 nothing changes.
#include <cmath>
#include <cstddef>
#include <vector>

#include "common.cuh"
#include "records.cuh"
#include "streams.cuh"

int gccnmf_stft_segments(gccnmf_handle* h, const float* samples, int64_t sample_stride, int channels, int segments, int frames_per_seg,
                         int64_t seg_stride, const double* window, int n_fft, int hop, int conjugate, float* X, float* V, void* stream);
int gccnmf_istft_frames(gccnmf_handle* h, const float* spec, int batch, int n_fft, int T, int conjugate, float* frames, void* stream);
int gccnmf_tdoa_gccnmf_gated(gccnmf_handle* h, const float* coherence, int F, int T, const double* E, int D, const float* W, int K,
                             int32_t* argmax, const int32_t* gate, int capacity, int32_t* ran, void* stream);
int gccnmf_phat_angspec_bank(gccnmf_handle* h, const float* X, int F, int T, const SteerBank& bank, int D, float* coherence, double* angular,
                             void* stream);
int gccnmf_tdoa_argmax_bank(gccnmf_handle* h, const float* coherence, int F, int T, const SteerBank& bank, int D, const float* W, int K,
                            int32_t* argmax, int32_t* overflow_flag, void* workspace, size_t workspace_bytes, void* stream);
int gccnmf_tdoa_gccnmf_bank(gccnmf_handle* h, const float* coherence, int F, int T, const SteerBank& bank, int D, const float* W, int K,
                            int32_t* argmax, const int32_t* gate, int capacity, int32_t* ran, void* stream);
int gccnmf_target_gccnmf_bank(gccnmf_handle* h, const float* coherence, int F, int T, const SteerBank& bank, int D, const float* W, int K,
                              const int32_t* targets, int P, float* values, void* stream);
int gccnmf_steering_transpose(gccnmf_handle* h, const double* E, int F, int D, double* ET, int64_t Fp, void* stream);
int gccnmf_lldict_prepare(gccnmf_handle* h, const DictBank& dict, int entry, const float* W, int F, int K, void* stream);
int gccnmf_tdoa_argmax_dict(gccnmf_handle* h, const float* coherence, int F, int T, const SteerBank& bank, const DictBank& dict, int D,
                            int32_t* argmax, int32_t* overflow_flag, void* workspace, size_t workspace_bytes, void* stream);
size_t gccnmf_tdoa_argmax_dict_workspace_bytes(int F, int T, int D, int K);
int gccnmf_tdoa_gccnmf_dict(gccnmf_handle* h, const float* coherence, int F, int T, const SteerBank& bank, const DictBank& dict, int D,
                            int32_t* argmax, const int32_t* gate, int capacity, int32_t* ran, void* stream);
int gccnmf_target_gccnmf_dict(gccnmf_handle* h, const float* coherence, int F, int T, const SteerBank& bank, const DictBank& dict, int D,
                              const int32_t* targets, int P, float* values, void* stream);
int gccnmf_wiener_dict(gccnmf_handle* h, const float* mask, const DictBank& dict, const float* H, const float* X, int F, int T, float* Y, float* wiener,
                       void* stream);
int gccnmf_rowsum_w(gccnmf_handle* h, const float* W, int F, int K, float* rowsum, void* stream);

namespace {

struct LLStream {
  long long hops;          // hops pushed since init / reset
  float epsilon;
  int active;
  int target_override;     // >= 0: replaces the localised target
  int pad;
};

struct LLHeader {
  float gain;
  int z;                   // first nonzero synthesis weight
};

struct LLLayout {
  int S, N, hop, C, K, D, F, Q, R;   // Q = ceil(N / hop): hops a frame spans; R = (Q - 1) hop: input ring length
  int P;                             // sources per stream (0: one enhanced target)
  size_t bytes;
  LLHeader* head;
  LLStream* streams;
  double *win_a, *w_syn, *E, *carry, *acc, *ang;
  float *W, *WT, *colsumW, *H0, *in_ring, *out_ring, *stage, *X, *V, *coh, *mask, *wiener, *Y, *H, *frames, *ws_wiener;
  // counters: [0] refined count, [1] status; with sources [2] coeff_mask's all-NaN flag, [3] the call's status word
  int32_t *targets, *valid, *argmax, *counters;
  void* ws_argmax;
  size_t n_argmax;
  // sources only: per stream the carried targets and overrides (kLLMaxSources each) and a status word; per call the values and
  // masks (P, K, T) and the column targets (T, P).  out_ring, wiener, Y and frames then hold P times as much.
  int32_t *src_targets, *src_override, *src_status, *col_targets;
  float *values, *src_mask;
  // history (gccnmf_llhist_*, Lh > 0): per stream one block of hist_stride bytes, the ring (D, Lh) f64 followed by the ring's write
  // index, the window w (i32 each) and 8 zero bytes; per call the window means (D, T)
  int Lh;
  size_t hist_stride;
  char* hist;
  double* means;
  // steering bank (gccnmf_llbank_*, Qe >= 1): E holds Qe tables (F, D) at a stride of 2 F D doubles; appended last, their
  // transposes ET (Qe, D, Fp) complex128 for the argmax refinement, the stream -> entry assignment (S), the streams sorted by entry
  // (S) and each entry's first position in that order (Qe + 1)
  int Qe;
  int64_t Fp;
  double* ET;
  int32_t *assign, *order, *seg;
  // dictionary bank (gccnmf_lldict_*, Qd >= 1, always with Qe >= 1): appended last, per entry e in slots of stride Kp = K rounded up
  // to 128 (K = Kmax, the largest entry): dW (F, K_e) f32 at e F Kp, packed (row stride K_e, as a plain engine on K_e holds W: the
  // content digest and the SIMT kernels read it so; only the planes are padded to Kp columns); the bf16 planes dWp, two (F, Qd Kp) arrays, entry e in columns
  // [e Kp, e Kp + K_e), zero beyond; dcolsum |W| column sums (Kp); dWTr the refinement's transpose (Kp, Fp); dWTi, dcolsumW and dH0
  // (inference only) ll_dict_kernel's W^T (K_e, F) and column sums, and H0 (K_e, 2); drowsum rowsum(W) (F); then the K_e table (Qd),
  // the stream -> entry assignment (S), the streams sorted by entry (S) and each entry's first position (Qd + 1)
  int Qd, Kp;
  float *dW, *dcolsum, *dWTr, *dWTi, *dcolsumW, *dH0, *drowsum;
  void* dWp;
  int32_t *dK, *dassign, *dorder, *dseg;
  // the grouped argmax's workspace (gccnmf_tdoa_argmax's carve at Kmax, whatever shape the plain argmax supports), when the tensor
  // path can run (D in [32, 128], F >= 32)
  void* ws_dict;
  size_t n_dict;
};

bool is_pow2(int x) { return x > 0 && (x & (x - 1)) == 0; }
constexpr int kLLMaxSources = 8;
constexpr int kLLInferMaxSmem = 227 * 1024;   // the H100's opt-in dynamic shared memory per block
constexpr int kLLMaxHistory = 1024;
constexpr int kLLMaxSteerings = 64;
constexpr int kLLMaxDictionaries = 64;
static_assert(kLLMaxSteerings <= kStreamMaxEntries && kLLMaxDictionaries <= kStreamMaxEntries, "sort_by_entry_kernel");

int ll_check(gccnmf_handle* h, const gccnmf_ll_config* cfg) {
  GCCNMF_REQUIRE(h, cfg != nullptr, "ll: NULL config");
  const gccnmf_ll_config& c = *cfg;
  GCCNMF_REQUIRE(h, is_pow2(c.window_size) && c.window_size >= 32 && c.window_size <= 4096, "ll: window_size must be a power of two in [32, 4096] (got %d)",
                 c.window_size);
  GCCNMF_REQUIRE(h, c.hop_size >= 1 && c.hop_size <= c.window_size, "ll: hop_size must be in [1, window_size] (got %d)", c.hop_size);
  GCCNMF_REQUIRE(h, c.hops_per_call >= 1 && c.hops_per_call <= 64, "ll: hops_per_call must be in [1, 64] (got %d)", c.hops_per_call);
  GCCNMF_REQUIRE(h, c.num_atoms >= 1, "ll: num_atoms must be positive (got %d)", c.num_atoms);
  GCCNMF_REQUIRE(h, is_pow2(c.num_tdoas) && c.num_tdoas >= 4 && c.num_tdoas <= 128, "ll: num_tdoas must be a power of two in [4, 128] (got %d)",
                 c.num_tdoas);
  GCCNMF_REQUIRE(h, c.num_streams >= 1 && c.num_streams <= 4096, "ll: num_streams must be in [1, 4096] (got %d)", c.num_streams);
  GCCNMF_REQUIRE(h, c.inference_iterations >= 0, "ll: inference_iterations must be >= 0 (got %d)", c.inference_iterations);
  GCCNMF_REQUIRE(h, (int64_t)c.num_streams * c.hops_per_call * c.num_tdoas < ((int64_t)1 << 31), "ll: S x C x D overflows int32");
  // ll_infer holds one column's H (K) and ratio (F) in shared memory
  GCCNMF_REQUIRE(h, c.inference_iterations == 0 || ((int64_t)c.num_atoms + c.window_size / 2 + 1) * 4 <= kLLInferMaxSmem,
                 "ll: inference needs (K + F) x 4 <= %d bytes of shared memory (K = %d)", kLLInferMaxSmem, c.num_atoms);
  return 0;
}

// P = 0: the single-target entries; 2 <= P <= 8: gccnmf_llsep_*
int ll_check(gccnmf_handle* h, const gccnmf_ll_config* cfg, int P) {
  if (int st = ll_check(h, cfg)) return st;
  if (P == 0) return 0;
  GCCNMF_REQUIRE(h, P >= 2 && P <= kLLMaxSources, "llsep: num_sources must be in [2, %d] (got %d)", kLLMaxSources, P);
  const int64_t T = (int64_t)cfg->num_streams * cfg->hops_per_call;
  GCCNMF_REQUIRE(h, T * P < ((int64_t)1 << 31) && (int64_t)P * cfg->num_atoms * T < ((int64_t)1 << 31),
                 "llsep: T x P or P x K x T overflows int32 (T = S x C)");
  return 0;
}

// Lh = 0: gccnmf_ll_* / gccnmf_llsep_*; 1 <= Lh <= 1024: a history ring of Lh frames per stream (gccnmf_llhist_*)
int ll_check(gccnmf_handle* h, const gccnmf_ll_config* cfg, int P, int Lh) {
  if (int st = ll_check(h, cfg, P)) return st;
  GCCNMF_REQUIRE(h, Lh >= 0 && Lh <= kLLMaxHistory, "llhist: history_length must be in [0, %d] (got %d)", kLLMaxHistory, Lh);
  GCCNMF_REQUIRE(h, (int64_t)cfg->num_streams * cfg->num_tdoas * Lh < ((int64_t)1 << 31), "llhist: S x D x history_length overflows int32");
  return 0;
}

// Qe = 0: no bank (gccnmf_llhist_*); 1 <= Qe <= 64: a bank of Qe steering tables (gccnmf_llbank_*)
int ll_check(gccnmf_handle* h, const gccnmf_ll_config* cfg, int P, int Lh, int Qe) {
  if (int st = ll_check(h, cfg, P, Lh)) return st;
  GCCNMF_REQUIRE(h, Qe >= 0 && Qe <= kLLMaxSteerings, "llbank: num_steerings must be in [0, %d] (got %d)", kLLMaxSteerings, Qe);
  return 0;
}

// Qd = 0: no dictionary bank; 1 <= Qd <= 64 (gccnmf_lldict_*): a bank of Qd dictionaries, with 1 <= Qe <= 64 steering tables
int ll_check(gccnmf_handle* h, const gccnmf_ll_config* cfg, int P, int Lh, int Qe, int Qd) {
  if (int st = ll_check(h, cfg, P, Lh, Qe)) return st;
  if (Qd == 0) return 0;
  GCCNMF_REQUIRE(h, Qd >= 1 && Qd <= kLLMaxDictionaries, "lldict: num_dictionaries must be in [1, %d] (got %d)", kLLMaxDictionaries, Qd);
  GCCNMF_REQUIRE(h, Qe >= 1, "lldict: num_steerings must be in [1, %d] (got %d)", kLLMaxSteerings, Qe);
  return 0;
}

LLLayout ll_carve(const gccnmf_ll_config& c, int P, void* base, int Lh = 0, int Qe = 0, int Qd = 0) {
  WorkspaceCarver w(base ? base : reinterpret_cast<void*>(256), base ? ~size_t(0) >> 1 : ~size_t(0) >> 1);
  LLLayout l{};
  l.S = c.num_streams; l.N = c.window_size; l.hop = c.hop_size; l.C = c.hops_per_call; l.K = c.num_atoms; l.D = c.num_tdoas;
  l.F = l.N / 2 + 1; l.Q = (l.N + l.hop - 1) / l.hop; l.R = (l.Q - 1) * l.hop;
  const size_t S = l.S, N = l.N, F = l.F, K = l.K, D = l.D, T = S * l.C;
  const bool inf = c.inference_iterations > 0;
  l.P = P;
  const size_t Pm = P > 0 ? P : 1;   // copies of the per-target buffers
  l.head = w.take<LLHeader>(1);
  l.streams = w.take<LLStream>(S);
  l.counters = w.take<int32_t>(4);
  l.win_a = w.take<double>(N);
  l.w_syn = w.take<double>(N);
  l.E = w.take<double>((Qe ? Qe : 1) * 2 * F * D);
  l.W = w.take<float>(F * K);
  l.WT = w.take<float>(inf ? K * F : 0);
  l.colsumW = w.take<float>(inf ? K : 0);
  l.H0 = w.take<float>(inf ? K * 2 : 0);
  l.in_ring = w.take<float>(S * 2 * l.R);
  l.out_ring = w.take<float>(S * Pm * 2 * N);
  l.carry = w.take<double>(S * D);
  l.stage = w.take<float>(2 * S * (l.R + (size_t)l.C * l.hop));
  l.X = w.take<float>(2 * 2 * F * T);
  l.V = w.take<float>(inf ? F * 2 * T : 0);
  l.coh = w.take<float>(2 * F * T);
  l.ang = w.take<double>(D * T);
  l.acc = w.take<double>(D * T);
  l.targets = w.take<int32_t>(T);
  l.valid = w.take<int32_t>(T);
  l.argmax = w.take<int32_t>(K * T);
  l.mask = w.take<float>(K * T);
  l.wiener = w.take<float>(Pm * (inf ? 2 : 1) * F * T);
  l.Y = w.take<float>(Pm * 2 * 2 * F * T);
  l.H = w.take<float>(inf ? K * 2 * T : 0);
  l.frames = w.take<float>(Pm * 2 * T * N);
  l.ws_wiener = w.take<float>(gccnmf_wiener_apply_workspace_bytes((int)F) / sizeof(float));
  l.n_argmax = gccnmf_tdoa_argmax_workspace_bytes((int)F, (int)T, (int)D, (int)K);
  l.ws_argmax = w.take<unsigned char>(l.n_argmax);
  // sources: appended to the single-target layout (nothing is taken with P = 0, so that layout is unchanged)
  const size_t Ps = P;
  l.src_targets = w.take<int32_t>(P ? S * kLLMaxSources : 0);
  l.src_override = w.take<int32_t>(P ? S * kLLMaxSources : 0);
  l.src_status = w.take<int32_t>(P ? S : 0);
  l.col_targets = w.take<int32_t>(T * Ps);
  l.values = w.take<float>(Ps * K * T);
  l.src_mask = w.take<float>(Ps * K * T);
  // history: appended last (nothing is taken with Lh = 0, so the layouts above are unchanged)
  l.Lh = Lh;
  l.hist_stride = Lh ? D * Lh * sizeof(double) + 16 : 0;
  l.hist = w.take<char>(S * l.hist_stride);
  l.means = w.take<double>(Lh ? D * T : 0);
  // bank: appended last (nothing is taken with Qe = 0, so the layouts above are unchanged)
  l.Qe = Qe;
  l.Fp = (F + 7) & ~size_t(7);                 // gccnmf_tdoa_argmax's padded bin count
  l.ET = w.take<double>(Qe ? Qe * 2 * D * l.Fp : 0);
  l.assign = w.take<int32_t>(Qe ? S : 0);
  l.order = w.take<int32_t>(Qe ? S : 0);
  l.seg = w.take<int32_t>(Qe ? Qe + 1 : 0);
  // dictionary bank: appended last (nothing is taken with Qd = 0)
  l.Qd = Qd;
  l.Kp = (int)((K + 127) / 128 * 128);
  const size_t Qs = Qd, Kp = l.Kp;
  l.dW = w.take<float>(Qs * F * Kp);
  l.dWp = w.take<uint16_t>(2 * F * Qs * Kp);
  l.dcolsum = w.take<float>(Qs * Kp);
  l.dWTr = w.take<float>(Qs * Kp * l.Fp);
  l.dWTi = w.take<float>(inf ? Qs * Kp * F : 0);
  l.dcolsumW = w.take<float>(inf ? Qs * Kp : 0);
  l.dH0 = w.take<float>(inf ? Qs * Kp * 2 : 0);
  l.drowsum = w.take<float>(Qs * F);
  l.dK = w.take<int32_t>(Qs);
  l.dassign = w.take<int32_t>(Qd ? S : 0);
  l.dorder = w.take<int32_t>(Qd ? S : 0);
  l.dseg = w.take<int32_t>(Qd ? Qd + 1 : 0);
  l.n_dict = Qd && D >= 32 && D <= 128 && F >= 32 ? gccnmf_tdoa_argmax_dict_workspace_bytes((int)F, (int)T, (int)D, (int)K) : 0;
  l.ws_dict = w.take<unsigned char>(l.n_dict);
  // (the plain W, WT, colsumW and H0 regions above stay carved and unused with Qd >= 1, so the llbank offsets hold)
  l.bytes = align_up(w.used, 256);
  return l;
}

#define LLD_CARVE_OR_FAIL(l, P, Lh, Qe, Qd)                                                                          \
  if (int st__ = ll_check(h, cfg, P, Lh, Qe, Qd)) return st__;                                                       \
  GCCNMF_REQUIRE(h, state != nullptr, "ll: NULL state");                                                             \
  const LLLayout l = ll_carve(*cfg, P, state, Lh, Qe, Qd);                                                           \
  if (state_bytes < l.bytes) return gccnmf_fail(h, GCCNMF_ERR_WORKSPACE, "ll: state too small: need %zu bytes", l.bytes);
#define LL_CARVE_OR_FAIL(l, P, Lh, Qe) LLD_CARVE_OR_FAIL(l, P, Lh, Qe, 0)

SteerBank ll_bank(const LLLayout& l, int hops) {
  return SteerBank{reinterpret_cast<const double2*>(l.E), reinterpret_cast<const double2*>(l.ET), l.assign, l.order, l.seg, l.Qe, hops, l.Fp};
}

DictBank ll_dict(const LLLayout& l, int hops) {
  return DictBank{l.dW, l.dcolsum, l.dWTr, l.drowsum, l.dWp, l.dK, l.dassign, l.dorder, l.dseg, l.Qd, hops, l.Kp, l.K, (int64_t)l.F * l.Kp, l.Fp};
}

// ---------------------------------------------------------------------------------------------- kernels
__global__ void ll_reset_kernel(LLStream* streams, int first, int count, float* in_ring, float* out_ring, double* carry, int R, int N, int D,
                                int set_defaults) {
  const int s = first + blockIdx.x;
  if (blockIdx.x >= count) return;
  for (int i = threadIdx.x; i < 2 * R; i += blockDim.x) in_ring[(int64_t)s * 2 * R + i] = 0.f;
  for (int i = threadIdx.x; i < 2 * N; i += blockDim.x) out_ring[(int64_t)s * 2 * N + i] = 0.f;
  for (int d = threadIdx.x; d < D; d += blockDim.x) carry[(int64_t)s * D + d] = -INFINITY;
  if (threadIdx.x == 0) {
    streams[s].hops = 0;
    if (set_defaults) {
      streams[s].epsilon = 1.f;
      streams[s].active = 1;
      streams[s].target_override = -1;
    }
  }
}

constexpr int kLLParamsPerLaunch = 64;
struct LLParamsBatch { gccnmf_ll_stream_params p[kLLParamsPerLaunch]; };

__global__ void ll_params_kernel(LLStream* streams, int first, int count, LLParamsBatch b) {
  const int i = threadIdx.x;
  if (i >= count) return;
  streams[first + i].epsilon = b.p[i].epsilon;
  streams[first + i].active = b.p[i].active ? 1 : 0;
  streams[first + i].target_override = b.p[i].target_override;
}

// first nonzero synthesis weight (N if none)
__global__ void ll_header_kernel(LLHeader* head, const double* w, int N, float gain) {
  int z = N;
  for (int r = 0; r < N; ++r)
    if (w[r] != 0.0) { z = r; break; }
  head->z = z;
  head->gain = gain;
}

// WT (K, F) = W^T and colsumW[k] = sum_f W[f][k] in f order (inference only)
__global__ void ll_dict_kernel(const float* __restrict__ W, int F, int K, float* __restrict__ WT, float* __restrict__ colsum) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= K) return;
  float s = 0.f;
  for (int f = 0; f < F; ++f) {
    const float v = W[(int64_t)f * K + k];
    WT[(int64_t)k * F + f] = v;
    s += v;
  }
  colsum[k] = s;
}

// stage[ch][s][0 .. R) = input ring, stage[ch][s][R .. R + n) = the call's new samples; valid[s hops + i] = frame i is a whole frame
__global__ void ll_push_kernel(const LLStream* __restrict__ streams, const float* __restrict__ in, const float* __restrict__ in_ring, int S, int R,
                               int n, int hops, int frames_before_first, float* __restrict__ stage, int32_t* __restrict__ valid) {
  const int s = blockIdx.x, ch = blockIdx.y;
  const int64_t Lseg = (int64_t)R + n;
  float* dst = stage + ((int64_t)ch * S + s) * Lseg;
  const float* ring = in_ring + ((int64_t)s * 2 + ch) * R;
  const float* x = in + ((int64_t)s * 2 + ch) * n;
  for (int64_t i = threadIdx.x; i < Lseg; i += blockDim.x) dst[i] = i < R ? ring[i] : x[i - R];
  if (ch == 0 && threadIdx.x < hops) {
    // frame j = hops_before + i + 1 - ceil(N / hop) is the stream's frame j (it ends in hop i); j < 0 starts before the first sample
    const long long j = streams[s].hops + threadIdx.x + 1 - frames_before_first;
    valid[s * hops + threadIdx.x] = streams[s].active && j >= 0 ? 1 : 0;
  }
}

// numpy.argmax ordering: NaN is a maximum, first occurrence wins (gcc.cu's argmax_better).
__device__ __forceinline__ bool ll_argmax_better(double v, int i, double bv, int bi) {
  const bool vn = isnan(v), bn = isnan(bv);
  if (vn || bn) return vn && (!bn || i < bi);
  return v > bv || (v == bv && i < bi);
}

// The running maximum of cummax_time_kernel from the carried one over stream s's valid frames of the call (thread d = TDOA), written
// to acc for every frame of the call; the carry is stored when the stream is active.
__device__ __forceinline__ void ll_running_max(const LLStream* __restrict__ streams, const double* __restrict__ ang, const int32_t* __restrict__ valid,
                                               int D, int hops, int T, double* __restrict__ carry, double* __restrict__ acc) {
  const int s = blockIdx.x, d = threadIdx.x;
  const int t0 = s * hops;
  if (d < D) {
    double m = carry[(int64_t)s * D + d];
    for (int i = 0; i < hops; ++i) {
      if (valid[t0 + i]) {
        const double v = ang[(int64_t)d * T + t0 + i];
        if (v > m || v != v) m = v;          // numpy.max: NaN propagates (and then sticks)
      }
      acc[(int64_t)d * T + t0 + i] = m;
    }
    if (streams[s].active) carry[(int64_t)s * D + d] = m;
  }
}

// One CTA per stream, thread d = TDOA: the running maximum, then target[t] = argmax over d (argmax_tdoa_kernel), or the stream's
// override.
__global__ void ll_targets_kernel(const LLStream* __restrict__ streams, const double* __restrict__ ang, const int32_t* __restrict__ valid, int D,
                                  int hops, int T, double* __restrict__ carry, double* __restrict__ acc, int32_t* __restrict__ targets) {
  const int s = blockIdx.x, d = threadIdx.x;
  const int t0 = s * hops;
  ll_running_max(streams, ang, valid, D, hops, T, carry, acc);
  __syncthreads();
  if (d < hops) {
    const int t = t0 + d;
    double bv = acc[t];
    int bi = 0;
    for (int e = 1; e < D; ++e) {
      const double v = acc[(int64_t)e * T + t];
      if (ll_argmax_better(v, e, bv, bi)) { bv = v; bi = e; }
    }
    const int o = streams[s].target_override;
    targets[t] = o >= 0 ? o : bi;
  }
}

// Sources: one CTA per stream (128 threads, thread d = TDOA).  The running maximum as above, then frame by frame in order: the P
// largest strict local maxima of the frame's running maximum (select_peaks, ascending) become the stream's targets; with fewer
// peaks the targets stay and status bit 0 is set.  Column targets (T, P) = the targets, or the source's override where it is >= 0.
// Invalid frames (before the first sample, inactive stream) change nothing.
__global__ void __launch_bounds__(128)
ll_src_targets_kernel(const LLStream* __restrict__ streams, const double* __restrict__ ang, const int32_t* __restrict__ valid, int D, int hops,
                      int T, int P, double* __restrict__ carry, double* __restrict__ acc, int32_t* __restrict__ src_targets,
                      const int32_t* __restrict__ src_override, int32_t* __restrict__ src_status, int32_t* __restrict__ col_targets) {
  __shared__ double x_s[128];
  __shared__ unsigned char peak_s[128], chosen_s[128];
  __shared__ int num_peaks_s;
  __shared__ int32_t pick_s[kLLMaxSources], cur_s[kLLMaxSources];
  const int s = blockIdx.x, d = threadIdx.x;
  const int t0 = s * hops;
  ll_running_max(streams, ang, valid, D, hops, T, carry, acc);
  if (d < P) cur_s[d] = src_targets[(int64_t)s * kLLMaxSources + d];
  __syncthreads();
  for (int i = 0; i < hops; ++i) {
    const int t = t0 + i;
    if (valid[t]) {                      // the same for every thread of the CTA
      if (d < D) x_s[d] = acc[(int64_t)d * T + t];
      const int peaks = select_peaks(x_s, D, P, peak_s, chosen_s, &num_peaks_s, pick_s);
      if (d == 0) {
        if (peaks >= P)
          for (int q = 0; q < P; ++q) cur_s[q] = pick_s[q];
        else
          src_status[s] |= GCCNMF_LLSEP_STATUS_FEW_PEAKS;
      }
      __syncthreads();
    }
    if (d < P) {
      const int o = src_override[(int64_t)s * kLLMaxSources + d];
      col_targets[(int64_t)t * P + d] = o >= 0 ? o : cur_s[d];
    }
  }
  if (d < P) src_targets[(int64_t)s * kLLMaxSources + d] = cur_s[d];
}

// History (gccnmf_llhist_*), thread d = TDOA of stream s: each valid frame's angular column goes into the ring at the write index,
// which moves on; then, whatever the frame's validity, means[d][t] = the nanmean of the newest w ring columns, summed newest first
// in float64 and skipping NaN (rt_localize's loop, restated), NaN when all of them are NaN or w = 0.  The zero columns of a ring
// that has seen fewer than w frames count in the denominator.  The write index is stored by thread 0 after `__syncthreads`.
// Returns w (the same in every thread).
__device__ __forceinline__ int ll_hist_means(const double* __restrict__ ang, const int32_t* __restrict__ valid, int D, int hops, int T, char* hist,
                                             size_t hist_stride, int Lh, double* __restrict__ means) {
  const int s = blockIdx.x, d = threadIdx.x;
  const int t0 = s * hops;
  double* ring = reinterpret_cast<double*>(hist + (size_t)s * hist_stride);
  int32_t* slot = reinterpret_cast<int32_t*>(ring + (size_t)D * Lh);      // [0] write index, [1] window
  int idx = slot[0];
  const int w = slot[1];
  if (d < D) {
    double* row = ring + (size_t)d * Lh;
    for (int i = 0; i < hops; ++i) {
      const int t = t0 + i;
      if (valid[t]) {
        row[idx] = ang[(int64_t)d * T + t];
        idx = idx + 1 == Lh ? 0 : idx + 1;
      }
      double m = __longlong_as_double(0x7ff8000000000000LL);
      if (w > 0) {
        double sum = 0.0;
        int n = 0;
        for (int j = 0, p = idx; j < w; ++j) {
          p = p == 0 ? Lh - 1 : p - 1;
          const double v = row[p];
          if (v == v) { sum += v; ++n; }
        }
        if (n > 0) m = sum / (double)n;
      }
      means[(int64_t)d * T + t] = m;
    }
  }
  __syncthreads();
  if (d == 0) slot[0] = idx;
  return w;
}

// History, one CTA per stream, thread d = TDOA: the running maximum and its carry as ll_targets_kernel, the ring and the window
// means, then target[t] = argmax over d of the means (w >= 1) or of the running maximum (w = 0), or the stream's override.
__global__ void __launch_bounds__(128)
ll_hist_targets_kernel(const LLStream* __restrict__ streams, const double* __restrict__ ang, const int32_t* __restrict__ valid, int D, int hops,
                       int T, double* __restrict__ carry, double* __restrict__ acc, char* __restrict__ hist, size_t hist_stride, int Lh,
                       double* __restrict__ means, int32_t* __restrict__ targets) {
  const int s = blockIdx.x, d = threadIdx.x;
  ll_running_max(streams, ang, valid, D, hops, T, carry, acc);
  const int w = ll_hist_means(ang, valid, D, hops, T, hist, hist_stride, Lh, means);
  if (d < hops) {
    const double* x = w > 0 ? means : acc;
    const int t = s * hops + d;
    double bv = x[t];
    int bi = 0;
    for (int e = 1; e < D; ++e) {
      const double v = x[(int64_t)e * T + t];
      if (ll_argmax_better(v, e, bv, bi)) { bv = v; bi = e; }
    }
    const int o = streams[s].target_override;
    targets[t] = o >= 0 ? o : bi;
  }
}

// History with sources: ll_src_targets_kernel's rule on the window means (w >= 1) or on the running maximum (w = 0).
__global__ void __launch_bounds__(128)
ll_hist_src_targets_kernel(const LLStream* __restrict__ streams, const double* __restrict__ ang, const int32_t* __restrict__ valid, int D,
                           int hops, int T, int P, double* __restrict__ carry, double* __restrict__ acc, char* __restrict__ hist,
                           size_t hist_stride, int Lh, double* __restrict__ means, int32_t* __restrict__ src_targets,
                           const int32_t* __restrict__ src_override, int32_t* __restrict__ src_status, int32_t* __restrict__ col_targets) {
  __shared__ double x_s[128];
  __shared__ unsigned char peak_s[128], chosen_s[128];
  __shared__ int num_peaks_s;
  __shared__ int32_t pick_s[kLLMaxSources], cur_s[kLLMaxSources];
  const int s = blockIdx.x, d = threadIdx.x;
  const int t0 = s * hops;
  ll_running_max(streams, ang, valid, D, hops, T, carry, acc);
  if (d < P) cur_s[d] = src_targets[(int64_t)s * kLLMaxSources + d];
  const int w = ll_hist_means(ang, valid, D, hops, T, hist, hist_stride, Lh, means);
  const double* x = w > 0 ? means : acc;
  for (int i = 0; i < hops; ++i) {
    const int t = t0 + i;
    if (valid[t]) {                      // the same for every thread of the CTA
      if (d < D) x_s[d] = x[(int64_t)d * T + t];
      const int peaks = select_peaks(x_s, D, P, peak_s, chosen_s, &num_peaks_s, pick_s);
      if (d == 0) {
        if (peaks >= P)
          for (int q = 0; q < P; ++q) cur_s[q] = pick_s[q];
        else
          src_status[s] |= GCCNMF_LLSEP_STATUS_FEW_PEAKS;
      }
      __syncthreads();
    }
    if (d < P) {
      const int o = src_override[(int64_t)s * kLLMaxSources + d];
      col_targets[(int64_t)t * P + d] = o >= 0 ? o : cur_s[d];
    }
  }
  if (d < P) src_targets[(int64_t)s * kLLMaxSources + d] = cur_s[d];
}

// History: streams [first, first + count) back to a zero ring, write index 0 and window 0 (16-byte words: the stride is a multiple of 16).
__global__ void ll_hist_reset_kernel(char* __restrict__ hist, size_t hist_stride, int first, int count) {
  if ((int)blockIdx.x >= count) return;
  uint4* b = reinterpret_cast<uint4*>(hist + (size_t)(first + blockIdx.x) * hist_stride);
  for (size_t i = threadIdx.x; i < hist_stride / 16; i += blockDim.x) b[i] = make_uint4(0, 0, 0, 0);
}

// mask[k][t] = |argmax[k][t] - target[t]| < epsilon of t's stream   (atom_mask_kernel mode 0)
__global__ void ll_mask_kernel(const LLStream* __restrict__ streams, const int32_t* __restrict__ argmax, const int32_t* __restrict__ targets, int K,
                               int T, int hops, float* __restrict__ mask) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)K * T) return;
  const int t = (int)(i % T);
  const float mu = (float)targets[t];
  const float dist = fabsf((float)argmax[i] - mu);
  mask[i] = dist < streams[t / hops].epsilon ? 1.f : 0.f;
}

// H-only KL updates (gccNMFFunctions.py:76) of one (frame, channel) column from H0: CTA = column, 8 warps.
//   R[f] = V[f] / sum_k W[f][k] H[k]              warp per bin, lane-strided fmaf over k from 0.f, xor butterfly
//   H[k] *= (sum_f W[f][k] R[f]) / (colsum(W)[k] + alpha + eps)     warp per atom over W^T, the same reduction
// The order of every sum is fixed per column, so a column's result does not depend on how many columns share the launch.
__global__ void __launch_bounds__(256)
ll_infer_kernel(const float* __restrict__ W, const float* __restrict__ WT, const float* __restrict__ colsumW, const float* __restrict__ H0,
                const float* __restrict__ V, int F, int K, int T, int iterations, float alpha, float eps, float* __restrict__ Hout) {
  extern __shared__ float sm[];
  float* Hs = sm;          // K
  float* Rs = sm + K;      // F
  const int t = blockIdx.x, ch = blockIdx.y;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, warps = blockDim.x >> 5;
  const int64_t col = (int64_t)ch * T + t;
  for (int k = threadIdx.x; k < K; k += blockDim.x) Hs[k] = H0[(int64_t)k * 2 + ch];
  __syncthreads();
  for (int it = 0; it < iterations; ++it) {
    for (int f = warp; f < F; f += warps) {
      float a = 0.f;
      for (int k = lane; k < K; k += 32) a = fmaf(W[(int64_t)f * K + k], Hs[k], a);
      for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
      if (lane == 0) Rs[f] = V[(int64_t)f * (2 * T) + col] / a;
    }
    __syncthreads();
    for (int k = warp; k < K; k += warps) {
      float a = 0.f;
      for (int f = lane; f < F; f += 32) a = fmaf(WT[(int64_t)k * F + f], Rs[f], a);
      for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
      if (lane == 0) Hs[k] = Hs[k] * (a / ((colsumW[k] + alpha) + eps));
    }
    __syncthreads();
  }
  for (int k = threadIdx.x; k < K; k += blockDim.x) Hout[(int64_t)k * (2 * T) + col] = Hs[k];
}

// For each frame of the call in order: ring[p] = float32(fma(w[r], frame[r], ring[p])) for r >= z, p = (j hop + r) mod N
// (ola_gather_kernel's chain: the weights below z are zero and would leave every sum as it is), then emit the hop samples
// [j hop + z, j hop + z + hop) times the gain and zero them.  frames (2, T, N) of one target, ring (2, N), o (2, hops hop).
__device__ __forceinline__ void ll_ola_emit(const LLHeader* __restrict__ head, const double* __restrict__ w, const float* __restrict__ frames,
                                            int N, int hop, int hops, int T, int frames_before_first, long long h0, int s, float* __restrict__ ring,
                                            float* __restrict__ o) {
  const int n = hops * hop;
  const int z = head->z;
  const float gain = head->gain;
  for (int i = 0; i < hops; ++i) {
    const long long j = h0 + i + 1 - frames_before_first;
    const int base = (int)(((j % N) * hop % N + N) % N);          // (j hop) mod N
    if (j >= 0) {
      const int t = s * hops + i;
      for (int e = threadIdx.x; e < 2 * N; e += blockDim.x) {
        const int ch = e >= N, r = e - ch * N;
        if (r < z) continue;
        const int p = (base + r) & (N - 1);
        float* a = ring + ch * N + p;
        *a = (float)fma(w[r], (double)frames[((int64_t)ch * T + t) * N + r], (double)*a);
      }
    }
    __syncthreads();
    for (int e = threadIdx.x; e < 2 * hop; e += blockDim.x) {
      const int ch = e >= hop, q = e - ch * hop;
      const int p = (base + z + q) & (N - 1);
      o[(int64_t)ch * n + i * hop + q] = ring[ch * N + p] * gain;
      ring[ch * N + p] = 0.f;
    }
    __syncthreads();
  }
}

// The last R samples of stream s's staging rows are the next call's input ring; the stream has pushed `hops` more hops.
__device__ __forceinline__ void ll_advance(LLStream* __restrict__ streams, int s, int S, const float* __restrict__ stage, float* __restrict__ in_ring,
                                           int R, int n, int hops, long long h0) {
  const int64_t Lseg = (int64_t)R + n;
  for (int e = threadIdx.x; e < 2 * R; e += blockDim.x) {
    const int ch = e >= R, q = e - ch * R;
    in_ring[((int64_t)s * 2 + ch) * R + q] = stage[((int64_t)ch * S + s) * Lseg + n + q];
  }
  if (threadIdx.x == 0) streams[s].hops = h0 + hops;
}

// One CTA per stream: overlap-add and emit, then the input ring moves on.
__global__ void __launch_bounds__(256)
ll_ola_emit_kernel(LLStream* __restrict__ streams, const LLHeader* __restrict__ head, const double* __restrict__ w, const float* __restrict__ frames,
                   int N, int hop, int hops, int T, int frames_before_first, float* __restrict__ out_ring, float* __restrict__ out,
                   const float* __restrict__ stage, float* __restrict__ in_ring, int R) {
  const int s = blockIdx.x;
  const int n = hops * hop;
  float* o = out + (int64_t)s * 2 * n;
  if (!streams[s].active) {
    for (int i = threadIdx.x; i < 2 * n; i += blockDim.x) o[i] = 0.f;
    return;
  }
  const long long h0 = streams[s].hops;
  ll_ola_emit(head, w, frames, N, hop, hops, T, frames_before_first, h0, s, out_ring + (int64_t)s * 2 * N, o);
  ll_advance(streams, s, gridDim.x, stage, in_ring, R, n, hops, h0);
}

// Sources: CTA (s, q) overlap-adds source q's frames (P, 2, T, N) into its own ring and emits into out (S, P, 2, hops hop).  It
// only reads the stream's hop count: ll_src_advance_kernel moves the stream on once every source has emitted.
__global__ void __launch_bounds__(256)
ll_src_ola_emit_kernel(const LLStream* __restrict__ streams, const LLHeader* __restrict__ head, const double* __restrict__ w,
                       const float* __restrict__ frames, int N, int hop, int hops, int T, int frames_before_first, float* __restrict__ out_ring,
                       float* __restrict__ out) {
  const int s = blockIdx.x, q = blockIdx.y, P = gridDim.y;
  const int n = hops * hop;
  const int64_t sq = (int64_t)s * P + q;
  float* o = out + sq * 2 * n;
  if (!streams[s].active) {
    for (int i = threadIdx.x; i < 2 * n; i += blockDim.x) o[i] = 0.f;
    return;
  }
  ll_ola_emit(head, w, frames + (int64_t)q * 2 * T * N, N, hop, hops, T, frames_before_first, streams[s].hops, s, out_ring + sq * 2 * N, o);
}

// Sources: one CTA per stream after every source has emitted; CTA 0 also turns coeff_mask's all-NaN flag into the call's status.
__global__ void __launch_bounds__(256)
ll_src_advance_kernel(LLStream* __restrict__ streams, int hops, int hop, const float* __restrict__ stage, float* __restrict__ in_ring, int R,
                      int32_t* __restrict__ counters) {
  const int s = blockIdx.x;
  if (s == 0 && threadIdx.x == 0) counters[3] = counters[2] ? GCCNMF_LLSEP_STATUS_ALL_NAN : 0;
  if (!streams[s].active) return;
  ll_advance(streams, s, gridDim.x, stage, in_ring, R, hops * hop, hops, streams[s].hops);
}

// Sources: stream s's P output rings zeroed, targets back to the defaults floor((2 q + 1) D / (2 P)), status cleared; with
// set_defaults (init) no overrides.
__global__ void ll_src_reset_kernel(int first, int count, int P, int D, int N, float* __restrict__ out_ring, int32_t* __restrict__ src_targets,
                                    int32_t* __restrict__ src_override, int32_t* __restrict__ src_status, int set_defaults) {
  const int s = first + blockIdx.x;
  if (blockIdx.x >= count) return;
  for (int i = threadIdx.x; i < P * 2 * N; i += blockDim.x) out_ring[(int64_t)s * P * 2 * N + i] = 0.f;
  if (threadIdx.x < kLLMaxSources) {
    const int q = threadIdx.x;
    src_targets[(int64_t)s * kLLMaxSources + q] = q < P ? (2 * q + 1) * D / (2 * P) : 0;
    if (set_defaults) src_override[(int64_t)s * kLLMaxSources + q] = -1;
  }
  if (threadIdx.x == 0) src_status[s] = 0;
}

// ---- dictionary bank (gccnmf_lldict_*): column t is on entry dassign[t / hops] with K_e atoms
// ll_mask_kernel's mask on rows k < K_e; rows [K_e, Kmax) get 0
__global__ void ll_dict_mask_kernel(const LLStream* __restrict__ streams, const int32_t* __restrict__ argmax, const int32_t* __restrict__ targets,
                                    const int32_t* __restrict__ dK, const int32_t* __restrict__ dassign, int K, int T, int hops,
                                    float* __restrict__ mask) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)K * T) return;
  const int t = (int)(i % T), k = (int)(i / T);
  if (k >= __ldg(dK + __ldg(dassign + t / hops))) { mask[i] = 0.f; return; }
  const float mu = (float)targets[t];
  const float dist = fabsf((float)argmax[i] - mu);
  mask[i] = dist < streams[t / hops].epsilon ? 1.f : 0.f;
}

// ll_infer_kernel on the column's dictionary: its W, W^T, column sums, H0 and K_e; H (Kmax, 2T) rows < K_e
__global__ void __launch_bounds__(256)
ll_dict_infer_kernel(DictBank dict, const float* __restrict__ WT, const float* __restrict__ colsumW, const float* __restrict__ H0,
                     const float* __restrict__ V, int F, int T, int iterations, float alpha, float eps, float* __restrict__ Hout) {
  extern __shared__ float sm[];
  const int t = blockIdx.x, ch = blockIdx.y;
  const int e = dict.entry(t), K = __ldg(dict.K + e);
  const float* __restrict__ W = dict.W + e * dict.wstride;
  WT += (int64_t)e * dict.Kp * F;
  colsumW += (int64_t)e * dict.Kp;
  H0 += (int64_t)e * dict.Kp * 2;
  float* Hs = sm;          // K
  float* Rs = sm + K;      // F
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, warps = blockDim.x >> 5;
  const int64_t col = (int64_t)ch * T + t;
  for (int k = threadIdx.x; k < K; k += blockDim.x) Hs[k] = H0[(int64_t)k * 2 + ch];
  __syncthreads();
  for (int it = 0; it < iterations; ++it) {
    for (int f = warp; f < F; f += warps) {
      float a = 0.f;
      for (int k = lane; k < K; k += 32) a = fmaf(W[(int64_t)f * K + k], Hs[k], a);
      for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
      if (lane == 0) Rs[f] = V[(int64_t)f * (2 * T) + col] / a;
    }
    __syncthreads();
    for (int k = warp; k < K; k += warps) {
      float a = 0.f;
      for (int f = lane; f < F; f += 32) a = fmaf(WT[(int64_t)k * F + f], Rs[f], a);
      for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
      if (lane == 0) Hs[k] = Hs[k] * (a / ((colsumW[k] + alpha) + eps));
    }
    __syncthreads();
  }
  for (int k = threadIdx.x; k < K; k += blockDim.x) Hout[(int64_t)k * (2 * T) + col] = Hs[k];
}

// The defined fill of the rows [K_e, Kmax) of column t's K-shaped items (NULL: not touched): argmax -1; values, source masks
// (P of each, (P, Kmax, T)) and H (Kmax, 2T) 0
__global__ void ll_dict_fill_kernel(const int32_t* __restrict__ dK, const int32_t* __restrict__ dassign, int K, int T, int hops, int P,
                                    int32_t* __restrict__ argmax, float* __restrict__ values, float* __restrict__ H) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)K * T) return;
  const int t = (int)(i % T), k = (int)(i / T);
  if (k < __ldg(dK + __ldg(dassign + t / hops))) return;
  if (argmax) argmax[i] = -1;
  if (values)
    for (int q = 0; q < P; ++q) values[(int64_t)q * K * T + i] = 0.f;
  if (H) {
    H[(int64_t)k * 2 * T + t] = 0.f;
    H[(int64_t)k * 2 * T + T + t] = 0.f;
  }
}

__global__ void ll_set_int_kernel(int32_t* p, int v) { *p = v; }

// Sources, after the shared front (push, STFT, PHAT / angular): targets, the target contraction, coeff_mask, per source the
// filter (with inference on the shared H), then one inverse FFT of all (P, 2) spectra, emit per (stream, source), advance.
int ll_enqueue_sources(gccnmf_handle* h, const gccnmf_ll_config* cfg, const LLLayout& l, int hops, float* out, void* stream) {
  const int S = l.S, N = l.N, hop = l.hop, F = l.F, K = l.K, D = l.D, P = l.P, T = S * hops;
  const bool inf = cfg->inference_iterations > 0;
  if (l.Lh)
    GCCNMF_LAUNCH(h, ll_hist_src_targets_kernel, S, 128, 0, stream, l.streams, l.ang, l.valid, D, hops, T, P, l.carry, l.acc, l.hist, l.hist_stride,
                  l.Lh, l.means, l.src_targets, l.src_override, l.src_status, l.col_targets);
  else
    GCCNMF_LAUNCH(h, ll_src_targets_kernel, S, 128, 0, stream, l.streams, l.ang, l.valid, D, hops, T, P, l.carry, l.acc, l.src_targets,
                  l.src_override, l.src_status, l.col_targets);
  const unsigned fill_ctas = (unsigned)(((int64_t)K * T + 255) / 256);
  if (l.Qd) {
    if (int e = gccnmf_target_gccnmf_dict(h, l.coh, F, T, ll_bank(l, hops), ll_dict(l, hops), D, l.col_targets, P, l.values, stream)) return e;
    // rows past a column's dictionary hold 0, so coeff_mask's all-NaN flag comes from real atoms only
    GCCNMF_LAUNCH(h, ll_dict_fill_kernel, fill_ctas, 256, 0, stream, l.dK, l.dassign, K, T, hops, P, nullptr, l.values, nullptr);
  } else if (l.Qe) {
    if (int e = gccnmf_target_gccnmf_bank(h, l.coh, F, T, ll_bank(l, hops), D, l.W, K, l.col_targets, P, l.values, stream)) return e;
  } else if (int e = gccnmf_target_gccnmf(h, l.coh, F, T, l.E, D, l.W, K, l.col_targets, P, l.values, stream)) {
    return e;
  }
  if (int e = gccnmf_coeff_mask(h, l.values, P, K, T, l.src_mask, l.counters + 2, stream)) return e;
  const size_t KT = (size_t)K * T, FT = (size_t)F * T;
  if (l.Qd) {
    const DictBank dict = ll_dict(l, hops);
    if (inf) {
      const size_t smem = (size_t)(K + F) * sizeof(float);
      if (smem > 48 * 1024) GCCNMF_CHECK_CUDA(h, cudaFuncSetAttribute(ll_dict_infer_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      GCCNMF_LAUNCH(h, ll_dict_infer_kernel, dim3(T, 2), 256, smem, stream, dict, l.dWTi, l.dcolsumW, l.dH0, l.V, F, T, cfg->inference_iterations,
                    cfg->sparsity_alpha, cfg->epsilon, l.H);
    }
    for (int q = 0; q < P; ++q)
      if (int e = gccnmf_wiener_dict(h, l.src_mask + q * KT, dict, inf ? l.H : nullptr, l.X, F, T, l.Y + q * 4 * FT, l.wiener + q * (inf ? 2 : 1) * FT,
                                     stream))
        return e;
    GCCNMF_LAUNCH(h, ll_dict_fill_kernel, fill_ctas, 256, 0, stream, l.dK, l.dassign, K, T, hops, P, nullptr, l.src_mask, inf ? l.H : nullptr);
  } else if (inf) {
    const size_t smem = (size_t)(K + F) * sizeof(float);
    if (smem > 48 * 1024) GCCNMF_CHECK_CUDA(h, cudaFuncSetAttribute(ll_infer_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    GCCNMF_LAUNCH(h, ll_infer_kernel, dim3(T, 2), 256, smem, stream, l.W, l.WT, l.colsumW, l.H0, l.V, F, K, T, cfg->inference_iterations,
                  cfg->sparsity_alpha, cfg->epsilon, l.H);
    for (int q = 0; q < P; ++q)
      if (int e = gccnmf_wiener_apply_h(h, l.src_mask + q * KT, l.W, l.H, l.X, F, T, K, l.Y + q * 4 * FT, l.wiener + q * 2 * FT, stream)) return e;
  } else {
    for (int q = 0; q < P; ++q)
      if (int e = gccnmf_wiener_apply(h, l.src_mask + q * KT, l.W, l.X, F, T, K, l.Y + q * 4 * FT, l.wiener + q * FT, l.ws_wiener,
                                      gccnmf_wiener_apply_workspace_bytes(F), stream))
        return e;
  }
  if (int e = gccnmf_istft_frames(h, l.Y, 2 * P, N, T, 0, l.frames, stream)) return e;
  GCCNMF_LAUNCH(h, ll_src_ola_emit_kernel, dim3(S, P), 256, 0, stream, l.streams, l.head, l.w_syn, l.frames, N, hop, hops, T, l.Q, l.out_ring, out);
  GCCNMF_LAUNCH(h, ll_src_advance_kernel, S, 256, 0, stream, l.streams, hops, hop, l.stage, l.in_ring, l.R, l.counters);
  return GCCNMF_OK;
}

int ll_enqueue(gccnmf_handle* h, const gccnmf_ll_config* cfg, const LLLayout& l, int hops, const float* in, float* out, void* stream) {
  GCCNMF_REQUIRE(h, hops >= 1 && hops <= l.C, "ll_process: hops must be in [1, %d] (got %d)", l.C, hops);
  GCCNMF_REQUIRE(h, in && out, "ll_process: NULL pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const int S = l.S, N = l.N, hop = l.hop, F = l.F, K = l.K, D = l.D, T = S * hops, n = hops * hop;
  const bool inf = cfg->inference_iterations > 0;
  const int before_first = l.Q;
  GCCNMF_CHECK_CUDA(h, cudaMemsetAsync(l.counters, 0, 4 * sizeof(int32_t), st));
  GCCNMF_LAUNCH(h, ll_push_kernel, dim3(S, 2), 256, 0, stream, l.streams, in, l.in_ring, S, l.R, n, hops, before_first, l.stage, l.valid);
  const int64_t Lseg = (int64_t)l.R + n;
  if (int e = gccnmf_stft_segments(h, l.stage, (int64_t)S * Lseg, 2, S, hops, Lseg, l.win_a, N, hop, 0, l.X, inf ? l.V : nullptr, stream)) return e;
  if (l.Qe) {
    if (int e = gccnmf_phat_angspec_bank(h, l.X, F, T, ll_bank(l, hops), D, l.coh, l.ang, stream)) return e;
  } else if (int e = gccnmf_phat_angspec(h, l.X, F, T, 0, l.E, D, l.coh, l.ang, nullptr, nullptr, 0, stream)) {
    return e;
  }
  if (l.P) return ll_enqueue_sources(h, cfg, l, hops, out, stream);
  if (l.Lh)
    GCCNMF_LAUNCH(h, ll_hist_targets_kernel, S, 128, 0, stream, l.streams, l.ang, l.valid, D, hops, T, l.carry, l.acc, l.hist, l.hist_stride, l.Lh,
                  l.means, l.targets);
  else
    GCCNMF_LAUNCH(h, ll_targets_kernel, S, 128, 0, stream, l.streams, l.ang, l.valid, D, hops, T, l.carry, l.acc, l.targets);
  if (l.Qd) {
    const SteerBank b = ll_bank(l, hops);
    const DictBank dict = ll_dict(l, hops);
    if (int e = gccnmf_tdoa_argmax_dict(h, l.coh, F, T, b, dict, D, l.argmax, l.counters, l.ws_dict, l.n_dict, stream)) return e;
    if (int e = gccnmf_tdoa_gccnmf_dict(h, l.coh, F, T, b, dict, D, l.argmax, l.counters, gccnmf_tdoa_argmax_refine_capacity(K, T), l.counters + 1,
                                        stream))
      return e;
    const int64_t KT = (int64_t)K * T;
    const unsigned ctas = (unsigned)((KT + 255) / 256);
    GCCNMF_LAUNCH(h, ll_dict_mask_kernel, ctas, 256, 0, stream, l.streams, l.argmax, l.targets, l.dK, l.dassign, K, T, hops, l.mask);
    if (inf) {
      const size_t smem = (size_t)(K + F) * sizeof(float);
      if (smem > 48 * 1024) GCCNMF_CHECK_CUDA(h, cudaFuncSetAttribute(ll_dict_infer_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      GCCNMF_LAUNCH(h, ll_dict_infer_kernel, dim3(T, 2), 256, smem, stream, dict, l.dWTi, l.dcolsumW, l.dH0, l.V, F, T, cfg->inference_iterations,
                    cfg->sparsity_alpha, cfg->epsilon, l.H);
    }
    if (int e = gccnmf_wiener_dict(h, l.mask, dict, inf ? l.H : nullptr, l.X, F, T, l.Y, l.wiener, stream)) return e;
    GCCNMF_LAUNCH(h, ll_dict_fill_kernel, ctas, 256, 0, stream, l.dK, l.dassign, K, T, hops, 0, l.argmax, nullptr, inf ? l.H : nullptr);
    if (int e = gccnmf_istft_frames(h, l.Y, 2, N, T, 0, l.frames, stream)) return e;
    GCCNMF_LAUNCH(h, ll_ola_emit_kernel, S, 256, 0, stream, l.streams, l.head, l.w_syn, l.frames, N, hop, hops, T, before_first, l.out_ring, out,
                  l.stage, l.in_ring, l.R);
    return GCCNMF_OK;
  }
  if (l.Qe) {
    const SteerBank b = ll_bank(l, hops);
    if (int e = gccnmf_tdoa_argmax_bank(h, l.coh, F, T, b, D, l.W, K, l.argmax, l.counters, l.ws_argmax, l.n_argmax, stream)) return e;
    if (int e = gccnmf_tdoa_gccnmf_bank(h, l.coh, F, T, b, D, l.W, K, l.argmax, l.counters, gccnmf_tdoa_argmax_refine_capacity(K, T),
                                        l.counters + 1, stream))
      return e;
  } else {
    if (int e = gccnmf_tdoa_argmax(h, l.coh, F, T, l.E, D, l.W, K, l.argmax, l.counters, l.ws_argmax, l.n_argmax, stream)) return e;
    if (int e = gccnmf_tdoa_gccnmf_gated(h, l.coh, F, T, l.E, D, l.W, K, l.argmax, l.counters, gccnmf_tdoa_argmax_refine_capacity(K, T),
                                         l.counters + 1, stream))
      return e;
  }
  const int64_t KT = (int64_t)K * T;
  GCCNMF_LAUNCH(h, ll_mask_kernel, (unsigned)((KT + 255) / 256), 256, 0, stream, l.streams, l.argmax, l.targets, K, T, hops, l.mask);
  if (inf) {
    const size_t smem = (size_t)(K + F) * sizeof(float);
    if (smem > 48 * 1024) GCCNMF_CHECK_CUDA(h, cudaFuncSetAttribute(ll_infer_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    GCCNMF_LAUNCH(h, ll_infer_kernel, dim3(T, 2), 256, smem, stream, l.W, l.WT, l.colsumW, l.H0, l.V, F, K, T, cfg->inference_iterations,
                  cfg->sparsity_alpha, cfg->epsilon, l.H);
    if (int e = gccnmf_wiener_apply_h(h, l.mask, l.W, l.H, l.X, F, T, K, l.Y, l.wiener, stream)) return e;
  } else if (int e = gccnmf_wiener_apply(h, l.mask, l.W, l.X, F, T, K, l.Y, l.wiener, l.ws_wiener, gccnmf_wiener_apply_workspace_bytes(F), stream)) {
    return e;
  }
  if (int e = gccnmf_istft_frames(h, l.Y, 2, N, T, 0, l.frames, stream)) return e;
  GCCNMF_LAUNCH(h, ll_ola_emit_kernel, S, 256, 0, stream, l.streams, l.head, l.w_syn, l.frames, N, hop, hops, T, before_first, l.out_ring, out,
                l.stage, l.in_ring, l.R);
  return GCCNMF_OK;
}

// ---------------------------------------------------------------------------------------------- entry points (P = 0: gccnmf_ll_*)
int ll_init(gccnmf_handle* h, const gccnmf_ll_config* cfg, int P, int Lh, int Qe, int Qd, const float* W, const double* E, const double* analysis_window,
            const double* synthesis_weights, float gain, const float* H0, void* state, size_t state_bytes, void* stream) {
  GCCNMF_ENTER(h);
  LLD_CARVE_OR_FAIL(l, P, Lh, Qe, Qd);
  GCCNMF_REQUIRE(h, (W || Qd) && E && analysis_window && synthesis_weights, "ll_init: NULL pointer");
  GCCNMF_REQUIRE(h, cfg->inference_iterations == 0 || H0 != nullptr || Qd, "ll_init: inference needs H0");
  cudaStream_t s = (cudaStream_t)stream;
  // the synthesis weights decide the latency: read them here, before anything is enqueued
  double* wh = new double[l.N];
  cudaError_t err = cudaMemcpyAsync(wh, synthesis_weights, (size_t)l.N * sizeof(double), cudaMemcpyDeviceToHost, s);
  if (err == cudaSuccess) err = cudaStreamSynchronize(s);
  int z = l.N;
  for (int r = 0; r < l.N && err == cudaSuccess; ++r)
    if (wh[r] != 0.0) { z = r; break; }
  delete[] wh;
  GCCNMF_CHECK_CUDA(h, err);
  GCCNMF_REQUIRE(h, z <= l.R, "ll_init: the first nonzero synthesis weight (%d) must be at most (ceil(N / hop) - 1) hop = %d", z, l.R);
  // twiddles are cached per handle on first use (a cudaMalloc): make that happen outside any capture
  if (int st = gccnmf_get_twiddles(h, l.N, nullptr, nullptr)) return st;
  GCCNMF_CHECK_CUDA(h, cudaMemsetAsync(state, 0, l.bytes, s));
  GCCNMF_CHECK_CUDA(h, cudaMemcpyAsync(l.win_a, analysis_window, (size_t)l.N * sizeof(double), cudaMemcpyDeviceToDevice, s));
  GCCNMF_CHECK_CUDA(h, cudaMemcpyAsync(l.w_syn, synthesis_weights, (size_t)l.N * sizeof(double), cudaMemcpyDeviceToDevice, s));
  GCCNMF_CHECK_CUDA(h, cudaMemcpyAsync(l.E, E, (size_t)(Qe ? Qe : 1) * 2 * l.F * l.D * sizeof(double), cudaMemcpyDeviceToDevice, s));
  for (int j = 0; j < Qe; ++j)
    if (int st = gccnmf_steering_transpose(h, l.E + (size_t)j * 2 * l.F * l.D, l.F, l.D, l.ET + (size_t)j * 2 * l.D * l.Fp, l.Fp, stream)) return st;
  // with a bank every stream is on entry 0 (the memset above): sorted in stream order
  if (Qe) GCCNMF_LAUNCH(h, sort_by_entry_kernel, 1, 32, 0, stream, l.assign, sizeof(int32_t), l.S, Qe, l.order, l.seg);
  if (!Qd) GCCNMF_CHECK_CUDA(h, cudaMemcpyAsync(l.W, W, (size_t)l.F * l.K * sizeof(float), cudaMemcpyDeviceToDevice, s));
  if (!Qd && cfg->inference_iterations > 0) {
    GCCNMF_CHECK_CUDA(h, cudaMemcpyAsync(l.H0, H0, (size_t)l.K * 2 * sizeof(float), cudaMemcpyDeviceToDevice, s));
    GCCNMF_LAUNCH(h, ll_dict_kernel, (l.K + 127) / 128, 128, 0, stream, l.W, l.F, l.K, l.WT, l.colsumW);
  }
  GCCNMF_LAUNCH(h, ll_header_kernel, 1, 1, 0, stream, l.head, l.w_syn, l.N, gain);
  // with sources the P output rings of a stream are zeroed by ll_src_reset_kernel (N = 0 here: no single ring)
  GCCNMF_LAUNCH(h, ll_reset_kernel, l.S, 256, 0, stream, l.streams, 0, l.S, l.in_ring, l.out_ring, l.carry, l.R, P ? 0 : l.N, l.D, 1);
  if (P)
    GCCNMF_LAUNCH(h, ll_src_reset_kernel, l.S, 256, 0, stream, 0, l.S, P, l.D, l.N, l.out_ring, l.src_targets, l.src_override, l.src_status, 1);
  // the history is zeroed by the memset above: ring, write index 0, window 0
  return GCCNMF_OK;
}

int ll_reset_streams(gccnmf_handle* h, const gccnmf_ll_config* cfg, int P, int Lh, int Qe, int Qd, void* state, size_t state_bytes, int first, int count,
                     void* stream) {
  GCCNMF_ENTER(h);
  LLD_CARVE_OR_FAIL(l, P, Lh, Qe, Qd);
  if (int st = stream_range_check(h, "ll_reset_streams", l.S, first, count)) return st;
  GCCNMF_LAUNCH(h, ll_reset_kernel, count, 256, 0, stream, l.streams, first, count, l.in_ring, l.out_ring, l.carry, l.R, P ? 0 : l.N, l.D, 0);
  if (P)
    GCCNMF_LAUNCH(h, ll_src_reset_kernel, count, 256, 0, stream, first, count, P, l.D, l.N, l.out_ring, l.src_targets, l.src_override, l.src_status, 0);
  if (Lh) GCCNMF_LAUNCH(h, ll_hist_reset_kernel, count, 256, 0, stream, l.hist, l.hist_stride, first, count);
  if (Qe) {
    if (int st = enqueue_stream_fill(h, l.assign, sizeof(int32_t), first, count, 0, stream)) return st;
    GCCNMF_LAUNCH(h, sort_by_entry_kernel, 1, 32, 0, stream, l.assign, sizeof(int32_t), l.S, Qe, l.order, l.seg);
  }
  if (Qd) {
    if (int st = enqueue_stream_fill(h, l.dassign, sizeof(int32_t), first, count, 0, stream)) return st;
    GCCNMF_LAUNCH(h, sort_by_entry_kernel, 1, 32, 0, stream, l.dassign, sizeof(int32_t), l.S, Qd, l.dorder, l.dseg);
  }
  return GCCNMF_OK;
}

int ll_set_params(gccnmf_handle* h, const gccnmf_ll_config* cfg, int P, int Lh, int Qe, int Qd, void* state, size_t state_bytes, int first, int count,
                  const gccnmf_ll_stream_params* params_host, void* stream) {
  GCCNMF_ENTER(h);
  LLD_CARVE_OR_FAIL(l, P, Lh, Qe, Qd);
  if (int st = stream_range_check(h, "ll_set_params", l.S, first, count)) return st;
  GCCNMF_REQUIRE(h, params_host != nullptr, "ll_set_params: NULL parameters");
  for (int i = 0; i < count; ++i) {
    GCCNMF_REQUIRE(h, !std::isnan(params_host[i].epsilon), "ll_set_params: stream %d: epsilon is NaN", first + i);
    GCCNMF_REQUIRE(h, params_host[i].target_override >= -1 && params_host[i].target_override < l.D,
                   "ll_set_params: stream %d: target_override %d outside [0, %d) (or -1)", first + i, params_host[i].target_override, l.D);
  }
  for (int i0 = 0; i0 < count; i0 += kLLParamsPerLaunch) {
    const int n = count - i0 < kLLParamsPerLaunch ? count - i0 : kLLParamsPerLaunch;
    LLParamsBatch b{};
    memcpy(b.p, params_host + i0, (size_t)n * sizeof(gccnmf_ll_stream_params));
    GCCNMF_LAUNCH(h, ll_params_kernel, 1, kLLParamsPerLaunch, 0, stream, l.streams, first + i0, n, b);
  }
  return GCCNMF_OK;
}

int ll_graph_create(gccnmf_handle* h, const gccnmf_ll_config* cfg, int P, int Lh, int Qe, int Qd, void* state, size_t state_bytes, int hops, float* in, float* out,
                    const float* in_host, float* out_host, void** graph_exec, void* stream) {
  GCCNMF_ENTER(h);
  GCCNMF_REQUIRE(h, graph_exec != nullptr && stream != nullptr, "ll_graph_create: needs a non-default stream and an output slot");
  *graph_exec = nullptr;
  LLD_CARVE_OR_FAIL(l, P, Lh, Qe, Qd);
  GCCNMF_REQUIRE(h, hops >= 1 && hops <= l.C, "ll_graph_create: hops must be in [1, %d] (got %d)", l.C, hops);
  GCCNMF_REQUIRE(h, in && out, "ll_graph_create: NULL pointer");
  if (int st = gccnmf_get_twiddles(h, l.N, nullptr, nullptr)) return st;
  const size_t bytes = (size_t)l.S * 2 * hops * l.hop * sizeof(float);
  return capture_graph(h, "ll_graph_create", stream, in, in_host, bytes, out, out_host, bytes * (P ? P : 1),
                       [&] { return ll_enqueue(h, cfg, l, hops, in, out, stream); }, graph_exec);
}

int ll_export(gccnmf_handle* h, const gccnmf_ll_config* cfg, int P, int Lh, int Qe, int Qd, void* state, size_t state_bytes, int hops, int what, void* dst,
              void* stream) {
  GCCNMF_ENTER(h);
  LLD_CARVE_OR_FAIL(l, P, Lh, Qe, Qd);
  GCCNMF_REQUIRE(h, dst != nullptr, "ll_export: NULL destination");
  GCCNMF_REQUIRE(h, hops >= 1 && hops <= l.C, "ll_export: hops must be in [1, %d] (got %d)", l.C, hops);
  const bool inf = cfg->inference_iterations > 0;
  const size_t T = (size_t)l.S * hops, F = l.F, K = l.K, D = l.D, Ps = P;
  if (what == GCCNMF_LLBANK_EXPORT_ASSIGNMENT) {
    GCCNMF_REQUIRE(h, Qe > 0, "ll_export: item %d needs num_steerings > 0", what);
    GCCNMF_CHECK_CUDA(h, cudaMemcpyAsync(dst, l.assign, (size_t)l.S * sizeof(int32_t), cudaMemcpyDefault, (cudaStream_t)stream));
    return GCCNMF_OK;
  }
  if (what == GCCNMF_LLDICT_EXPORT_DICTIONARY_ASSIGNMENT || what == GCCNMF_LLDICT_EXPORT_DICTIONARY_ATOMS) {
    GCCNMF_REQUIRE(h, Qd > 0, "ll_export: item %d needs num_dictionaries > 0", what);
    const bool atoms = what == GCCNMF_LLDICT_EXPORT_DICTIONARY_ATOMS;
    GCCNMF_CHECK_CUDA(h, cudaMemcpyAsync(dst, atoms ? l.dK : l.dassign, (size_t)(atoms ? Qd : l.S) * sizeof(int32_t), cudaMemcpyDefault,
                                         (cudaStream_t)stream));
    return GCCNMF_OK;
  }
  if (what >= GCCNMF_LLHIST_EXPORT_RING && what <= GCCNMF_LLHIST_EXPORT_MEANS) {
    GCCNMF_REQUIRE(h, Lh > 0, "ll_export: item %d needs history_length > 0", what);
    const size_t ring = D * Lh * sizeof(double);
    cudaStream_t st = (cudaStream_t)stream;
    switch (what) {
      case GCCNMF_LLHIST_EXPORT_RING:
        GCCNMF_CHECK_CUDA(h, cudaMemcpy2DAsync(dst, ring, l.hist, l.hist_stride, ring, l.S, cudaMemcpyDefault, st));
        break;
      case GCCNMF_LLHIST_EXPORT_INDEX: case GCCNMF_LLHIST_EXPORT_WINDOWS:
        GCCNMF_CHECK_CUDA(h, cudaMemcpy2DAsync(dst, 4, l.hist + ring + (what == GCCNMF_LLHIST_EXPORT_WINDOWS ? 4 : 0), l.hist_stride, 4, l.S,
                                               cudaMemcpyDefault, st));
        break;
      default: GCCNMF_CHECK_CUDA(h, cudaMemcpyAsync(dst, l.means, D * T * sizeof(double), cudaMemcpyDefault, st)); break;
    }
    return GCCNMF_OK;
  }
  const void* src = nullptr;
  size_t bytes = 0;
  if (P) {   // the items of the single-target chain that this mode does not compute are refused
    switch (what) {
      case 0: case 1: case 2: case 3: case 11: case 12: case 13: break;
      case GCCNMF_LLSEP_EXPORT_TARGETS: src = l.col_targets; bytes = T * Ps * 4; break;
      case GCCNMF_LLSEP_EXPORT_VALUES: src = l.values; bytes = Ps * K * T * 4; break;
      case GCCNMF_LLSEP_EXPORT_MASKS: src = l.src_mask; bytes = Ps * K * T * 4; break;
      case GCCNMF_LLSEP_EXPORT_WIENER: src = l.wiener; bytes = Ps * (inf ? 2 : 1) * F * T * 4; break;
      case GCCNMF_LLSEP_EXPORT_Y: src = l.Y; bytes = Ps * 2 * F * T * 8; break;
      case GCCNMF_LLSEP_EXPORT_STREAM_STATUS: src = l.src_status; bytes = (size_t)l.S * 4; break;
      case GCCNMF_LLSEP_EXPORT_CARRIED_TARGETS:
        GCCNMF_CHECK_CUDA(h, cudaMemcpy2DAsync(dst, Ps * 4, l.src_targets, kLLMaxSources * 4, Ps * 4, l.S, cudaMemcpyDefault, (cudaStream_t)stream));
        return GCCNMF_OK;
      case GCCNMF_LLSEP_EXPORT_CALL_STATUS: src = l.counters + 3; bytes = 4; break;
      default: return gccnmf_fail(h, GCCNMF_ERR_INVALID_ARGUMENT, "llsep_export: item %d is not computed with sources", what);
    }
  }
  if (!src) {
    switch (what) {
      case 0: src = l.X; bytes = 2 * F * T * 8; break;
      case 1: src = l.coh; bytes = F * T * 8; break;
      case 2: src = l.ang; bytes = D * T * 8; break;
      case 3: src = l.acc; bytes = D * T * 8; break;
      case 4: src = l.targets; bytes = T * 4; break;
      case 5: src = l.argmax; bytes = K * T * 4; break;
      case 6: src = l.mask; bytes = K * T * 4; break;
      case 7: src = l.wiener; bytes = (inf ? 2 : 1) * F * T * 4; break;
      case 8: src = l.Y; bytes = 2 * F * T * 8; break;
      case 9: src = l.counters; bytes = 4; break;
      case 10: src = l.counters + 1; bytes = 4; break;
      case 11: if (inf) { src = l.H; bytes = K * 2 * T * 4; } break;
      case 12: src = l.valid; bytes = T * 4; break;
      case 13: src = l.carry; bytes = (size_t)l.S * D * 8; break;
      default: break;
    }
  }
  if (!src) return gccnmf_fail(h, GCCNMF_ERR_INVALID_ARGUMENT, "ll_export: unknown item %d", what);
  GCCNMF_CHECK_CUDA(h, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDefault, (cudaStream_t)stream));
  return GCCNMF_OK;
}

// ---------------------------------------------------------------------------------------------- stream records
// The persistent state of stream s is every byte a later call reads that an earlier call or a setting wrote:
//   streams[s]        hops (frame validity, ring positions), epsilon, active, target_override       (ll_push, ll_mask, ll_*emit)
//   carry[s]          D running maxima                                                               (ll_running_max)
//   in_ring[s]        the last R samples of both channels                                            (ll_push <- ll_advance)
//   out_ring[s]       the N-sample overlap-add ring of both channels, P of them with sources         (ll_ola_emit)
//   src_targets[s], src_override[s], src_status[s]    (sources only)                                (ll_src_targets_kernel)
//   hist[s]           history only: the ring, its write index, the window and 8 zero bytes          (ll_hist_means, set_window)
// Everything else is either shared by the streams (header, windows, E, W and what init derives from it) or rewritten by every call
// before it is read (stage, valid, X ... frames, counters).  A region is an array of per-stream blocks in the state (RecordMapBuilder
// with stride 0), and the payload's padding after each region is zero.  Rings are copied whole: their
// positions derive from hops, which travels with them.
constexpr size_t kRecordHeaderBytes = GCCNMF_RECORD_HEADER_BYTES;
static_assert(sizeof(gccnmf_llbank_record_header) <= kRecordHeaderBytes, "record header");
static_assert(offsetof(gccnmf_llbank_record_header, config) == offsetof(gccnmf_record_header, config), "shared prefix");

// A bank (Qe >= 1) moves the regions' offsets in the state (E holds Qe tables), not the payload.
RecordMap ll_record_map(const gccnmf_ll_config& c, int P, int Lh = 0, int Qe = 0) {
  char* const base = reinterpret_cast<char*>(256);
  const LLLayout l = ll_carve(c, P, base, Lh, Qe);
  const size_t N = l.N, R = l.R, D = l.D, Pm = P > 0 ? P : 1;
  RecordMapBuilder b{base, 0};
  b.add(l.streams, sizeof(LLStream));
  b.add(l.carry, D * sizeof(double));
  b.add(l.in_ring, 2 * R * sizeof(float));  // nothing when hop = N (R = 0)
  b.add(l.out_ring, Pm * 2 * N * sizeof(float));
  if (P) {
    b.add(l.src_targets, kLLMaxSources * sizeof(int32_t));
    b.add(l.src_override, kLLMaxSources * sizeof(int32_t));
    b.add(l.src_status, sizeof(int32_t));
  }
  b.add(l.hist, l.hist_stride);            // nothing with Lh = 0: the records of gccnmf_llrec_*
  return b.m;
}

size_t ll_record_bytes(const gccnmf_ll_config& c, int P, int Lh = 0) {
  return kRecordHeaderBytes + align_up(ll_record_map(c, P, Lh).payload, 256);
}

// Grid (count, regions): CTA (i, g) copies region g of stream first + i between the state and payload i of the staging buffer.
__global__ void __launch_bounds__(256)
ll_record_copy_kernel(char* __restrict__ state, int first, RecordMap m, char* __restrict__ staging, int to_staging) {
  record_copy_region(state, first + blockIdx.x, m.r[blockIdx.y], staging + (size_t)blockIdx.x * m.payload, to_staging);
}

// What a record must agree on, from the host arguments alone: magic, ABI version, kind, P, payload size and the configuration without
// S and C, followed by the history length (0 without history, so those records are gccnmf_llrec_*'s).  The synthesis digest is left
// 0: see ll_synthesis_digest.
constexpr int kRecordConfigHistory = sizeof(gccnmf_ll_config) / sizeof(int32_t);    // config[9]
constexpr int kConfigAtoms = offsetof(gccnmf_ll_config, num_atoms) / sizeof(int32_t);
// With a bank (Qe >= 1) the kind is GCCNMF_RECORD_KIND_LLBANK, and the content digests of the dictionary and of the stream's
// steering table follow the same fields (gccnmf_llbank_record_header; 0 without a bank).
gccnmf_llbank_record_header ll_record_header(const gccnmf_ll_config& cfg, int P, int Lh = 0, int Qe = 0) {
  gccnmf_llbank_record_header r{};
  r.magic = GCCNMF_RECORD_MAGIC;
  r.abi_version = GCCNMF_ABI_VERSION;
  r.kind = Qe ? GCCNMF_RECORD_KIND_LLBANK : GCCNMF_RECORD_KIND_LL;
  r.num_sources = P;
  r.payload_bytes = ll_record_map(cfg, P, Lh).payload;
  gccnmf_ll_config c = cfg;
  c.num_streams = 0;
  c.hops_per_call = 0;
  static_assert(sizeof(c) + sizeof(int32_t) <= sizeof(r.config), "record config");
  memcpy(r.config, &c, sizeof(c));
  r.config[kRecordConfigHistory] = Lh;
  return r;
}

// FNV-1a 64 of the synthesis weights' bytes followed by the gain's.  Both live only in the state, so they are read back on the
// stream and waited for, as init reads the weights.
int ll_synthesis_digest(gccnmf_handle* h, const LLLayout& l, uint64_t* digest, void* stream) {
  const size_t wb = (size_t)l.N * sizeof(double);
  unsigned char* w = new unsigned char[wb + sizeof(LLHeader)];
  cudaStream_t s = (cudaStream_t)stream;
  cudaError_t err = cudaMemcpyAsync(w, l.w_syn, wb, cudaMemcpyDeviceToHost, s);
  if (err == cudaSuccess) err = cudaMemcpyAsync(w + wb, l.head, sizeof(LLHeader), cudaMemcpyDeviceToHost, s);
  if (err == cudaSuccess) err = cudaStreamSynchronize(s);
  uint64_t d = 1469598103934665603ull;
  for (size_t i = 0; i < wb + sizeof(float); ++i) d = (d ^ w[i]) * 1099511628211ull;    // the weights, then LLHeader::gain
  delete[] w;
  GCCNMF_CHECK_CUDA(h, err);
  *digest = d;
  return GCCNMF_OK;
}

// ---- bank records (Qe >= 1): the content digests of the dictionaries and the steering tables.  A steering bank's state is one
// dictionary, l.W and l.H0 with the config's K; a dictionary bank's dictionary e is dW and dH0 of entry e with K_e atoms.  The
// workspace holds the records' payloads, then chunk slots for one dictionary of K_max atoms and for each table, then the digests:
// [0] dictionary 0, [1 .. Qe] the tables, [Qe + e] dictionary e >= 1.  Each dictionary's digest is the llbank digest of an engine
// built with it.
struct LLRecordWork {
  int cd, ce;                            // chunk slots of a dictionary and of a table
  size_t chunks, digests, bytes;
};
LLRecordWork ll_record_work(const gccnmf_ll_config& c, int P, int Lh, int Qe, int Qd, int count) {
  LLRecordWork w{};
  w.bytes = (size_t)count * ll_record_map(c, P, Lh).payload;
  if (!Qe) return w;
  const size_t F = c.window_size / 2 + 1, K = c.num_atoms;
  w.cd = digest_chunks(F * K + (c.inference_iterations > 0 ? 2 * K : 0));
  w.ce = digest_chunks(4 * F * c.num_tdoas);
  w.chunks = align_up(w.bytes, 256);
  w.digests = w.chunks + align_up((size_t)(w.cd + Qe * w.ce) * sizeof(uint64_t), 256);
  w.bytes = w.digests + (size_t)((Qd ? Qd : 1) + Qe) * sizeof(uint64_t);
  return w;
}

// The digests of this state's dictionaries and tables, with their K (dict_digest, K_host: max(Qd, 1); steer_digest: Qe), and when
// the entry arrays are not NULL the entries of streams [first, first + count), back to the host.  One launch pair per dictionary,
// the tables with the first, and one wait, after another for the K_e table of a dictionary bank.
int ll_record_digests(gccnmf_handle* h, const gccnmf_ll_config& c, const LLLayout& l, const LLRecordWork& w, char* workspace, int first, int count,
                      uint64_t* dict_digest, uint64_t* steer_digest, int32_t* K_host, int32_t* dict_entries, int32_t* steer_entries, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  const int nd = l.Qd ? l.Qd : 1;
  const size_t inf = c.inference_iterations > 0 ? 2 : 0;
  K_host[0] = l.K;
  if (l.Qd) {
    GCCNMF_CHECK_CUDA(h, cudaMemcpyAsync(K_host, l.dK, (size_t)nd * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    GCCNMF_CHECK_CUDA(h, cudaStreamSynchronize(s));
  }
  uint64_t* chunks = reinterpret_cast<uint64_t*>(workspace + w.chunks);
  uint64_t* dev = reinterpret_cast<uint64_t*>(workspace + w.digests);
  for (int e = 0; e < nd; ++e) {
    GCCNMF_REQUIRE(h, K_host[e] >= 1 && K_host[e] <= l.K, "lldict: dictionary entry %d has %d atoms", e, K_host[e]);
    DigestItems d{};
    d.g[d.n++] = l.Qd ? DigestGroup{l.dW + (size_t)e * l.F * l.Kp, l.dH0 + (size_t)e * l.Kp * 2, 0, 0, (size_t)l.F, inf, l.dK + e, 0, 1, w.cd}
                      : DigestGroup{l.W, l.H0, 0, 0, (size_t)l.F * l.K, inf * l.K, nullptr, l.K, 1, w.cd};
    const size_t table = (size_t)4 * l.F * l.D;       // words of one (F, D) complex128 table
    if (e == 0) d.g[d.n++] = DigestGroup{l.E, nullptr, table * sizeof(uint32_t), 0, table, 0, nullptr, 0, l.Qe, w.ce};
    if (int st = record_enqueue_digests(h, d, chunks, dev + (e == 0 ? 0 : l.Qe + e), nullptr, stream)) return st;
  }
  uint64_t all[kLLMaxDictionaries + kLLMaxSteerings];
  GCCNMF_CHECK_CUDA(h, cudaMemcpyAsync(all, dev, (size_t)(nd + l.Qe) * sizeof(uint64_t), cudaMemcpyDeviceToHost, s));
  if (dict_entries && l.Qd)
    GCCNMF_CHECK_CUDA(h, cudaMemcpyAsync(dict_entries, l.dassign + first, (size_t)count * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  if (steer_entries) GCCNMF_CHECK_CUDA(h, cudaMemcpyAsync(steer_entries, l.assign + first, (size_t)count * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  GCCNMF_CHECK_CUDA(h, cudaStreamSynchronize(s));
  dict_digest[0] = all[0];
  for (int j = 0; j < l.Qe; ++j) steer_digest[j] = all[1 + j];
  for (int e = 1; e < nd; ++e) dict_digest[e] = all[l.Qe + e];
  return GCCNMF_OK;
}

// Qd >= 1 only with Qe >= 1 (ll_check); the lldict entries check Qd >= 1 themselves.
#define LL_RECORD_ARGS_OR_FAIL(what)                                                                                                   \
  LLD_CARVE_OR_FAIL(l, P, Lh, Qe, Qd);                                                                                                 \
  if (int st__ = stream_range_check(h, what, l.S, first, count)) return st__;                                                          \
  const RecordMap m = ll_record_map(*cfg, P, Lh, Qe);                                                                                  \
  const size_t rec_bytes = ll_record_bytes(*cfg, P, Lh);                                                                               \
  GCCNMF_REQUIRE(h, record != nullptr && record_bytes >= (size_t)count * rec_bytes, "%s: record needs %zu bytes for %d streams", what,  \
                 (size_t)count * rec_bytes, count);                                                                                    \
  const LLRecordWork w = ll_record_work(*cfg, P, Lh, Qe, Qd, count);                                                                   \
  if (workspace == nullptr || workspace_bytes < w.bytes || ((uintptr_t)workspace & (Qe ? 7 : 3)) != 0)                                 \
    return gccnmf_fail(h, GCCNMF_ERR_WORKSPACE, "%s: workspace needs %zu bytes, %d-byte aligned", what, w.bytes, Qe ? 8 : 4);

// Every record byte a save writes is defined: the header's tail and the record's tail past the payload are zeroed here, the
// payload's padding by the copy kernel.  The host writes its bytes while the device copies the payloads (other bytes of the same
// records): at thousands of streams those writes miss the cache and would otherwise add to the save.
int ll_save_streams(gccnmf_handle* h, const gccnmf_ll_config* cfg, int P, int Lh, int Qe, int Qd, void* state, size_t state_bytes, int first, int count, void* record,
                    size_t record_bytes, void* workspace, size_t workspace_bytes, void* stream) {
  GCCNMF_ENTER(h);
  const char* what = Qd ? "lldict_save_streams" : "ll_save_streams";
  LL_RECORD_ARGS_OR_FAIL(what);
  gccnmf_llbank_record_header head = ll_record_header(*cfg, P, Lh, Qe);
  if (int st = ll_synthesis_digest(h, l, &head.synthesis_digest, stream)) return st;
  uint64_t dd[kLLMaxDictionaries], sd[kLLMaxSteerings];
  int32_t Kh[kLLMaxDictionaries];
  std::vector<int32_t> de(count, 0), se(count, 0);
  if (Qe)
    if (int st = ll_record_digests(h, *cfg, l, w, (char*)workspace, first, count, dd, sd, Kh, de.data(), se.data(), stream)) return st;
  GCCNMF_LAUNCH(h, ll_record_copy_kernel, dim3(count, m.n), 256, 0, stream, (char*)state, first, m, (char*)workspace, 1);
  GCCNMF_CHECK_CUDA(h, cudaMemcpy2DAsync((char*)record + kRecordHeaderBytes, rec_bytes, workspace, m.payload, m.payload, count,
                                         cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  for (int i = 0; i < count; ++i) {
    char* rec = (char*)record + (size_t)i * rec_bytes;
    if (Qe) {                            // the bank header: the digests of the stream's dictionary and table
      head.dictionary_digest = dd[de[i]];
      head.steering_digest = sd[se[i]];
      if (Qd) head.config[kConfigAtoms] = Kh[de[i]];     // the header an llbank engine built with the stream's dictionary writes
    }
    memcpy(rec, &head, sizeof(head));
    memset(rec + sizeof(head), 0, kRecordHeaderBytes - sizeof(head));
    memset(rec + kRecordHeaderBytes + m.payload, 0, rec_bytes - kRecordHeaderBytes - m.payload);
  }
  return GCCNMF_OK;
}

int ll_load_streams(gccnmf_handle* h, const gccnmf_ll_config* cfg, int P, int Lh, int Qe, int Qd, void* state, size_t state_bytes, int first, int count, const void* record,
                    size_t record_bytes, void* workspace, size_t workspace_bytes, void* stream) {
  GCCNMF_ENTER(h);
  const char* what = Qd ? "lldict_load_streams" : "ll_load_streams";
  LL_RECORD_ARGS_OR_FAIL(what);
  const gccnmf_llbank_record_header want = ll_record_header(*cfg, P, Lh, Qe);
  auto header = [&](int i) {
    gccnmf_llbank_record_header got;
    memcpy(&got, (const char*)record + (size_t)i * rec_bytes, sizeof(got));
    return got;
  };
  for (int i = 0; i < count; ++i) {      // everything but the digests, before the device is touched
    gccnmf_llbank_record_header got = header(i);
    const int K = got.config[kConfigAtoms];
    if (Qd) {                            // a dictionary bank's records carry the stream's K_i
      GCCNMF_REQUIRE(h, K >= 1 && K <= l.K, "%s: record %d: %d atoms, this engine holds at most %d", what, i, K, l.K);
      got.config[kConfigAtoms] = want.config[kConfigAtoms];
    }
    if (int st = record_check_header(h, what, i, &got, &want, offsetof(gccnmf_record_header, config))) return st;
  }
  uint64_t digest = 0;
  if (int st = ll_synthesis_digest(h, l, &digest, stream)) return st;
  for (int i = 0; i < count; ++i)
    GCCNMF_REQUIRE(h, header(i).synthesis_digest == digest, "%s: record %d: other synthesis weights or gain", what, i);
  // bank: the lowest entries holding the record's dictionary (same content and K) and table (only the read-only digest kernels have
  // run when this refuses)
  std::vector<int32_t> de(count), se(count);
  if (Qe) {
    const int nd = Qd ? Qd : 1;
    uint64_t dd[kLLMaxDictionaries], sd[kLLMaxSteerings];
    int32_t Kh[kLLMaxDictionaries];
    if (int st = ll_record_digests(h, *cfg, l, w, (char*)workspace, first, count, dd, sd, Kh, nullptr, nullptr, stream)) return st;
    for (int i = 0; i < count; ++i) {
      const gccnmf_llbank_record_header got = header(i);
      const int K = got.config[kConfigAtoms], same = record_find_entry(dd, nullptr, nd, got.dictionary_digest, 0);
      de[i] = record_find_entry(dd, Kh, nd, got.dictionary_digest, K);
      se[i] = record_find_entry(sd, nullptr, Qe, got.steering_digest, 0);
      GCCNMF_REQUIRE(h, same >= 0, "%s: record %d: no dictionary entry of this engine holds the stream's dictionary", what, i);
      GCCNMF_REQUIRE(h, de[i] >= 0, "%s: record %d: the stream's dictionary has %d atoms, the entry holding it %d", what, i, K, Kh[same]);
      GCCNMF_REQUIRE(h, se[i] >= 0, "%s: record %d: no steering entry of this engine has the stream's table", what, i);
    }
  }
  GCCNMF_CHECK_CUDA(h, cudaMemcpy2DAsync(workspace, m.payload, (const char*)record + kRecordHeaderBytes, rec_bytes, m.payload, count,
                                         cudaMemcpyHostToDevice, (cudaStream_t)stream));
  GCCNMF_LAUNCH(h, ll_record_copy_kernel, dim3(count, m.n), 256, 0, stream, (char*)state, first, m, (char*)workspace, 0);
  for (int pass = Qd ? 0 : 1; Qe && pass < 2; ++pass)      // the dictionary entries (Qd >= 1), then the tables
    if (int st = enqueue_stream_rows(h, pass ? l.assign : l.dassign, sizeof(int32_t), 0, first, count, 1, (pass ? se : de).data(), false, stream))
      return st;
  if (Qe) GCCNMF_LAUNCH(h, sort_by_entry_kernel, 1, 32, 0, stream, l.assign, sizeof(int32_t), l.S, Qe, l.order, l.seg);
  if (Qd) GCCNMF_LAUNCH(h, sort_by_entry_kernel, 1, 32, 0, stream, l.dassign, sizeof(int32_t), l.S, Qd, l.dorder, l.dseg);
  return GCCNMF_OK;
}

int ll_set_targets(gccnmf_handle* h, const gccnmf_ll_config* cfg, int P, int Lh, int Qe, int Qd, void* state, size_t state_bytes, int first, int count,
                   const int32_t* targets_host, void* stream) {
  GCCNMF_ENTER(h);
  LLD_CARVE_OR_FAIL(l, P, Lh, Qe, Qd);
  if (int st = stream_range_check(h, "llsep_set_targets", l.S, first, count)) return st;
  GCCNMF_REQUIRE(h, targets_host != nullptr, "llsep_set_targets: NULL targets");
  for (int i = 0; i < count * P; ++i)
    GCCNMF_REQUIRE(h, targets_host[i] >= -1 && targets_host[i] < l.D, "llsep_set_targets: stream %d source %d: target %d outside [0, %d) (or -1)",
                   first + i / P, i % P, targets_host[i], l.D);
  return enqueue_stream_rows(h, l.src_override, kLLMaxSources * sizeof(int32_t), 0, first, count, P, targets_host, false, stream);
}

int ll_set_window(gccnmf_handle* h, const gccnmf_ll_config* cfg, int P, int Lh, int Qe, int Qd, void* state, size_t state_bytes, int first, int count,
                  const int32_t* windows_host, void* stream) {
  GCCNMF_ENTER(h);
  LLD_CARVE_OR_FAIL(l, P, Lh, Qe, Qd);
  GCCNMF_REQUIRE(h, Lh > 0, "llhist_set_window: needs history_length > 0");
  if (int st = stream_range_check(h, "llhist_set_window", l.S, first, count)) return st;
  GCCNMF_REQUIRE(h, windows_host != nullptr, "llhist_set_window: NULL windows");
  for (int i = 0; i < count; ++i)
    GCCNMF_REQUIRE(h, windows_host[i] >= 0 && windows_host[i] <= Lh, "llhist_set_window: stream %d: window %d outside [0, %d]", first + i,
                   windows_host[i], Lh);
  return enqueue_stream_rows(h, l.hist, l.hist_stride, (size_t)l.D * Lh * sizeof(double) + 4, first, count, 1, windows_host, false, stream);
}

// Bank: table j <- E (F, D) complex128 on the device, and its transpose; stream-ordered, from the next call on.
int ll_load_steering(gccnmf_handle* h, const gccnmf_ll_config* cfg, int P, int Lh, int Qe, int Qd, void* state, size_t state_bytes, int entry,
                     const double* E, void* stream) {
  GCCNMF_ENTER(h);
  LLD_CARVE_OR_FAIL(l, P, Lh, Qe, Qd);
  GCCNMF_REQUIRE(h, entry >= 0 && entry < Qe, "llbank_load_steering: entry %d outside [0, %d)", entry, Qe);
  GCCNMF_REQUIRE(h, E != nullptr, "llbank_load_steering: NULL table");
  double* dst = l.E + (size_t)entry * 2 * l.F * l.D;
  GCCNMF_CHECK_CUDA(h, cudaMemcpyAsync(dst, E, (size_t)2 * l.F * l.D * sizeof(double), cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return gccnmf_steering_transpose(h, dst, l.F, l.D, l.ET + (size_t)entry * 2 * l.D * l.Fp, l.Fp, stream);
}

// Bank: streams [first, first + count) onto entries_host[0 .. count), then the streams sorted again; stream-ordered.
int ll_assign(gccnmf_handle* h, const gccnmf_ll_config* cfg, int P, int Lh, int Qe, int Qd, void* state, size_t state_bytes, int first, int count,
              const int32_t* entries_host, void* stream) {
  GCCNMF_ENTER(h);
  LLD_CARVE_OR_FAIL(l, P, Lh, Qe, Qd);
  if (int st = stream_range_check(h, "llbank_assign", l.S, first, count)) return st;
  GCCNMF_REQUIRE(h, entries_host != nullptr, "llbank_assign: NULL entries");
  for (int i = 0; i < count; ++i)
    GCCNMF_REQUIRE(h, entries_host[i] >= 0 && entries_host[i] < Qe, "llbank_assign: stream %d: entry %d outside [0, %d)", first + i, entries_host[i], Qe);
  if (int st = enqueue_stream_rows(h, l.assign, sizeof(int32_t), 0, first, count, 1, entries_host, false, stream)) return st;
  GCCNMF_LAUNCH(h, sort_by_entry_kernel, 1, 32, 0, stream, l.assign, sizeof(int32_t), l.S, Qe, l.order, l.seg);
  return GCCNMF_OK;
}


// ---- dictionary bank (gccnmf_lldict_*)

// Entry e <- W (F, K) f32 and, with inference, H0 (K, 2) f32 (device arrays), with every form derived from them; stream-ordered.
int lld_load_entry(gccnmf_handle* h, const gccnmf_ll_config* cfg, const LLLayout& l, int e, const float* W, int K, const float* H0, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  float* dst = l.dW + (size_t)e * l.F * l.Kp;
  GCCNMF_CHECK_CUDA(h, cudaMemcpyAsync(dst, W, (size_t)l.F * K * sizeof(float), cudaMemcpyDeviceToDevice, s));
  if (int st = gccnmf_lldict_prepare(h, ll_dict(l, 1), e, dst, l.F, K, stream)) return st;
  if (int st = gccnmf_rowsum_w(h, dst, l.F, K, l.drowsum + (size_t)e * l.F, stream)) return st;
  if (cfg->inference_iterations > 0) {
    GCCNMF_CHECK_CUDA(h, cudaMemcpyAsync(l.dH0 + (size_t)e * l.Kp * 2, H0, (size_t)K * 2 * sizeof(float), cudaMemcpyDeviceToDevice, s));
    GCCNMF_LAUNCH(h, ll_dict_kernel, (K + 127) / 128, 128, 0, stream, dst, l.F, K, l.dWTi + (size_t)e * l.Kp * l.F, l.dcolsumW + (size_t)e * l.Kp);
  }
  GCCNMF_LAUNCH(h, ll_set_int_kernel, 1, 1, 0, stream, l.dK + e, K);
  return GCCNMF_OK;
}

int lld_check_entry(gccnmf_handle* h, const gccnmf_ll_config* cfg, const LLLayout& l, int e, const float* W, int K, const float* H0) {
  GCCNMF_REQUIRE(h, e >= 0 && e < l.Qd, "lldict: dictionary entry %d outside [0, %d)", e, l.Qd);
  GCCNMF_REQUIRE(h, W != nullptr, "lldict: entry %d: NULL W", e);
  GCCNMF_REQUIRE(h, K >= 1 && K <= l.K, "lldict: entry %d: num_atoms %d outside [1, %d] (the config's num_atoms)", e, K, l.K);
  GCCNMF_REQUIRE(h, cfg->inference_iterations == 0 || H0 != nullptr, "lldict: entry %d: inference needs H0", e);
  return 0;
}

int lld_init(gccnmf_handle* h, const gccnmf_ll_config* cfg, int P, int Lh, int Qd, int Qe, const float* const* W, const int* num_atoms, const double* E,
             const double* analysis_window, const double* synthesis_weights, float gain, const float* const* H0, void* state, size_t state_bytes,
             void* stream) {
  GCCNMF_ENTER(h);
  GCCNMF_REQUIRE(h, Qd >= 1, "lldict: num_dictionaries must be in [1, %d] (got %d)", kLLMaxDictionaries, Qd);
  LLD_CARVE_OR_FAIL(l, P, Lh, Qe, Qd);
  GCCNMF_REQUIRE(h, W && num_atoms, "lldict_init: NULL dictionaries");
  GCCNMF_REQUIRE(h, cfg->inference_iterations == 0 || H0, "lldict_init: inference needs H0");
  for (int e = 0; e < Qd; ++e)
    if (int st = lld_check_entry(h, cfg, l, e, W[e], num_atoms[e], H0 ? H0[e] : nullptr)) return st;
  if (int st = ll_init(h, cfg, P, Lh, Qe, Qd, nullptr, E, analysis_window, synthesis_weights, gain, nullptr, state, state_bytes, stream)) return st;
  for (int e = 0; e < Qd; ++e)
    if (int st = lld_load_entry(h, cfg, l, e, W[e], num_atoms[e], H0 ? H0[e] : nullptr, stream)) return st;
  GCCNMF_LAUNCH(h, sort_by_entry_kernel, 1, 32, 0, stream, l.dassign, sizeof(int32_t), l.S, Qd, l.dorder, l.dseg);     // every stream on entry 0
  return GCCNMF_OK;
}

int lld_load_dictionary(gccnmf_handle* h, const gccnmf_ll_config* cfg, int P, int Lh, int Qd, int Qe, void* state, size_t state_bytes, int index,
                        const float* W, int K, const float* H0, void* stream) {
  GCCNMF_ENTER(h);
  GCCNMF_REQUIRE(h, Qd >= 1, "lldict: num_dictionaries must be in [1, %d] (got %d)", kLLMaxDictionaries, Qd);
  LLD_CARVE_OR_FAIL(l, P, Lh, Qe, Qd);
  if (int st = lld_check_entry(h, cfg, l, index, W, K, H0)) return st;
  return lld_load_entry(h, cfg, l, index, W, K, H0, stream);
}

// streams [first, first + count) onto dictionary_host[i] / steering_host[i] (-1 or a NULL array: keep), then both sorts; stream-ordered
int lld_assign(gccnmf_handle* h, const gccnmf_ll_config* cfg, int P, int Lh, int Qd, int Qe, void* state, size_t state_bytes, int first, int count,
               const int32_t* dictionary_host, const int32_t* steering_host, void* stream) {
  GCCNMF_ENTER(h);
  GCCNMF_REQUIRE(h, Qd >= 1, "lldict: num_dictionaries must be in [1, %d] (got %d)", kLLMaxDictionaries, Qd);
  LLD_CARVE_OR_FAIL(l, P, Lh, Qe, Qd);
  if (int st = stream_range_check(h, "lldict_assign", l.S, first, count)) return st;
  for (int i = 0; i < count; ++i) {
    const int d = dictionary_host ? dictionary_host[i] : -1, e = steering_host ? steering_host[i] : -1;
    GCCNMF_REQUIRE(h, d >= -1 && d < Qd, "lldict_assign: stream %d: dictionary entry %d outside [0, %d) (or -1)", first + i, d, Qd);
    GCCNMF_REQUIRE(h, e >= -1 && e < Qe, "lldict_assign: stream %d: steering entry %d outside [0, %d) (or -1)", first + i, e, Qe);
  }
  for (int pass = 0; pass < 2; ++pass) {
    const int32_t* src = pass ? steering_host : dictionary_host;
    if (!src) continue;
    if (int st = enqueue_stream_rows(h, pass ? l.assign : l.dassign, sizeof(int32_t), 0, first, count, 1, src, true, stream)) return st;
    if (pass) GCCNMF_LAUNCH(h, sort_by_entry_kernel, 1, 32, 0, stream, l.assign, sizeof(int32_t), l.S, Qe, l.order, l.seg);
    else GCCNMF_LAUNCH(h, sort_by_entry_kernel, 1, 32, 0, stream, l.dassign, sizeof(int32_t), l.S, Qd, l.dorder, l.dseg);
  }
  return GCCNMF_OK;
}

}  // namespace

extern "C" {

size_t gccnmf_ll_state_bytes(const gccnmf_ll_config* cfg) {
  if (ll_check(nullptr, cfg, 0) != 0) return 0;
  return ll_carve(*cfg, 0, nullptr).bytes;
}

int gccnmf_ll_init(gccnmf_handle* h, const gccnmf_ll_config* cfg, const float* W, const double* E, const double* analysis_window,
                   const double* synthesis_weights, float gain, const float* H0, void* state, size_t state_bytes, void* stream) {
  return ll_init(h, cfg, 0, 0, 0, 0, W, E, analysis_window, synthesis_weights, gain, H0, state, state_bytes, stream);
}

int gccnmf_ll_reset_streams(gccnmf_handle* h, const gccnmf_ll_config* cfg, void* state, size_t state_bytes, int first, int count, void* stream) {
  return ll_reset_streams(h, cfg, 0, 0, 0, 0, state, state_bytes, first, count, stream);
}

int gccnmf_ll_set_params(gccnmf_handle* h, const gccnmf_ll_config* cfg, void* state, size_t state_bytes, int first, int count,
                         const gccnmf_ll_stream_params* params_host, void* stream) {
  return ll_set_params(h, cfg, 0, 0, 0, 0, state, state_bytes, first, count, params_host, stream);
}

int gccnmf_ll_process(gccnmf_handle* h, const gccnmf_ll_config* cfg, void* state, size_t state_bytes, int hops, const float* in, float* out,
                      void* stream) {
  GCCNMF_ENTER(h);
  LL_CARVE_OR_FAIL(l, 0, 0, 0);
  return ll_enqueue(h, cfg, l, hops, in, out, stream);
}

int gccnmf_ll_graph_create(gccnmf_handle* h, const gccnmf_ll_config* cfg, void* state, size_t state_bytes, int hops, float* in, float* out,
                           const float* in_host, float* out_host, void** graph_exec, void* stream) {
  return ll_graph_create(h, cfg, 0, 0, 0, 0, state, state_bytes, hops, in, out, in_host, out_host, graph_exec, stream);
}

int gccnmf_ll_export(gccnmf_handle* h, const gccnmf_ll_config* cfg, void* state, size_t state_bytes, int hops, int what, void* dst, void* stream) {
  return ll_export(h, cfg, 0, 0, 0, 0, state, state_bytes, hops, what, dst, stream);
}

// ---- sources (2 <= num_sources <= 8)
size_t gccnmf_llsep_state_bytes(const gccnmf_ll_config* cfg, int num_sources) {
  if (num_sources == 0 || ll_check(nullptr, cfg, num_sources) != 0) return 0;
  return ll_carve(*cfg, num_sources, nullptr).bytes;
}

int gccnmf_llsep_init(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, const float* W, const double* E,
                      const double* analysis_window, const double* synthesis_weights, float gain, const float* H0, void* state,
                      size_t state_bytes, void* stream) {
  GCCNMF_REQUIRE(h, num_sources != 0, "llsep: num_sources must be in [2, %d] (got 0)", kLLMaxSources);
  return ll_init(h, cfg, num_sources, 0, 0, 0, W, E, analysis_window, synthesis_weights, gain, H0, state, state_bytes, stream);
}

int gccnmf_llsep_reset_streams(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, void* state, size_t state_bytes, int first,
                               int count, void* stream) {
  GCCNMF_REQUIRE(h, num_sources != 0, "llsep: num_sources must be in [2, %d] (got 0)", kLLMaxSources);
  return ll_reset_streams(h, cfg, num_sources, 0, 0, 0, state, state_bytes, first, count, stream);
}

int gccnmf_llsep_set_params(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, void* state, size_t state_bytes, int first,
                            int count, const gccnmf_ll_stream_params* params_host, void* stream) {
  GCCNMF_REQUIRE(h, num_sources != 0, "llsep: num_sources must be in [2, %d] (got 0)", kLLMaxSources);
  return ll_set_params(h, cfg, num_sources, 0, 0, 0, state, state_bytes, first, count, params_host, stream);
}

int gccnmf_llsep_set_targets(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, void* state, size_t state_bytes, int first,
                             int count, const int32_t* targets_host, void* stream) {
  GCCNMF_REQUIRE(h, num_sources != 0, "llsep: num_sources must be in [2, %d] (got 0)", kLLMaxSources);
  return ll_set_targets(h, cfg, num_sources, 0, 0, 0, state, state_bytes, first, count, targets_host, stream);
}

int gccnmf_llsep_process(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, void* state, size_t state_bytes, int hops,
                         const float* in, float* out, void* stream) {
  GCCNMF_ENTER(h);
  GCCNMF_REQUIRE(h, num_sources != 0, "llsep: num_sources must be in [2, %d] (got 0)", kLLMaxSources);
  LL_CARVE_OR_FAIL(l, num_sources, 0, 0);
  return ll_enqueue(h, cfg, l, hops, in, out, stream);
}

int gccnmf_llsep_graph_create(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, void* state, size_t state_bytes, int hops,
                              float* in, float* out, const float* in_host, float* out_host, void** graph_exec, void* stream) {
  GCCNMF_REQUIRE(h, num_sources != 0, "llsep: num_sources must be in [2, %d] (got 0)", kLLMaxSources);
  return ll_graph_create(h, cfg, num_sources, 0, 0, 0, state, state_bytes, hops, in, out, in_host, out_host, graph_exec, stream);
}

int gccnmf_llsep_export(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, void* state, size_t state_bytes, int hops, int what,
                        void* dst, void* stream) {
  GCCNMF_REQUIRE(h, num_sources != 0, "llsep: num_sources must be in [2, %d] (got 0)", kLLMaxSources);
  return ll_export(h, cfg, num_sources, 0, 0, 0, state, state_bytes, hops, what, dst, stream);
}

// ---- stream records (0 <= num_sources <= 8)
size_t gccnmf_llrec_record_bytes(const gccnmf_ll_config* cfg, int num_sources) {
  if (ll_check(nullptr, cfg, num_sources) != 0) return 0;
  return ll_record_bytes(*cfg, num_sources);
}

size_t gccnmf_llrec_workspace_bytes(const gccnmf_ll_config* cfg, int num_sources, int count) {
  if (ll_check(nullptr, cfg, num_sources) != 0 || count < 1) return 0;
  return ll_record_work(*cfg, num_sources, 0, 0, 0, count).bytes;
}

int gccnmf_llrec_save_streams(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, void* state, size_t state_bytes, int first,
                              int count, void* record, size_t record_bytes, void* workspace, size_t workspace_bytes, void* stream) {
  return ll_save_streams(h, cfg, num_sources, 0, 0, 0, state, state_bytes, first, count, record, record_bytes, workspace, workspace_bytes, stream);
}

int gccnmf_llrec_load_streams(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, void* state, size_t state_bytes, int first,
                              int count, const void* record, size_t record_bytes, void* workspace, size_t workspace_bytes, void* stream) {
  return ll_load_streams(h, cfg, num_sources, 0, 0, 0, state, state_bytes, first, count, record, record_bytes, workspace, workspace_bytes, stream);
}

// ---- history (0 <= num_sources <= 8, 0 <= history_length <= 1024)
size_t gccnmf_llhist_state_bytes(const gccnmf_ll_config* cfg, int num_sources, int history_length) {
  if (ll_check(nullptr, cfg, num_sources, history_length) != 0) return 0;
  return ll_carve(*cfg, num_sources, nullptr, history_length).bytes;
}

int gccnmf_llhist_init(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, const float* W, const double* E,
                       const double* analysis_window, const double* synthesis_weights, float gain, const float* H0, void* state,
                       size_t state_bytes, void* stream) {
  return ll_init(h, cfg, num_sources, history_length, 0, 0, W, E, analysis_window, synthesis_weights, gain, H0, state, state_bytes, stream);
}

int gccnmf_llhist_reset_streams(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, void* state,
                                size_t state_bytes, int first, int count, void* stream) {
  return ll_reset_streams(h, cfg, num_sources, history_length, 0, 0, state, state_bytes, first, count, stream);
}

int gccnmf_llhist_set_params(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, void* state,
                             size_t state_bytes, int first, int count, const gccnmf_ll_stream_params* params_host, void* stream) {
  return ll_set_params(h, cfg, num_sources, history_length, 0, 0, state, state_bytes, first, count, params_host, stream);
}

int gccnmf_llhist_set_targets(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, void* state,
                              size_t state_bytes, int first, int count, const int32_t* targets_host, void* stream) {
  GCCNMF_REQUIRE(h, num_sources != 0, "llhist_set_targets: needs num_sources in [2, %d] (got 0)", kLLMaxSources);
  return ll_set_targets(h, cfg, num_sources, history_length, 0, 0, state, state_bytes, first, count, targets_host, stream);
}

int gccnmf_llhist_set_window(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, void* state,
                             size_t state_bytes, int first, int count, const int32_t* windows_host, void* stream) {
  return ll_set_window(h, cfg, num_sources, history_length, 0, 0, state, state_bytes, first, count, windows_host, stream);
}

int gccnmf_llhist_process(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, void* state, size_t state_bytes,
                          int hops, const float* in, float* out, void* stream) {
  GCCNMF_ENTER(h);
  LL_CARVE_OR_FAIL(l, num_sources, history_length, 0);
  return ll_enqueue(h, cfg, l, hops, in, out, stream);
}

int gccnmf_llhist_graph_create(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, void* state,
                               size_t state_bytes, int hops, float* in, float* out, const float* in_host, float* out_host, void** graph_exec,
                               void* stream) {
  return ll_graph_create(h, cfg, num_sources, history_length, 0, 0, state, state_bytes, hops, in, out, in_host, out_host, graph_exec, stream);
}

int gccnmf_llhist_export(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, void* state, size_t state_bytes,
                         int hops, int what, void* dst, void* stream) {
  return ll_export(h, cfg, num_sources, history_length, 0, 0, state, state_bytes, hops, what, dst, stream);
}

size_t gccnmf_llhist_record_bytes(const gccnmf_ll_config* cfg, int num_sources, int history_length) {
  if (ll_check(nullptr, cfg, num_sources, history_length) != 0) return 0;
  return ll_record_bytes(*cfg, num_sources, history_length);
}

size_t gccnmf_llhist_workspace_bytes(const gccnmf_ll_config* cfg, int num_sources, int history_length, int count) {
  if (ll_check(nullptr, cfg, num_sources, history_length) != 0 || count < 1) return 0;
  return ll_record_work(*cfg, num_sources, history_length, 0, 0, count).bytes;
}

int gccnmf_llhist_save_streams(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, void* state,
                               size_t state_bytes, int first, int count, void* record, size_t record_bytes, void* workspace,
                               size_t workspace_bytes, void* stream) {
  return ll_save_streams(h, cfg, num_sources, history_length, 0, 0, state, state_bytes, first, count, record, record_bytes, workspace, workspace_bytes,
                         stream);
}

int gccnmf_llhist_load_streams(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, void* state,
                               size_t state_bytes, int first, int count, const void* record, size_t record_bytes, void* workspace,
                               size_t workspace_bytes, void* stream) {
  return ll_load_streams(h, cfg, num_sources, history_length, 0, 0, state, state_bytes, first, count, record, record_bytes, workspace, workspace_bytes,
                         stream);
}

// ---- steering bank (0 <= num_sources <= 8, 0 <= history_length <= 1024, 0 <= num_steerings <= 64)
size_t gccnmf_llbank_state_bytes(const gccnmf_ll_config* cfg, int num_sources, int history_length, int num_steerings) {
  if (ll_check(nullptr, cfg, num_sources, history_length, num_steerings) != 0) return 0;
  return ll_carve(*cfg, num_sources, nullptr, history_length, num_steerings).bytes;
}

int gccnmf_llbank_init(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, int num_steerings, const float* W,
                       const double* E, const double* analysis_window, const double* synthesis_weights, float gain, const float* H0, void* state,
                       size_t state_bytes, void* stream) {
  return ll_init(h, cfg, num_sources, history_length, num_steerings, 0, W, E, analysis_window, synthesis_weights, gain, H0, state, state_bytes, stream);
}

int gccnmf_llbank_load_steering(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, int num_steerings, void* state,
                                size_t state_bytes, int entry, const double* E, void* stream) {
  return ll_load_steering(h, cfg, num_sources, history_length, num_steerings, 0, state, state_bytes, entry, E, stream);
}

int gccnmf_llbank_assign(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, int num_steerings, void* state,
                         size_t state_bytes, int first, int count, const int32_t* entries_host, void* stream) {
  return ll_assign(h, cfg, num_sources, history_length, num_steerings, 0, state, state_bytes, first, count, entries_host, stream);
}

int gccnmf_llbank_reset_streams(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, int num_steerings, void* state,
                                size_t state_bytes, int first, int count, void* stream) {
  return ll_reset_streams(h, cfg, num_sources, history_length, num_steerings, 0, state, state_bytes, first, count, stream);
}

int gccnmf_llbank_set_params(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, int num_steerings, void* state,
                             size_t state_bytes, int first, int count, const gccnmf_ll_stream_params* params_host, void* stream) {
  return ll_set_params(h, cfg, num_sources, history_length, num_steerings, 0, state, state_bytes, first, count, params_host, stream);
}

int gccnmf_llbank_set_targets(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, int num_steerings, void* state,
                              size_t state_bytes, int first, int count, const int32_t* targets_host, void* stream) {
  GCCNMF_REQUIRE(h, num_sources != 0, "llbank_set_targets: needs num_sources in [2, %d] (got 0)", kLLMaxSources);
  return ll_set_targets(h, cfg, num_sources, history_length, num_steerings, 0, state, state_bytes, first, count, targets_host, stream);
}

int gccnmf_llbank_set_window(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, int num_steerings, void* state,
                             size_t state_bytes, int first, int count, const int32_t* windows_host, void* stream) {
  return ll_set_window(h, cfg, num_sources, history_length, num_steerings, 0, state, state_bytes, first, count, windows_host, stream);
}

int gccnmf_llbank_process(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, int num_steerings, void* state,
                          size_t state_bytes, int hops, const float* in, float* out, void* stream) {
  GCCNMF_ENTER(h);
  LL_CARVE_OR_FAIL(l, num_sources, history_length, num_steerings);
  return ll_enqueue(h, cfg, l, hops, in, out, stream);
}

int gccnmf_llbank_graph_create(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, int num_steerings, void* state,
                               size_t state_bytes, int hops, float* in, float* out, const float* in_host, float* out_host, void** graph_exec,
                               void* stream) {
  return ll_graph_create(h, cfg, num_sources, history_length, num_steerings, 0, state, state_bytes, hops, in, out, in_host, out_host, graph_exec, stream);
}

int gccnmf_llbank_export(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, int num_steerings, void* state,
                         size_t state_bytes, int hops, int what, void* dst, void* stream) {
  return ll_export(h, cfg, num_sources, history_length, num_steerings, 0, state, state_bytes, hops, what, dst, stream);
}

size_t gccnmf_llbank_record_bytes(const gccnmf_ll_config* cfg, int num_sources, int history_length, int num_steerings) {
  if (ll_check(nullptr, cfg, num_sources, history_length, num_steerings) != 0) return 0;
  return ll_record_bytes(*cfg, num_sources, history_length);
}

size_t gccnmf_llbank_workspace_bytes(const gccnmf_ll_config* cfg, int num_sources, int history_length, int num_steerings, int count) {
  if (ll_check(nullptr, cfg, num_sources, history_length, num_steerings) != 0 || count < 1) return 0;
  return ll_record_work(*cfg, num_sources, history_length, num_steerings, 0, count).bytes;
}

int gccnmf_llbank_save_streams(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, int num_steerings, void* state,
                               size_t state_bytes, int first, int count, void* record, size_t record_bytes, void* workspace, size_t workspace_bytes,
                               void* stream) {
  return ll_save_streams(h, cfg, num_sources, history_length, num_steerings, 0, state, state_bytes, first, count, record, record_bytes, workspace,
                         workspace_bytes, stream);
}

int gccnmf_llbank_load_streams(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, int num_steerings, void* state,
                               size_t state_bytes, int first, int count, const void* record, size_t record_bytes, void* workspace,
                               size_t workspace_bytes, void* stream) {
  return ll_load_streams(h, cfg, num_sources, history_length, num_steerings, 0, state, state_bytes, first, count, record, record_bytes, workspace,
                         workspace_bytes, stream);
}

// ---- dictionary bank (0 <= num_sources <= 8, 0 <= history_length <= 1024, 1 <= num_dictionaries <= 64, 1 <= num_steerings <= 64)
#define LLD_ARGS cfg, num_sources, history_length, num_steerings, num_dictionaries
size_t gccnmf_lldict_state_bytes(const gccnmf_ll_config* cfg, int num_sources, int history_length, int num_dictionaries, int num_steerings) {
  if (num_dictionaries < 1 || ll_check(nullptr, LLD_ARGS) != 0) return 0;
  return ll_carve(*cfg, num_sources, nullptr, history_length, num_steerings, num_dictionaries).bytes;
}

int gccnmf_lldict_init(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, int num_dictionaries, int num_steerings,
                       const float* const* W, const int* num_atoms, const float* const* H0, const double* E, const double* analysis_window,
                       const double* synthesis_weights, float gain, void* state, size_t state_bytes, void* stream) {
  return lld_init(h, cfg, num_sources, history_length, num_dictionaries, num_steerings, W, num_atoms, E, analysis_window, synthesis_weights, gain, H0,
                  state, state_bytes, stream);
}

int gccnmf_lldict_load_dictionary(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, int num_dictionaries,
                                  int num_steerings, void* state, size_t state_bytes, int index, const float* W, int num_atoms, const float* H0,
                                  void* stream) {
  return lld_load_dictionary(h, cfg, num_sources, history_length, num_dictionaries, num_steerings, state, state_bytes, index, W, num_atoms, H0, stream);
}

int gccnmf_lldict_load_steering(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, int num_dictionaries,
                                int num_steerings, void* state, size_t state_bytes, int index, const double* E, void* stream) {
  GCCNMF_REQUIRE(h, num_dictionaries >= 1, "lldict: num_dictionaries must be in [1, %d] (got %d)", kLLMaxDictionaries, num_dictionaries);
  return ll_load_steering(h, LLD_ARGS, state, state_bytes, index, E, stream);
}

int gccnmf_lldict_assign(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, int num_dictionaries, int num_steerings,
                         void* state, size_t state_bytes, int first, int count, const int32_t* dictionary_host, const int32_t* steering_host,
                         void* stream) {
  return lld_assign(h, cfg, num_sources, history_length, num_dictionaries, num_steerings, state, state_bytes, first, count, dictionary_host,
                    steering_host, stream);
}

int gccnmf_lldict_reset_streams(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, int num_dictionaries,
                                int num_steerings, void* state, size_t state_bytes, int first, int count, void* stream) {
  GCCNMF_REQUIRE(h, num_dictionaries >= 1, "lldict: num_dictionaries must be in [1, %d] (got %d)", kLLMaxDictionaries, num_dictionaries);
  return ll_reset_streams(h, LLD_ARGS, state, state_bytes, first, count, stream);
}

int gccnmf_lldict_set_params(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, int num_dictionaries,
                             int num_steerings, void* state, size_t state_bytes, int first, int count, const gccnmf_ll_stream_params* params_host,
                             void* stream) {
  GCCNMF_REQUIRE(h, num_dictionaries >= 1, "lldict: num_dictionaries must be in [1, %d] (got %d)", kLLMaxDictionaries, num_dictionaries);
  return ll_set_params(h, LLD_ARGS, state, state_bytes, first, count, params_host, stream);
}

int gccnmf_lldict_set_targets(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, int num_dictionaries,
                              int num_steerings, void* state, size_t state_bytes, int first, int count, const int32_t* targets_host, void* stream) {
  GCCNMF_REQUIRE(h, num_dictionaries >= 1, "lldict: num_dictionaries must be in [1, %d] (got %d)", kLLMaxDictionaries, num_dictionaries);
  GCCNMF_REQUIRE(h, num_sources != 0, "lldict_set_targets: needs num_sources in [2, %d] (got 0)", kLLMaxSources);
  return ll_set_targets(h, LLD_ARGS, state, state_bytes, first, count, targets_host, stream);
}

int gccnmf_lldict_set_window(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, int num_dictionaries,
                             int num_steerings, void* state, size_t state_bytes, int first, int count, const int32_t* windows_host, void* stream) {
  GCCNMF_REQUIRE(h, num_dictionaries >= 1, "lldict: num_dictionaries must be in [1, %d] (got %d)", kLLMaxDictionaries, num_dictionaries);
  return ll_set_window(h, LLD_ARGS, state, state_bytes, first, count, windows_host, stream);
}

int gccnmf_lldict_process(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, int num_dictionaries, int num_steerings,
                          void* state, size_t state_bytes, int hops, const float* in, float* out, void* stream) {
  GCCNMF_ENTER(h);
  GCCNMF_REQUIRE(h, num_dictionaries >= 1, "lldict: num_dictionaries must be in [1, %d] (got %d)", kLLMaxDictionaries, num_dictionaries);
  LLD_CARVE_OR_FAIL(l, num_sources, history_length, num_steerings, num_dictionaries);
  return ll_enqueue(h, cfg, l, hops, in, out, stream);
}

int gccnmf_lldict_graph_create(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, int num_dictionaries,
                               int num_steerings, void* state, size_t state_bytes, int hops, float* in, float* out, const float* in_host,
                               float* out_host, void** graph_exec, void* stream) {
  GCCNMF_REQUIRE(h, num_dictionaries >= 1, "lldict: num_dictionaries must be in [1, %d] (got %d)", kLLMaxDictionaries, num_dictionaries);
  return ll_graph_create(h, LLD_ARGS, state, state_bytes, hops, in, out, in_host, out_host, graph_exec, stream);
}

int gccnmf_lldict_export(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, int num_dictionaries, int num_steerings,
                         void* state, size_t state_bytes, int hops, int what, void* dst, void* stream) {
  GCCNMF_REQUIRE(h, num_dictionaries >= 1, "lldict: num_dictionaries must be in [1, %d] (got %d)", kLLMaxDictionaries, num_dictionaries);
  return ll_export(h, LLD_ARGS, state, state_bytes, hops, what, dst, stream);
}

size_t gccnmf_lldict_record_bytes(const gccnmf_ll_config* cfg, int num_sources, int history_length, int num_dictionaries, int num_steerings) {
  if (num_dictionaries < 1 || ll_check(nullptr, LLD_ARGS) != 0) return 0;
  return ll_record_bytes(*cfg, num_sources, history_length);
}

size_t gccnmf_lldict_workspace_bytes(const gccnmf_ll_config* cfg, int num_sources, int history_length, int num_dictionaries, int num_steerings,
                                     int count) {
  if (num_dictionaries < 1 || ll_check(nullptr, LLD_ARGS) != 0 || count < 1) return 0;
  return ll_record_work(*cfg, num_sources, history_length, num_steerings, num_dictionaries, count).bytes;
}

int gccnmf_lldict_save_streams(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, int num_dictionaries,
                               int num_steerings, void* state, size_t state_bytes, int first, int count, void* record, size_t record_bytes,
                               void* workspace, size_t workspace_bytes, void* stream) {
  GCCNMF_REQUIRE(h, num_dictionaries >= 1, "lldict: num_dictionaries must be in [1, %d] (got %d)", kLLMaxDictionaries, num_dictionaries);
  return ll_save_streams(h, LLD_ARGS, state, state_bytes, first, count, record, record_bytes, workspace, workspace_bytes, stream);
}

int gccnmf_lldict_load_streams(gccnmf_handle* h, const gccnmf_ll_config* cfg, int num_sources, int history_length, int num_dictionaries,
                               int num_steerings, void* state, size_t state_bytes, int first, int count, const void* record, size_t record_bytes,
                               void* workspace, size_t workspace_bytes, void* stream) {
  GCCNMF_REQUIRE(h, num_dictionaries >= 1, "lldict: num_dictionaries must be in [1, %d] (got %d)", kLLMaxDictionaries, num_dictionaries);
  return ll_load_streams(h, LLD_ARGS, state, state_bytes, first, count, record, record_bytes, workspace, workspace_bytes, stream);
}
#undef LLD_ARGS

}  // extern "C"
