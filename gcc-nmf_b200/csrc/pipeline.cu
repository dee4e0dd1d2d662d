// The whole offline hot path as ONE C-ABI call with no host synchronisation inside (SURVEY.md section 8b, "fused gccnmf_separate"):
//   separation   gccNMF/runGCCNMF.py:36-52          STFT -> |X| -> KL-NMF -> PHAT coherence -> angular spectrogram -> peak picking ->
//                                                   per-target GCC-NMF -> one-hot masks -> masked reconstruction -> iSTFT
//   enhancement  notebooks/offlineSpeechEnhancement.ipynb cells 12-41 (:444-472): one target, argmax over ALL hypothesis TDOAs,
//                                                   mask = within target_window seconds of the target's TDOA
// The reference picks the target TDOAs on the host (scipy.signal.argrelmax on the D-element mean angular spectrum, gccNMFFunctions.py:94-116);
// here that decision is taken by a one-CTA kernel so that the stages after it can be enqueued without waiting for it: the target
// indexes, the gathered steering columns and the TDOA look-up table stay on the device.  Conditions the reference turns into Python
// exceptions are reported through a device-side status word the caller reads after the call (bit 0: fewer peaks than targets,
// bit 1: an all-NaN mask column, bit 2: more near-tie argmax decisions than the float64 refinement list holds).
// gccnmf_separate_tracked is the same flow with targets per frame (tracking.cu) in place of the one pick over the whole clip.
#include <cmath>

#include "common.cuh"

namespace {

constexpr int kPickMaxD = 1024;

// The numSources largest strict local maxima of the mean angular spectrum (select_peaks), ascending; missing ones are 0.
__global__ void pick_targets_kernel(const double* __restrict__ mean_angular, int D, int S, int32_t* __restrict__ targets, int32_t* __restrict__ status) {
  __shared__ double x[kPickMaxD];
  __shared__ unsigned char peak[kPickMaxD], chosen[kPickMaxD];
  __shared__ int num_peaks;
  for (int d = threadIdx.x; d < D; d += blockDim.x) x[d] = mean_angular[d];
  const int peaks = select_peaks(x, D, S, peak, chosen, &num_peaks, targets);
  if (threadIdx.x == 0) {
    for (int i = peaks < S ? peaks : S; i < S; ++i) targets[i] = 0;
    if (peaks < S) atomicOr(status, 1);              // the reference aborts here (:102-104)
  }
}

// E_sel[f][s] = E[f][targets[s]]   (the rotation of gccNMFFunctions.py:128-131 for the chosen TDOAs)
__global__ void gather_steering_kernel(const double2* __restrict__ E, int F, int D, const int32_t* __restrict__ targets, int S, double2* __restrict__ E_sel) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= F * S) return;
  const int f = i / S, s = i - f * S;
  E_sel[i] = E[(int64_t)f * D + targets[s]];
}

// lut[d] = |tdoa[d] - tdoa[target]| < window   (offlineSpeechEnhancement.ipynb:468-471, float64)
__global__ void tdoa_lut_kernel(const double* __restrict__ tdoas, int D, const int32_t* __restrict__ target, double window, uint8_t* __restrict__ lut) {
  const int d = blockIdx.x * blockDim.x + threadIdx.x;
  if (d < D) lut[d] = fabs(tdoas[d] - tdoas[target[0]]) < window ? 1 : 0;
}

__global__ void or_status_kernel(const int32_t* __restrict__ flag, int32_t threshold, int32_t bit, int32_t* __restrict__ status) {
  if (flag[0] > threshold) atomicOr(status, bit);
}

struct PipeLayout {
  float *X, *V, *coh, *values, *masks, *est;
  double *mean, *E_sel;
  int32_t *argmax, *flags;
  uint8_t* lut;
  double *angular, *means;       // tracked flow only: the angular spectrogram and its window means (D, T)
  uint8_t* table;                // tracked enhancement: the (D, D) TDOA table
  void *ws_nmf, *ws_ang, *ws_argmax, *ws_recon, *ws_istft;
  size_t n_nmf, n_ang, n_argmax, n_recon, n_istft, bytes;
  int F, T;
  bool ok;
};

// tracked: the gccnmf_separate_tracked layout, the gccnmf_separate one followed by its own buffers.
PipeLayout pipe_carve(const gccnmf_pipeline_config& c, int64_t num_samples, void* ws, size_t ws_bytes, bool tracked = false) {
  PipeLayout l{};
  const int N = c.window_size, K = c.num_atoms, D = c.num_tdoas;
  const int S = c.num_targets > 0 ? c.num_targets : 1;
  l.F = N / 2 + 1;
  l.T = gccnmf_stft_num_frames(num_samples, N, c.hop_size);
  if (l.T < 1) { l.ok = false; return l; }
  const size_t F = l.F, T = l.T;
  WorkspaceCarver w(ws ? ws : reinterpret_cast<void*>(256), ws ? ws_bytes : ~size_t(0) >> 1);
  l.mean = w.take<double>(D);
  l.E_sel = w.take<double>(2 * F * S);
  l.X = w.take<float>(2 * 2 * F * T);
  l.V = w.take<float>(F * 2 * T);
  l.coh = w.take<float>(2 * F * T);
  l.values = w.take<float>(c.num_targets > 0 ? (size_t)S * K * T : 1);
  l.masks = w.take<float>((size_t)S * K * T);
  l.est = w.take<float>((size_t)S * 2 * 2 * F * T);
  l.argmax = w.take<int32_t>(c.num_targets > 0 ? 1 : (size_t)K * T);
  l.flags = w.take<int32_t>(8);
  l.lut = w.take<uint8_t>(D);
  l.n_nmf = gccnmf_klnmf_workspace_bytes(l.F, 2 * l.T, K);
  l.n_ang = gccnmf_phat_angspec_workspace_bytes(l.F, l.T, D);
  l.n_argmax = c.num_targets > 0 ? 256 : gccnmf_tdoa_argmax_workspace_bytes(l.F, l.T, D, K);
  l.n_recon = gccnmf_masked_recon_workspace_bytes(S, l.F, l.T, K);
  l.n_istft = gccnmf_istft_workspace_bytes(S * 2, N, l.T);
  l.ws_nmf = w.take<char>(l.n_nmf);
  l.ws_ang = w.take<char>(l.n_ang);
  l.ws_argmax = w.take<char>(l.n_argmax);
  l.ws_recon = w.take<char>(l.n_recon);
  l.ws_istft = w.take<char>(l.n_istft);
  if (tracked) {
    l.angular = w.take<double>((size_t)D * T);
    l.means = w.take<double>((size_t)D * T);
    l.table = w.take<uint8_t>((size_t)D * D);
  }
  l.bytes = align_up(w.used, 256);
  l.ok = ws != nullptr && w.ok();
  return l;
}

}  // namespace

extern "C" {

size_t gccnmf_pipeline_workspace_bytes(const gccnmf_pipeline_config* cfg, int64_t num_samples) {
  if (!cfg || cfg->window_size < 2 || cfg->hop_size < 1 || cfg->num_atoms < 1 || cfg->num_tdoas < 1) return 0;
  const PipeLayout l = pipe_carve(*cfg, num_samples, nullptr, 0);
  return l.T >= 1 ? l.bytes : 0;
}

// Standalone peak picking (the host drop-in calls scipy like the reference; this is what the fused path uses).
int gccnmf_pick_targets(gccnmf_handle* h, const double* mean_angular, int D, int num_targets, int32_t* targets, int32_t* status, void* stream) {
  GCCNMF_ENTER(h);
  GCCNMF_REQUIRE(h, mean_angular && targets && status && D >= 3 && D <= kPickMaxD && num_targets >= 1 && num_targets <= D, "pick_targets: bad arguments");
  GCCNMF_LAUNCH(h, pick_targets_kernel, 1, 128, 0, stream, mean_angular, D, num_targets, targets, status);
  return GCCNMF_OK;
}

// samples (2, n) f32; window (N) f64 (numpy.hanning); E (F, D) complex128 steering table; tdoas (D) f64; W (F, K) / H (K, 2T) f32:
// in = the seeded initial values (gccNMFFunctions.py:70-73), out = the learnt dictionary / coefficients; signals (S, 2, L) f32 with
// L = gccnmf_istft_length(N, hop, T, 1) and S = num_targets (or 1 for the enhancement flow, num_targets == 0);
// target_indexes (S) i32 and status (1) i32 are DEVICE outputs (status bits: see the header of this file).
int gccnmf_separate(gccnmf_handle* h, const gccnmf_pipeline_config* cfg, const float* samples, int64_t num_samples, const double* window,
                    const double* E, const double* tdoas, float* W, float* H, float* signals, int32_t* target_indexes, int32_t* status,
                    void* workspace, size_t workspace_bytes, void* stream) {
  GCCNMF_ENTER(h);
  GCCNMF_REQUIRE(h, cfg && samples && window && E && tdoas && W && H && signals && target_indexes && status, "separate: NULL pointer");
  GCCNMF_REQUIRE(h, cfg->num_targets >= 0 && cfg->num_iterations >= 0 && cfg->num_tdoas >= 3 && cfg->num_tdoas <= kPickMaxD, "separate: bad configuration");
  PipeLayout l = pipe_carve(*cfg, num_samples, workspace, workspace_bytes);
  GCCNMF_REQUIRE(h, l.T >= 1, "Buffer is too short (n=%lld) for frame_length=%d", (long long)num_samples, cfg->window_size);
  if (!l.ok) return gccnmf_fail(h, GCCNMF_ERR_WORKSPACE, "separate: workspace too small: need %zu bytes", l.bytes);
  const int N = cfg->window_size, hop = cfg->hop_size, K = cfg->num_atoms, D = cfg->num_tdoas, F = l.F, T = l.T;
  const bool enhancement = cfg->num_targets == 0;
  const int S = enhancement ? 1 : cfg->num_targets;
  cudaStream_t s = (cudaStream_t)stream;
  GCCNMF_CHECK_CUDA(h, cudaMemsetAsync(status, 0, sizeof(int32_t), s));
  GCCNMF_CHECK_CUDA(h, cudaMemsetAsync(l.flags, 0, 8 * sizeof(int32_t), s));
  // a1 + the |X| of runGCCNMF.py:40
  if (int st = gccnmf_stft(h, samples, num_samples, 2, num_samples, window, N, hop, 1, l.X, l.V, stream)) return st;
  // a3 + a4 (+ the mean over frames of runGCCNMF.py:46) and a5 on the device
  if (int st = gccnmf_phat_angspec(h, l.X, F, T, 0, E, D, l.coh, nullptr, l.mean, l.ws_ang, l.n_ang, stream)) return st;
  GCCNMF_LAUNCH(h, pick_targets_kernel, 1, 128, 0, stream, l.mean, D, S, target_indexes, status);
  // a2
  if (int st = gccnmf_klnmf(h, l.V, F, 2 * T, W, H, K, cfg->num_iterations, cfg->sparsity_alpha, cfg->epsilon, 1, l.ws_nmf, l.n_nmf, stream)) return st;
  if (enhancement) {
    // a10: argmax over all TDOAs, mask = TDOAs within the window of the target's
    if (int st = gccnmf_tdoa_argmax(h, l.coh, F, T, E, D, W, K, l.argmax, l.flags + 1, l.ws_argmax, l.n_argmax, stream)) return st;
    GCCNMF_LAUNCH(h, or_status_kernel, 1, 1, 0, stream, l.flags + 1, gccnmf_tdoa_argmax_refine_capacity(K, T), 4, status);
    GCCNMF_LAUNCH(h, tdoa_lut_kernel, (D + 127) / 128, 128, 0, stream, tdoas, D, target_indexes, (double)cfg->target_window_seconds, l.lut);
    if (int st = gccnmf_argmax_mask(h, l.argmax, K, T, l.lut, D, l.masks, stream)) return st;
  } else {
    // a6 + a7: per-target GCC-NMF at the chosen TDOAs, one-hot masks
    GCCNMF_LAUNCH(h, gather_steering_kernel, (F * S + 255) / 256, 256, 0, stream, reinterpret_cast<const double2*>(E), F, D, target_indexes, S,
                  reinterpret_cast<double2*>(l.E_sel));
    if (int st = gccnmf_tdoa_gccnmf(h, l.coh, F, T, l.E_sel, S, W, K, l.values, nullptr, stream)) return st;
    if (int st = gccnmf_coeff_mask(h, l.values, S, K, T, l.masks, l.flags + 2, stream)) return st;
    GCCNMF_LAUNCH(h, or_status_kernel, 1, 1, 0, stream, l.flags + 2, 0, 2, status);
  }
  // a8 + a9
  if (int st = gccnmf_masked_recon_phase(h, l.masks, l.X, W, H, S, F, T, K, l.est, l.ws_recon, l.n_recon, stream)) return st;
  return gccnmf_istft_ola(h, l.est, S * 2, N, hop, T, window, (float)((double)hop / (double)N * 2.0), 1, 1, signals, l.ws_istft, l.n_istft, stream);
}

size_t gccnmf_pipeline_tracked_workspace_bytes(const gccnmf_pipeline_config* cfg, int localization_window, int64_t num_samples) {
  if (!cfg || localization_window < 1 || cfg->window_size < 2 || cfg->hop_size < 1 || cfg->num_atoms < 1 || cfg->num_tdoas < 1) return 0;
  const PipeLayout l = pipe_carve(*cfg, num_samples, nullptr, 0, true);
  return l.T >= 1 ? l.bytes : 0;
}

// gccnmf_separate with targets per frame: the window targets of the angular spectrogram (tracking.cu) in place of the one pick
// over the whole clip.  frame_targets (T, S) i32 and status are device outputs; window_means (D, T) f64 may be NULL.  Status bit
// 0 means that some frame held the targets of an earlier one (or the defaults), not that the flow failed.
int gccnmf_separate_tracked(gccnmf_handle* h, const gccnmf_pipeline_config* cfg, int localization_window, const float* samples,
                            int64_t num_samples, const double* window, const double* E, const double* tdoas, float* W, float* H,
                            float* signals, int32_t* frame_targets, double* window_means, int32_t* status, void* workspace,
                            size_t workspace_bytes, void* stream) {
  GCCNMF_ENTER(h);
  GCCNMF_REQUIRE(h, cfg && samples && window && E && tdoas && W && H && signals && frame_targets && status, "separate_tracked: NULL pointer");
  GCCNMF_REQUIRE(h, localization_window >= 1, "separate_tracked: localization window must be >= 1 (got %d)", localization_window);
  GCCNMF_REQUIRE(h, cfg->num_targets >= 0 && cfg->num_iterations >= 0 && cfg->num_tdoas >= 3 && cfg->num_tdoas <= kPickMaxD &&
                        cfg->num_targets <= cfg->num_tdoas && cfg->num_atoms >= 1,
                 "separate_tracked: bad configuration");
  PipeLayout l = pipe_carve(*cfg, num_samples, workspace, workspace_bytes, true);
  GCCNMF_REQUIRE(h, l.T >= 1, "Buffer is too short (n=%lld) for frame_length=%d", (long long)num_samples, cfg->window_size);
  const int N = cfg->window_size, hop = cfg->hop_size, K = cfg->num_atoms, D = cfg->num_tdoas, F = l.F, T = l.T;
  const bool enhancement = cfg->num_targets == 0;
  const int S = enhancement ? 1 : cfg->num_targets;
  GCCNMF_REQUIRE(h, (int64_t)T * S < (int64_t)1 << 31 && (int64_t)S * K * T < (int64_t)1 << 31,
                 "separate_tracked: T x S or S x K x T overflows int32");
  if (!l.ok) return gccnmf_fail(h, GCCNMF_ERR_WORKSPACE, "separate_tracked: workspace too small: need %zu bytes", l.bytes);
  double* means = window_means ? window_means : l.means;
  cudaStream_t s = (cudaStream_t)stream;
  GCCNMF_CHECK_CUDA(h, cudaMemsetAsync(status, 0, sizeof(int32_t), s));
  GCCNMF_CHECK_CUDA(h, cudaMemsetAsync(l.flags, 0, 8 * sizeof(int32_t), s));
  if (int st = gccnmf_stft(h, samples, num_samples, 2, num_samples, window, N, hop, 1, l.X, l.V, stream)) return st;
  if (int st = gccnmf_phat_angspec(h, l.X, F, T, 0, E, D, l.coh, l.angular, nullptr, l.ws_ang, l.n_ang, stream)) return st;
  if (int st = gccnmf_window_targets(h, l.angular, D, T, localization_window, S, means, frame_targets, status, stream)) return st;
  if (int st = gccnmf_klnmf(h, l.V, F, 2 * T, W, H, K, cfg->num_iterations, cfg->sparsity_alpha, cfg->epsilon, 1, l.ws_nmf, l.n_nmf, stream)) return st;
  if (enhancement) {
    if (int st = gccnmf_tdoa_argmax(h, l.coh, F, T, E, D, W, K, l.argmax, l.flags + 1, l.ws_argmax, l.n_argmax, stream)) return st;
    GCCNMF_LAUNCH(h, or_status_kernel, 1, 1, 0, stream, l.flags + 1, gccnmf_tdoa_argmax_refine_capacity(K, T), 4, status);
    if (int st = gccnmf_argmax_mask_frames(h, l.argmax, K, T, tdoas, D, frame_targets, (double)cfg->target_window_seconds, l.table, l.masks, stream))
      return st;
  } else {
    if (int st = gccnmf_target_gccnmf(h, l.coh, F, T, E, D, W, K, frame_targets, S, l.values, stream)) return st;
    if (int st = gccnmf_coeff_mask(h, l.values, S, K, T, l.masks, l.flags + 2, stream)) return st;
    GCCNMF_LAUNCH(h, or_status_kernel, 1, 1, 0, stream, l.flags + 2, 0, 2, status);
  }
  if (int st = gccnmf_masked_recon_phase(h, l.masks, l.X, W, H, S, F, T, K, l.est, l.ws_recon, l.n_recon, stream)) return st;
  return gccnmf_istft_ola(h, l.est, S * 2, N, hop, T, window, (float)((double)hop / (double)N * 2.0), 1, 1, signals, l.ws_istft, l.n_istft, stream);
}

}  // extern "C"
