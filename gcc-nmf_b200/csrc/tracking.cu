// Offline localisation that follows a moving talker: each frame's target TDOAs from a sliding window of the clip's angular
// spectrogram, the rule rt_localize (realtime/gccNMFProcessor.py:219-226) and the gccnmf_llhist_* engines apply per frame, taken
// over a whole stored clip in three launches, and the per-frame enhancement mask of the all-TDOA argmax.
//   window_means   m[d][t] = nanmean of A[d][t], A[d][t - 1], ..., A[d][max(0, t - w + 1)], summed in float64 newest first,
//                  skipping NaN; NaN when every term is NaN.  The window is cut at the start of the clip (the engines' zeroed
//                  ring columns have no counterpart in a stored clip)
//   frame_peaks    per frame, select_peaks(m_t, P) (common.cuh): the P largest strict interior maxima, ascending; a frame with
//                  fewer than P peaks is marked by targets[t][0] = -1
//   hold_targets   a marked frame takes the targets of the latest earlier frame with P peaks, found by a max-scan over frame
//                  indexes, or the defaults floor((2 q + 1) D / (2 P)) before any; status bit 0 when a frame was held
//   tdoa_table     table[tau][d] = |tdoa[d] - tdoa[tau]| < window, float64 (row tau is tdoa_lut_kernel's LUT for target tau)
//   mask_frames    mask[k][t] = table[targets[t]][argmax[k][t]]
#include <cmath>

#include "common.cuh"

namespace {

constexpr int kMaxD = 1024;
constexpr int kMeanFrames = 64;      // output frames per CTA of window_means_kernel
constexpr int kMeanRows = 4;         // TDOA rows per CTA
constexpr int kMeanChunk = 256;      // input columns staged per pass

// CTA = kMeanFrames frames x kMeanRows rows, thread (r, j) = frame t0 + j of row d0 + r.  The input columns the tile needs,
// [max(0, t0 - w + 1), t0 + kMeanFrames), are staged in chunks from the newest down, so each output's terms are added newest
// first across chunks as within one, and A is read once per tile whatever w is.
__global__ void __launch_bounds__(kMeanFrames * kMeanRows)
window_means_kernel(const double* __restrict__ A, int D, int T, int w, double* __restrict__ means) {
  __shared__ double cols[kMeanRows][kMeanChunk];
  const int j = threadIdx.x % kMeanFrames, r = threadIdx.x / kMeanFrames;
  const int t0 = blockIdx.x * kMeanFrames, d0 = blockIdx.y * kMeanRows;
  const int t = t0 + j, d = d0 + r;
  const int lo = t0 - w + 1 > 0 ? t0 - w + 1 : 0;
  const int hi = t0 + kMeanFrames < T ? t0 + kMeanFrames : T;
  const int first = t - w + 1 > 0 ? t - w + 1 : 0;      // oldest column of this output's window
  double sum = 0.0;
  int n = 0;
  for (int c1 = hi; c1 > lo; c1 -= kMeanChunk) {
    const int c0 = c1 - kMeanChunk > lo ? c1 - kMeanChunk : lo;
    const int width = c1 - c0;
    for (int i = threadIdx.x; i < kMeanRows * kMeanChunk; i += blockDim.x) {
      const int rr = i / kMeanChunk, c = i % kMeanChunk;
      if (c < width && d0 + rr < D) cols[rr][c] = A[(int64_t)(d0 + rr) * T + c0 + c];
    }
    __syncthreads();
    if (t < T && d < D) {
      const int top = t < c1 - 1 ? t : c1 - 1;
      const int bottom = first > c0 ? first : c0;
      for (int c = top; c >= bottom; --c) {
        const double v = cols[r][c - c0];
        if (v == v) { sum += v; ++n; }
      }
    }
    __syncthreads();
  }
  if (t < T && d < D) means[(int64_t)d * T + t] = n > 0 ? sum / (double)n : __longlong_as_double(0x7ff8000000000000LL);
}

// One CTA per frame: the P largest peaks of the frame's window mean into targets[t], or -1 in targets[t][0] with fewer.
__global__ void __launch_bounds__(128)
frame_peaks_kernel(const double* __restrict__ means, int D, int T, int P, int32_t* __restrict__ targets) {
  __shared__ double x[kMaxD];
  __shared__ unsigned char peak[kMaxD], chosen[kMaxD];
  __shared__ int num_peaks;
  const int t = blockIdx.x;
  for (int d = threadIdx.x; d < D; d += blockDim.x) x[d] = means[(int64_t)d * T + t];
  int32_t* out = targets + (int64_t)t * P;
  const int peaks = select_peaks(x, D, P, peak, chosen, &num_peaks, out);
  if (threadIdx.x == 0 && peaks < P) out[0] = -1;
}

// One CTA of 1024 threads walks the frames in chunks of 1024.  In a chunk, src[t] = the largest frame index u <= t whose
// targets[u][0] >= 0 (an inclusive max-scan: warp shuffles, then one warp over the warp totals), with the carry of the chunks
// before.  A marked frame copies src's targets or takes the defaults.  Only marked frames are written and only unmarked frames
// are read as sources, so the pass runs in place.
__global__ void __launch_bounds__(1024)
hold_targets_kernel(int32_t* __restrict__ targets, int T, int P, int D, int32_t* __restrict__ status) {
  __shared__ int warp_max[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, warps = blockDim.x >> 5;
  int carry = -1;
  bool held = false;
  for (int base = 0; base < T; base += blockDim.x) {
    const int t = base + threadIdx.x;
    const bool ok = t < T && targets[(int64_t)t * P] >= 0;
    int v = ok ? t : -1;
    for (int o = 1; o < 32; o <<= 1) {
      const int u = __shfl_up_sync(0xffffffffu, v, o);
      if (lane >= o) v = max(v, u);
    }
    if (lane == 31) warp_max[warp] = v;
    __syncthreads();
    if (warp == 0) {
      int x = lane < warps ? warp_max[lane] : -1;
      for (int o = 1; o < 32; o <<= 1) {
        const int u = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x = max(x, u);
      }
      warp_max[lane] = x;
    }
    __syncthreads();
    const int src = max(carry, max(warp > 0 ? warp_max[warp - 1] : -1, v));
    if (t < T && !ok) {
      held = true;
      for (int q = 0; q < P; ++q)
        targets[(int64_t)t * P + q] = src >= 0 ? targets[(int64_t)src * P + q] : (2 * q + 1) * D / (2 * P);
    }
    carry = max(carry, warp_max[warps - 1]);
    __syncthreads();
  }
  if (__syncthreads_or(held) && threadIdx.x == 0) atomicOr(status, 1);
}

// table[tau][d]: tdoa_lut_kernel's expression with target tau.
__global__ void tdoa_table_kernel(const double* __restrict__ tdoas, int D, double window, uint8_t* __restrict__ table) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= D * D) return;
  const int tau = i / D, d = i - tau * D;
  table[i] = fabs(tdoas[d] - tdoas[tau]) < window ? 1 : 0;
}

__global__ void argmax_mask_frames_kernel(const int32_t* __restrict__ argmax, int T, int64_t KT, const uint8_t* __restrict__ table, int D,
                                          const int32_t* __restrict__ targets, float* __restrict__ mask) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= KT) return;
  const int a = argmax[i], tau = targets[i % T];
  mask[i] = (a >= 0 && a < D && tau >= 0 && tau < D && table[(int64_t)tau * D + a]) ? 1.f : 0.f;
}

// The three launches of gccnmf_window_targets, on arguments it has checked.
int window_targets_enqueue(gccnmf_handle* h, const double* angular, int D, int T, int window, int P, double* means, int32_t* targets,
                           int32_t* status, void* stream) {
  const dim3 grid((T + kMeanFrames - 1) / kMeanFrames, (D + kMeanRows - 1) / kMeanRows);
  GCCNMF_LAUNCH(h, window_means_kernel, grid, kMeanFrames * kMeanRows, 0, stream, angular, D, T, window, means);
  GCCNMF_LAUNCH(h, frame_peaks_kernel, T, 128, 0, stream, means, D, T, P, targets);
  GCCNMF_LAUNCH(h, hold_targets_kernel, 1, 1024, 0, stream, targets, T, P, D, status);
  return GCCNMF_OK;
}

}  // namespace

extern "C" {

// angular (D, T) f64 -> targets (T, P) i32 [, means (D, T) f64]; status |= 1 when a frame was held.  Without `means` the window
// means live in a stream-ordered allocation for the duration of the call.
int gccnmf_window_targets(gccnmf_handle* h, const double* angular, int D, int T, int window, int P, double* means, int32_t* targets,
                          int32_t* status, void* stream) {
  GCCNMF_ENTER(h);
  GCCNMF_REQUIRE(h, angular && targets && status, "window_targets: NULL pointer");
  GCCNMF_REQUIRE(h, window >= 1, "window_targets: window must be >= 1 (got %d)", window);
  GCCNMF_REQUIRE(h, D >= 3 && D <= kMaxD, "window_targets: numTDOAs must be in [3, %d] (got %d)", kMaxD, D);
  GCCNMF_REQUIRE(h, P >= 1 && P <= D, "window_targets: number of targets must be in [1, D] (got %d)", P);
  GCCNMF_REQUIRE(h, T >= 1 && (int64_t)T * P < (int64_t)1 << 31, "window_targets: T (%d) x P (%d) must be in [1, 2^31)", T, P);
  if (means) return window_targets_enqueue(h, angular, D, T, window, P, means, targets, status, stream);
  cudaStream_t s = (cudaStream_t)stream;
  double* m = nullptr;
  GCCNMF_CHECK_CUDA(h, cudaMallocAsync(reinterpret_cast<void**>(&m), (size_t)D * T * sizeof(double), s));
  const int st = window_targets_enqueue(h, angular, D, T, window, P, m, targets, status, stream);
  const cudaError_t freed = cudaFreeAsync(m, s);      // on every path, a failed launch included
  if (st != GCCNMF_OK) return st;
  if (freed != cudaSuccess) return gccnmf_fail(h, GCCNMF_ERR_CUDA, "window_targets: cudaFreeAsync failed: %s", cudaGetErrorString(freed));
  return GCCNMF_OK;
}

// mask (K, T) f32 = |tdoa[argmax[k][t]] - tdoa[targets[t]]| < window_seconds; lut_workspace holds the (D, D) u8 table.
int gccnmf_argmax_mask_frames(gccnmf_handle* h, const int32_t* argmax, int K, int T, const double* tdoas, int D, const int32_t* targets,
                              double window_seconds, uint8_t* lut_workspace, float* mask, void* stream) {
  GCCNMF_ENTER(h);
  GCCNMF_REQUIRE(h, argmax && tdoas && targets && lut_workspace && mask, "argmax_mask_frames: NULL pointer");
  GCCNMF_REQUIRE(h, K >= 1 && T >= 1 && D >= 1 && D <= kMaxD, "argmax_mask_frames: bad arguments (K %d, T %d, D %d)", K, T, D);
  const int64_t KT = (int64_t)K * T;
  GCCNMF_LAUNCH(h, tdoa_table_kernel, (D * D + 255) / 256, 256, 0, stream, tdoas, D, window_seconds, lut_workspace);
  GCCNMF_LAUNCH(h, argmax_mask_frames_kernel, (unsigned)((KT + 255) / 256), 256, 0, stream, argmax, T, KT, lut_workspace, D, targets, mask);
  return GCCNMF_OK;
}

}  // extern "C"
