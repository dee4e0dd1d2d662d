// Windowed STFT (reference: gccNMF/librosaSTFT.py:20-181) and inverse STFT with overlap-add
// (librosaSTFT.py:183-286) as shared-memory FFT kernels.
//
// Forward: the reference multiplies float32 frames by a float64 window and runs a double-precision
// FFT, rounding once to complex64; this kernel does the same arithmetic in float64 in shared memory
// so the complex64 output agrees to the last bit almost everywhere (and the PHAT normalisation
// downstream, which amplifies relative error in weak bins, sees the same numbers).  The two
// channels of a stereo frame are packed as one complex signal (left + i right), transformed once,
// and separated with the Hermitian split.  A block transforms FB consecutive frames and stages the
// results in shared memory so that the (channel, F, T) output is written in contiguous runs along T.
//
// Inverse: complex64 input keeps the reference's inverse FFT in single precision, so this is a
// float32 FFT; two real frames (batch entries 2j and 2j+1) share one complex inverse transform.
// Overlap-add is a gather: each output sample adds its <= ceil(N/hop) frames in frame order with the
// reference's float32 rounding after every add, so no atomics and bit-stable results.
#include <cmath>
#include <vector>

#include "common.cuh"
#include "fft.cuh"

namespace {

// ---------------------------------------------------------------------------------- forward
// dynamic smem: double2 fft[n] | float2 stage[channels][F][FB]
template <int FB>
__global__ void __launch_bounds__(kFftThreads)
stft_kernel(const float* __restrict__ samples, int64_t sample_stride, int channels, const double* __restrict__ window,
            const double2* __restrict__ tw, int n, int log2n, int hop, int T, int conjugate,
            float2* __restrict__ X, float* __restrict__ V, int frames_per_seg, int64_t seg_stride) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  double2* fft = reinterpret_cast<double2*>(smem_raw);
  float2* stage = reinterpret_cast<float2*>(smem_raw + (size_t)n * sizeof(double2));
  const int F = n / 2 + 1;
  const int t0 = blockIdx.x * FB;
  const int frames = min(FB, T - t0);

  for (int fb = 0; fb < frames; ++fb) {
    // frame t is frame t % frames_per_seg of segment t / frames_per_seg (one signal: frames_per_seg = T, seg_stride = 0)
    const int t = t0 + fb;
    const int64_t start = (int64_t)(t / frames_per_seg) * seg_stride + (int64_t)(t % frames_per_seg) * hop;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      const double w = window[i];
      const double l = w * (double)samples[start + i];
      const double r = channels > 1 ? w * (double)samples[sample_stride + start + i] : 0.0;
      fft[bitrev(i, log2n)] = double2{l, r};
    }
    __syncthreads();
    fft_inplace<double2, double>(fft, tw, n, log2n, false);
    // Hermitian split: XL[k] = (Z[k] + conj(Z[n-k])) / 2,  XR[k] = (Z[k] - conj(Z[n-k])) / (2i)
    for (int k = threadIdx.x; k < F; k += blockDim.x) {
      const double2 a = fft[k];
      const double2 b = fft[(n - k) & (n - 1)];
      double lr = 0.5 * (a.x + b.x), li = 0.5 * (a.y - b.y);
      double rr = 0.5 * (a.y + b.y), ri = 0.5 * (b.x - a.x);
      if (conjugate) { li = -li; ri = -ri; }
      stage[(0 * F + k) * FB + fb] = float2{(float)lr, (float)li};
      if (channels > 1) stage[(1 * F + k) * FB + fb] = float2{(float)rr, (float)ri};
    }
    __syncthreads();
  }
  // coalesced write-out: runs of `frames` consecutive t per (channel, f)
  const int total = channels * F * FB;
  for (int e = threadIdx.x; e < total; e += blockDim.x) {
    const int fb = e % FB;
    if (fb >= frames) continue;
    const int cf = e / FB;  // channel * F + f
    const int c = cf / F, f = cf - c * F;
    const float2 v = stage[e];
    X[(int64_t)cf * T + t0 + fb] = v;
    if (V) {
      const double mag = sqrt((double)v.x * (double)v.x + (double)v.y * (double)v.y);
      V[(int64_t)f * ((int64_t)channels * T) + (int64_t)c * T + t0 + fb] = (float)mag;
    }
  }
}

// ---------------------------------------------------------------------------------- inverse
// One block per (frame batch, batch pair).  dynamic smem: float2 fft[n] | float2 stage[2][F][FB]
template <int FB>
__global__ void __launch_bounds__(kFftThreads)
istft_frames_kernel(const float2* __restrict__ spec, int batch, const float2* __restrict__ tw, int n, int log2n, int T,
                    int conjugate, float* __restrict__ frames_out) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float2* fft = reinterpret_cast<float2*>(smem_raw);
  float2* stage = reinterpret_cast<float2*>(smem_raw + (size_t)n * sizeof(float2));
  const int F = n / 2 + 1;
  const int t0 = blockIdx.x * FB;
  const int frames = min(FB, T - t0);
  const int b0 = blockIdx.y * 2;
  const bool has_second = b0 + 1 < batch;

  // gather FB columns of both batch entries: runs of `frames` consecutive t per f
  const int total = 2 * F * FB;
  for (int e = threadIdx.x; e < total; e += blockDim.x) {
    const int fb = e % FB;
    const int bf = e / FB;
    const int which = bf / F, f = bf - which * F;
    float2 v = float2{0.f, 0.f};
    if (fb < frames && (which == 0 || has_second)) v = spec[((int64_t)(b0 + which) * F + f) * T + t0 + fb];
    stage[e] = v;
  }
  __syncthreads();

  const float inv_n = 1.0f / (float)n;
  for (int fb = 0; fb < frames; ++fb) {
    // full spectrum of (A + iB) with A, B the Hermitian extensions of conj(col) (librosaSTFT.py:278);
    // imaginary parts of the DC and Nyquist bins only feed the discarded imaginary output.
    for (int k = threadIdx.x; k < F; k += blockDim.x) {
      float2 a = stage[(0 * F + k) * FB + fb];
      float2 b = stage[(1 * F + k) * FB + fb];
      if (conjugate) { a.y = -a.y; b.y = -b.y; }
      if (k == 0 || k == n / 2) { a.y = 0.f; b.y = 0.f; }
      // Z[k] = A[k] + i B[k];  Z[n-k] = conj(A[k]) + i conj(B[k])
      fft[bitrev(k, log2n)] = float2{a.x - b.y, a.y + b.x};
      if (k != 0 && k != n / 2) fft[bitrev(n - k, log2n)] = float2{a.x + b.y, b.x - a.y};
    }
    __syncthreads();
    fft_inplace<float2, float>(fft, tw, n, log2n, true);
    float* out0 = frames_out + ((int64_t)b0 * T + t0 + fb) * n;
    float* out1 = frames_out + ((int64_t)(b0 + 1) * T + t0 + fb) * n;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      const float2 z = fft[i];
      out0[i] = z.x * inv_n;
      if (has_second) out1[i] = z.y * inv_n;
    }
    __syncthreads();
  }
}

// y[b][j] = gain * OLA[b][offset + j];  OLA[m] = sum over frames i (ascending) of window[m - i hop] * frame_i[m - i hop]
// rounded to float32 after every add like the reference (librosaSTFT.py:279-281), but the float64 product and sum are
// contracted into one DFMA: y = float32(fma(window, float64(frame), float64(y))), where the reference rounds the product first.
__global__ void ola_gather_kernel(const float* __restrict__ frames, const double* __restrict__ window, int n, int hop,
                                  int T, int64_t offset, int64_t length, float gain, float* __restrict__ y) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y;
  if (j >= length) return;
  const int64_t m = j + offset;
  int64_t i_first = (m - n + hop) / hop;  // ceil((m - n + 1) / hop) for m - n + 1 > 0
  if (m - n + 1 <= 0) i_first = 0;
  int64_t i_last = m / hop;
  if (i_last > T - 1) i_last = T - 1;
  float acc = 0.f;
  const float* fb = frames + (int64_t)b * T * n;
  for (int64_t i = i_first; i <= i_last; ++i) {
    const int r = (int)(m - i * hop);
    acc = (float)((double)acc + window[r] * (double)fb[i * n + r]);
  }
  y[(int64_t)b * length + j] = acc * gain;
}

template <typename K>
int set_smem(gccnmf_handle* h, K kernel, size_t bytes) {
  GCCNMF_CHECK_CUDA(h, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  return 0;
}

int ilog2_exact(int n) {
  int l = 0;
  while ((1 << l) < n) ++l;
  return (1 << l) == n ? l : -1;
}

}  // namespace

int gccnmf_get_twiddles(gccnmf_handle* h, int n, const double** tw64, const float** tw32) {
  int slot = -1;
  for (int i = 0; i < gccnmf_handle::kMaxPlans; ++i) {
    if (h->plan_n[i] == n) { slot = i; break; }
    if (h->plan_n[i] == 0 && slot < 0) slot = i;
  }
  if (slot < 0) return gccnmf_fail(h, GCCNMF_ERR_UNSUPPORTED, "more than %d distinct FFT sizes on one handle", gccnmf_handle::kMaxPlans);
  if (h->plan_n[slot] != n) {
    std::vector<double> t64(n);
    std::vector<float> t32(n);
    for (int j = 0; j < n / 2; ++j) {
      const double a = -2.0 * M_PI * (double)j / (double)n;
      t64[2 * j] = cos(a);  t64[2 * j + 1] = sin(a);
      t32[2 * j] = (float)cos(a);  t32[2 * j + 1] = (float)sin(a);
    }
    GCCNMF_CHECK_CUDA(h, cudaMalloc(&h->plan_tw64[slot], n * sizeof(double)));
    GCCNMF_CHECK_CUDA(h, cudaMalloc(&h->plan_tw32[slot], n * sizeof(float)));
    GCCNMF_CHECK_CUDA(h, cudaMemcpy(h->plan_tw64[slot], t64.data(), n * sizeof(double), cudaMemcpyHostToDevice));
    GCCNMF_CHECK_CUDA(h, cudaMemcpy(h->plan_tw32[slot], t32.data(), n * sizeof(float), cudaMemcpyHostToDevice));
    h->plan_n[slot] = n;
  }
  if (tw64) *tw64 = h->plan_tw64[slot];
  if (tw32) *tw32 = h->plan_tw32[slot];
  return 0;
}

// Frames of `segments` signals in one launch: frame (g, i) starts at g * seg_stride + i * hop of each channel row, for
// i < frames_per_seg, and is column g * frames_per_seg + i of X.  Every frame is transformed on its own, so its bits do not depend
// on how many frames share the launch.
int gccnmf_stft_segments(gccnmf_handle* h, const float* samples, int64_t sample_stride, int channels, int segments, int frames_per_seg,
                         int64_t seg_stride, const double* window, int n_fft, int hop, int conjugate, float* X, float* V, void* stream) {
  const int log2n = ilog2_exact(n_fft);
  if (log2n < 5 || log2n > 12) return gccnmf_fail(h, GCCNMF_ERR_UNSUPPORTED, "stft: n_fft must be a power of two in [32, 4096] (got %d)", n_fft);
  GCCNMF_REQUIRE(h, channels == 1 || channels == 2, "stft: channels must be 1 or 2 (got %d)", channels);
  GCCNMF_REQUIRE(h, hop >= 1, "Invalid hop_length: %d", hop);
  GCCNMF_REQUIRE(h, segments >= 1 && frames_per_seg >= 1 && (int64_t)segments * frames_per_seg < ((int64_t)1 << 31), "stft: bad frame count");
  const int T = segments * frames_per_seg;
  GCCNMF_REQUIRE(h, samples && window && X, "stft: NULL pointer");
  const double* tw = nullptr;
  if (int st = gccnmf_get_twiddles(h, n_fft, &tw, nullptr)) return st;
  const int F = n_fft / 2 + 1;
  auto smem_for = [&](int fb) { return (size_t)n_fft * sizeof(double2) + (size_t)channels * F * fb * sizeof(float2); };
#define GCCNMF_STFT_CASE(FB)                                                                                  \
  {                                                                                                           \
    auto k = stft_kernel<FB>;                                                                                 \
    const size_t smem = smem_for(FB);                                                                         \
    if (int st = set_smem(h, k, smem)) return st;                                                             \
    GCCNMF_LAUNCH(h, k, (T + FB - 1) / FB, kFftThreads, smem, stream, samples, sample_stride, channels,       \
                  window, reinterpret_cast<const double2*>(tw), n_fft, log2n, hop, T, conjugate,             \
                  reinterpret_cast<float2*>(X), V, frames_per_seg, seg_stride);                               \
  }
  if (T >= 8 && smem_for(8) <= 160 * 1024) GCCNMF_STFT_CASE(8)
  else if (T >= 4 && smem_for(4) <= 160 * 1024) GCCNMF_STFT_CASE(4)
  else GCCNMF_STFT_CASE(1)
#undef GCCNMF_STFT_CASE
  return GCCNMF_OK;
}

// The per-frame inverse transforms of gccnmf_istft_ola without the overlap-add: spec (batch, F, T) c64 -> frames (batch', T, n) f32
// (batch' = batch rounded up to even), the arithmetic of every frame exactly as there.
int gccnmf_istft_frames(gccnmf_handle* h, const float* spec, int batch, int n_fft, int T, int conjugate, float* frames, void* stream) {
  const int log2n = ilog2_exact(n_fft);
  if (log2n < 5 || log2n > 12) return gccnmf_fail(h, GCCNMF_ERR_UNSUPPORTED, "istft: n_fft must be a power of two in [32, 4096] (got %d)", n_fft);
  GCCNMF_REQUIRE(h, batch >= 1 && T >= 1 && spec && frames, "istft: bad arguments");
  const float* tw = nullptr;
  if (int st = gccnmf_get_twiddles(h, n_fft, nullptr, &tw)) return st;
  const int F = n_fft / 2 + 1;
  auto smem_for = [&](int fb) { return (size_t)n_fft * sizeof(float2) + (size_t)2 * F * fb * sizeof(float2); };
#define GCCNMF_ISTFT_CASE(FB)                                                                                 \
  {                                                                                                           \
    auto k = istft_frames_kernel<FB>;                                                                         \
    const size_t smem = smem_for(FB);                                                                         \
    if (int st = set_smem(h, k, smem)) return st;                                                             \
    GCCNMF_LAUNCH(h, k, dim3((T + FB - 1) / FB, (batch + 1) / 2), kFftThreads, smem, stream,                  \
                  reinterpret_cast<const float2*>(spec), batch, reinterpret_cast<const float2*>(tw), n_fft,   \
                  log2n, T, conjugate, frames);                                                               \
  }
  if (T >= 8 && smem_for(8) <= 160 * 1024) GCCNMF_ISTFT_CASE(8)
  else if (T >= 4 && smem_for(4) <= 160 * 1024) GCCNMF_ISTFT_CASE(4)
  else GCCNMF_ISTFT_CASE(1)
#undef GCCNMF_ISTFT_CASE
  return GCCNMF_OK;
}

extern "C" {

int gccnmf_stft_num_frames(int64_t num_samples, int n_fft, int hop) {
  if (n_fft <= 0 || hop < 1) return GCCNMF_ERR_INVALID_ARGUMENT;        // librosaSTFT.py:416-417
  if (num_samples < n_fft) return GCCNMF_ERR_INVALID_ARGUMENT;           // librosaSTFT.py:427-430
  return 1 + (int)((num_samples - n_fft) / hop);                         // librosaSTFT.py:425
}

int gccnmf_stft(gccnmf_handle* h, const float* samples, int64_t sample_stride, int channels, int64_t num_samples,
                const double* window, int n_fft, int hop, int conjugate, float* X, float* V, void* stream) {
  GCCNMF_ENTER(h);
  const int log2n = ilog2_exact(n_fft);
  if (log2n < 5 || log2n > 12) return gccnmf_fail(h, GCCNMF_ERR_UNSUPPORTED, "stft: n_fft must be a power of two in [32, 4096] (got %d)", n_fft);
  GCCNMF_REQUIRE(h, channels == 1 || channels == 2, "stft: channels must be 1 or 2 (got %d)", channels);
  GCCNMF_REQUIRE(h, hop >= 1, "Invalid hop_length: %d", hop);
  const int T = gccnmf_stft_num_frames(num_samples, n_fft, hop);
  GCCNMF_REQUIRE(h, T >= 1, "Buffer is too short (n=%lld) for frame_length=%d", (long long)num_samples, n_fft);
  return gccnmf_stft_segments(h, samples, sample_stride, channels, 1, T, 0, window, n_fft, hop, conjugate, X, V, stream);
}

int64_t gccnmf_istft_length(int n_fft, int hop, int T, int center) {
  if (n_fft <= 0 || hop < 1 || T < 1) return GCCNMF_ERR_INVALID_ARGUMENT;
  return (int64_t)n_fft + (int64_t)hop * (T - 1) - (center ? n_fft : 0);
}

size_t gccnmf_istft_workspace_bytes(int batch, int n_fft, int T) {
  if (batch <= 0 || n_fft <= 0 || T <= 0) return 0;
  return align_up((size_t)((batch + 1) / 2 * 2) * T * n_fft * sizeof(float), 256);
}

int gccnmf_istft_ola(gccnmf_handle* h, const float* spec, int batch, int n_fft, int hop, int T, const double* window,
                     float gain, int center, int conjugate, float* y, void* workspace, size_t workspace_bytes, void* stream) {
  GCCNMF_ENTER(h);
  const int log2n = ilog2_exact(n_fft);
  if (log2n < 5 || log2n > 12) return gccnmf_fail(h, GCCNMF_ERR_UNSUPPORTED, "istft: n_fft must be a power of two in [32, 4096] (got %d)", n_fft);
  GCCNMF_REQUIRE(h, batch >= 1 && T >= 1 && hop >= 1, "istft: batch, T, hop must be positive");
  GCCNMF_REQUIRE(h, spec && window, "istft: NULL pointer");
  if (gccnmf_istft_length(n_fft, hop, T, center) <= 0) return GCCNMF_OK;  // centre trim leaves nothing (single frame)
  GCCNMF_REQUIRE(h, y != nullptr, "istft: NULL output pointer");
  if (!workspace || workspace_bytes < gccnmf_istft_workspace_bytes(batch, n_fft, T))
    return gccnmf_fail(h, GCCNMF_ERR_WORKSPACE, "istft workspace too small: need %zu bytes", gccnmf_istft_workspace_bytes(batch, n_fft, T));
  float* frames = static_cast<float*>(workspace);
  if (int st = gccnmf_istft_frames(h, spec, batch, n_fft, T, conjugate, frames, stream)) return st;
  const int64_t length = gccnmf_istft_length(n_fft, hop, T, center);
  if (length > 0) {
    const int64_t offset = center ? n_fft / 2 : 0;
    GCCNMF_LAUNCH(h, ola_gather_kernel, dim3((unsigned)((length + 255) / 256), batch), 256, 0, stream, frames, window,
                  n_fft, hop, T, offset, length, gain, y);
  }
  return GCCNMF_OK;
}

}  // extern "C"
