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
#include <cmath>

#include "common.cuh"

int gccnmf_stft_segments(gccnmf_handle* h, const float* samples, int64_t sample_stride, int channels, int segments, int frames_per_seg,
                         int64_t seg_stride, const double* window, int n_fft, int hop, int conjugate, float* X, float* V, void* stream);
int gccnmf_istft_frames(gccnmf_handle* h, const float* spec, int batch, int n_fft, int T, int conjugate, float* frames, void* stream);
int gccnmf_tdoa_gccnmf_gated(gccnmf_handle* h, const float* coherence, int F, int T, const double* E, int D, const float* W, int K,
                             int32_t* argmax, const int32_t* gate, int capacity, int32_t* ran, void* stream);

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
  size_t bytes;
  LLHeader* head;
  LLStream* streams;
  double *win_a, *w_syn, *E, *carry, *acc, *ang;
  float *W, *WT, *colsumW, *H0, *in_ring, *out_ring, *stage, *X, *V, *coh, *mask, *wiener, *Y, *H, *frames, *ws_wiener;
  int32_t *targets, *valid, *argmax, *counters;   // counters: [0] refined count, [1] status
  void* ws_argmax;
  size_t n_argmax;
};

bool is_pow2(int x) { return x > 0 && (x & (x - 1)) == 0; }
constexpr int kLLInferMaxSmem = 227 * 1024;   // the H100's opt-in dynamic shared memory per block

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

LLLayout ll_carve(const gccnmf_ll_config& c, void* base) {
  WorkspaceCarver w(base ? base : reinterpret_cast<void*>(256), base ? ~size_t(0) >> 1 : ~size_t(0) >> 1);
  LLLayout l{};
  l.S = c.num_streams; l.N = c.window_size; l.hop = c.hop_size; l.C = c.hops_per_call; l.K = c.num_atoms; l.D = c.num_tdoas;
  l.F = l.N / 2 + 1; l.Q = (l.N + l.hop - 1) / l.hop; l.R = (l.Q - 1) * l.hop;
  const size_t S = l.S, N = l.N, F = l.F, K = l.K, D = l.D, T = S * l.C;
  const bool inf = c.inference_iterations > 0;
  l.head = w.take<LLHeader>(1);
  l.streams = w.take<LLStream>(S);
  l.counters = w.take<int32_t>(4);
  l.win_a = w.take<double>(N);
  l.w_syn = w.take<double>(N);
  l.E = w.take<double>(2 * F * D);
  l.W = w.take<float>(F * K);
  l.WT = w.take<float>(inf ? K * F : 0);
  l.colsumW = w.take<float>(inf ? K : 0);
  l.H0 = w.take<float>(inf ? K * 2 : 0);
  l.in_ring = w.take<float>(S * 2 * l.R);
  l.out_ring = w.take<float>(S * 2 * N);
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
  l.wiener = w.take<float>((inf ? 2 : 1) * F * T);
  l.Y = w.take<float>(2 * 2 * F * T);
  l.H = w.take<float>(inf ? K * 2 * T : 0);
  l.frames = w.take<float>(2 * T * N);
  l.ws_wiener = w.take<float>(gccnmf_wiener_apply_workspace_bytes((int)F) / sizeof(float));
  l.n_argmax = gccnmf_tdoa_argmax_workspace_bytes((int)F, (int)T, (int)D, (int)K);
  l.ws_argmax = w.take<unsigned char>(l.n_argmax);
  l.bytes = align_up(w.used, 256);
  return l;
}

#define LL_CARVE_OR_FAIL(l)                                                                                          \
  if (int st__ = ll_check(h, cfg)) return st__;                                                                      \
  GCCNMF_REQUIRE(h, state != nullptr, "ll: NULL state");                                                             \
  const LLLayout l = ll_carve(*cfg, state);                                                                          \
  if (state_bytes < l.bytes) return gccnmf_fail(h, GCCNMF_ERR_WORKSPACE, "ll: state too small: need %zu bytes", l.bytes);

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

// One CTA per stream, thread d = TDOA: the running maximum of cummax_time_kernel from the carried one over the call's valid frames,
// then target[t] = argmax over d (argmax_tdoa_kernel), or the stream's override.
__global__ void ll_targets_kernel(const LLStream* __restrict__ streams, const double* __restrict__ ang, const int32_t* __restrict__ valid, int D,
                                  int hops, int T, double* __restrict__ carry, double* __restrict__ acc, int32_t* __restrict__ targets) {
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

// One CTA per stream.  For each frame of the call in order: ring[p] = float32(fma(w[r], frame[r], ring[p])) for r >= z,
// p = (j hop + r) mod N (ola_gather_kernel's chain: the weights below z are zero and would leave every sum as it is), then
// emit the hop samples [j hop + z, j hop + z + hop) times the gain and zero them.  Then the input ring moves on.
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
  const int z = head->z;
  const float gain = head->gain;
  const long long h0 = streams[s].hops;
  float* ring = out_ring + (int64_t)s * 2 * N;
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
  // the last R samples of the staging rows are the next call's input ring
  const int S = gridDim.x;
  const int64_t Lseg = (int64_t)R + n;
  for (int e = threadIdx.x; e < 2 * R; e += blockDim.x) {
    const int ch = e >= R, q = e - ch * R;
    in_ring[((int64_t)s * 2 + ch) * R + q] = stage[((int64_t)ch * S + s) * Lseg + n + q];
  }
  if (threadIdx.x == 0) streams[s].hops = h0 + hops;
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
  if (int e = gccnmf_phat_angspec(h, l.X, F, T, 0, l.E, D, l.coh, l.ang, nullptr, nullptr, 0, stream)) return e;
  GCCNMF_LAUNCH(h, ll_targets_kernel, S, 128, 0, stream, l.streams, l.ang, l.valid, D, hops, T, l.carry, l.acc, l.targets);
  if (int e = gccnmf_tdoa_argmax(h, l.coh, F, T, l.E, D, l.W, K, l.argmax, l.counters, l.ws_argmax, l.n_argmax, stream)) return e;
  if (int e = gccnmf_tdoa_gccnmf_gated(h, l.coh, F, T, l.E, D, l.W, K, l.argmax, l.counters, gccnmf_tdoa_argmax_refine_capacity(K, T),
                                       l.counters + 1, stream))
    return e;
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

}  // namespace

extern "C" {

size_t gccnmf_ll_state_bytes(const gccnmf_ll_config* cfg) {
  if (ll_check(nullptr, cfg) != 0) return 0;
  return ll_carve(*cfg, nullptr).bytes;
}

int gccnmf_ll_init(gccnmf_handle* h, const gccnmf_ll_config* cfg, const float* W, const double* E, const double* analysis_window,
                   const double* synthesis_weights, float gain, const float* H0, void* state, size_t state_bytes, void* stream) {
  GCCNMF_ENTER(h);
  LL_CARVE_OR_FAIL(l);
  GCCNMF_REQUIRE(h, W && E && analysis_window && synthesis_weights, "ll_init: NULL pointer");
  GCCNMF_REQUIRE(h, cfg->inference_iterations == 0 || H0 != nullptr, "ll_init: inference needs H0");
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
  GCCNMF_CHECK_CUDA(h, cudaMemcpyAsync(l.E, E, (size_t)2 * l.F * l.D * sizeof(double), cudaMemcpyDeviceToDevice, s));
  GCCNMF_CHECK_CUDA(h, cudaMemcpyAsync(l.W, W, (size_t)l.F * l.K * sizeof(float), cudaMemcpyDeviceToDevice, s));
  if (cfg->inference_iterations > 0) {
    GCCNMF_CHECK_CUDA(h, cudaMemcpyAsync(l.H0, H0, (size_t)l.K * 2 * sizeof(float), cudaMemcpyDeviceToDevice, s));
    GCCNMF_LAUNCH(h, ll_dict_kernel, (l.K + 127) / 128, 128, 0, stream, l.W, l.F, l.K, l.WT, l.colsumW);
  }
  GCCNMF_LAUNCH(h, ll_header_kernel, 1, 1, 0, stream, l.head, l.w_syn, l.N, gain);
  GCCNMF_LAUNCH(h, ll_reset_kernel, l.S, 256, 0, stream, l.streams, 0, l.S, l.in_ring, l.out_ring, l.carry, l.R, l.N, l.D, 1);
  return GCCNMF_OK;
}

int gccnmf_ll_reset_streams(gccnmf_handle* h, const gccnmf_ll_config* cfg, void* state, size_t state_bytes, int first, int count, void* stream) {
  GCCNMF_ENTER(h);
  LL_CARVE_OR_FAIL(l);
  GCCNMF_REQUIRE(h, first >= 0 && count >= 1 && first < l.S && count <= l.S - first, "ll_reset_streams: streams [%d, %d + %d) outside [0, %d)", first,
                 first, count, l.S);
  GCCNMF_LAUNCH(h, ll_reset_kernel, count, 256, 0, stream, l.streams, first, count, l.in_ring, l.out_ring, l.carry, l.R, l.N, l.D, 0);
  return GCCNMF_OK;
}

int gccnmf_ll_set_params(gccnmf_handle* h, const gccnmf_ll_config* cfg, void* state, size_t state_bytes, int first, int count,
                         const gccnmf_ll_stream_params* params_host, void* stream) {
  GCCNMF_ENTER(h);
  LL_CARVE_OR_FAIL(l);
  GCCNMF_REQUIRE(h, first >= 0 && count >= 1 && first < l.S && count <= l.S - first, "ll_set_params: streams [%d, %d + %d) outside [0, %d)", first,
                 first, count, l.S);
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

int gccnmf_ll_process(gccnmf_handle* h, const gccnmf_ll_config* cfg, void* state, size_t state_bytes, int hops, const float* in, float* out,
                      void* stream) {
  GCCNMF_ENTER(h);
  LL_CARVE_OR_FAIL(l);
  return ll_enqueue(h, cfg, l, hops, in, out, stream);
}

int gccnmf_ll_graph_create(gccnmf_handle* h, const gccnmf_ll_config* cfg, void* state, size_t state_bytes, int hops, float* in, float* out,
                           const float* in_host, float* out_host, void** graph_exec, void* stream) {
  GCCNMF_ENTER(h);
  GCCNMF_REQUIRE(h, graph_exec != nullptr && stream != nullptr, "ll_graph_create: needs a non-default stream and an output slot");
  *graph_exec = nullptr;
  LL_CARVE_OR_FAIL(l);
  GCCNMF_REQUIRE(h, hops >= 1 && hops <= l.C, "ll_graph_create: hops must be in [1, %d] (got %d)", l.C, hops);
  GCCNMF_REQUIRE(h, in && out, "ll_graph_create: NULL pointer");
  if (int st = gccnmf_get_twiddles(h, l.N, nullptr, nullptr)) return st;
  cudaStream_t s = (cudaStream_t)stream;
  const size_t bytes = (size_t)l.S * 2 * hops * l.hop * sizeof(float);
  GCCNMF_CHECK_CUDA(h, cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
  int st = GCCNMF_OK;
  if (in_host && cudaMemcpyAsync(in, in_host, bytes, cudaMemcpyHostToDevice, s) != cudaSuccess) st = GCCNMF_ERR_CUDA;
  if (st == GCCNMF_OK) st = ll_enqueue(h, cfg, l, hops, in, out, stream);
  if (st == GCCNMF_OK && out_host && cudaMemcpyAsync(out_host, out, bytes, cudaMemcpyDeviceToHost, s) != cudaSuccess) st = GCCNMF_ERR_CUDA;
  cudaGraph_t graph = nullptr;
  const cudaError_t end = cudaStreamEndCapture(s, &graph);
  if (st != GCCNMF_OK || end != cudaSuccess) {
    if (graph) cudaGraphDestroy(graph);
    if (st == GCCNMF_OK) return gccnmf_fail(h, GCCNMF_ERR_CUDA, "ll_graph_create: stream capture failed: %s", cudaGetErrorString(end));
    return st;
  }
  cudaGraphExec_t exec = nullptr;
  const cudaError_t inst = cudaGraphInstantiate(&exec, graph, 0);
  cudaGraphDestroy(graph);
  if (inst != cudaSuccess) return gccnmf_fail(h, GCCNMF_ERR_CUDA, "ll_graph_create: cudaGraphInstantiate failed: %s", cudaGetErrorString(inst));
  *graph_exec = exec;
  return GCCNMF_OK;
}

int gccnmf_ll_export(gccnmf_handle* h, const gccnmf_ll_config* cfg, void* state, size_t state_bytes, int hops, int what, void* dst, void* stream) {
  GCCNMF_ENTER(h);
  LL_CARVE_OR_FAIL(l);
  GCCNMF_REQUIRE(h, dst != nullptr, "ll_export: NULL destination");
  GCCNMF_REQUIRE(h, hops >= 1 && hops <= l.C, "ll_export: hops must be in [1, %d] (got %d)", l.C, hops);
  const bool inf = cfg->inference_iterations > 0;
  const size_t T = (size_t)l.S * hops, F = l.F, K = l.K, D = l.D;
  const void* src = nullptr;
  size_t bytes = 0;
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
  if (!src) return gccnmf_fail(h, GCCNMF_ERR_INVALID_ARGUMENT, "ll_export: unknown item %d", what);
  GCCNMF_CHECK_CUDA(h, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDefault, (cudaStream_t)stream));
  return GCCNMF_OK;
}

}  // extern "C"
