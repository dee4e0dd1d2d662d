// GCC-PHAT localisation and GCC-NMF masking kernels.
//   phat_angspec       runGCCNMF.py:44 + gccNMFFunctions.py:85-92      (a3, a4)
//   tdoa_gccnmf        gccNMFFunctions.py:118-135; offlineSpeechEnhancement.ipynb:444-450; online :422  (a6, a10, a11)
//   target_gccnmf      gccNMFFunctions.py:118-135 at P targets that change per frame (the low-latency path's sources)
//   coeff_mask         gccNMFFunctions.py:137-143                        (a7)
//   argmax_mask        offlineSpeechEnhancement.ipynb:466-472            (a10 mask)
//   masked_recon_phase gccNMFFunctions.py:145-151                        (a8)
// Contractions that the reference evaluates in complex128 / float64 are accumulated in float64 here
// so that the integer decisions taken on them (peak picking, argmax over TDOA) are the reference's.
#include "common.cuh"
#include "gemm_simt.cuh"

namespace {

// ------------------------------------------------------------------ a3 + a4: coherence + angular spectrogram
constexpr int kAngT = 16;     // frames per CTA
constexpr int kAngWarps = 4;  // warps per CTA: each takes a quarter of the staged bins (partial sums added in warp order at the end)
constexpr int kAngMaxD = 128;

// X0 * conj(X1) / |X0| / |X1|  (runGCCNMF.py:44) by a fixed float32 formula: re = rn(rn(ax bx) + rn(ay by)),
// im = rn(rn(ay bx) - rn(ax by)) with every product rounded on its own (no FMA contraction), magnitudes
// float32(sqrt(double re^2 + double im^2)) (correctly rounded), then two multiplications by float32
// reciprocals (numpy divides a complex by a real magnitude that way).  This is not numpy's bits: numpy's
// complex64 product contracts one product of each part into an FMA and its abs() is not correctly
// rounded, both depending on the host's SIMD path; on an AVX-512 host about a third of the values are
// bit-equal and the largest difference is 8 * 2^-24 (oracle/offline_exact.py pins this formula bit for bit).
__device__ __forceinline__ float2 phat_coherence(float2 a, float2 b) {
  float re = __fadd_rn(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y));
  float im = __fsub_rn(__fmul_rn(a.y, b.x), __fmul_rn(a.x, b.y));
  const float ma = (float)sqrt((double)a.x * a.x + (double)a.y * a.y);
  const float mb = (float)sqrt((double)b.x * b.x + (double)b.y * b.y);
  const float ia = 1.0f / ma, ib = 1.0f / mb;
  re = __fmul_rn(re, ia); im = __fmul_rn(im, ia);
  re = __fmul_rn(re, ib); im = __fmul_rn(im, ib);
  return float2{re, im};
}

// CTA = 16 frames x all TDOAs, 4 warps.  A lane owns the TDOAs lane, lane + 32, ... (DPL of them) for ALL 16 frames of the tile:
// per staged bin it reads its DPL steering values once and then one broadcast coherence value per frame, i.e. 2 DPL float64 FMAs
// per shared-memory wavefront -- the previous layout (lane = frame, one broadcast E value per FMA pair) spent 6 wavefronts per 4 FMA
// instructions.  The four warps split the bins of every staged chunk; their partial sums are added in warp order at the end
// (deterministic).  The global loads of chunk i + 1 (spectrogram pair, steering rows) are issued into registers before chunk i is
// consumed: with one CTA of 4 warps per SM the un-overlapped load latency of 33-65 chunks was most of the kernel's time.
// Every CTA also writes the coherence of its frames.
template <int DPL, int BF>
__global__ void __launch_bounds__(kAngWarps * 32)
phat_angspec_kernel(const float2* __restrict__ X, int F, int T, int x_is_coherence, const double2* __restrict__ E, int D,
                    float2* __restrict__ coherence, double* __restrict__ angular, double* __restrict__ tile_sums) {
  constexpr int kThreads = kAngWarps * 32;
  constexpr int kCPerThread = BF * kAngT / kThreads;           // coherence values a thread stages per chunk
  constexpr int kEPerThread = BF * 32 * DPL / kThreads;         // steering values a thread stages per chunk (D <= 32 DPL)
  static_assert(BF * kAngT % kThreads == 0 && BF % kAngWarps == 0, "chunk shape");
  __shared__ double2 Cs[BF][kAngT];
  __shared__ double2 Es[(BF > kAngT / 2 ? BF : kAngT / 2)][32 * DPL];   // reused as the reduction buffer red[kAngT][32 DPL] (doubles) at the end
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int t0 = blockIdx.x * kAngT;
  const bool accumulate = angular != nullptr || tile_sums != nullptr;
  double acc[kAngT][DPL];
#pragma unroll
  for (int tt = 0; tt < kAngT; ++tt)
#pragma unroll
    for (int j = 0; j < DPL; ++j) acc[tt][j] = 0.0;

  float2 xa[kCPerThread], xb[kCPerThread];
  double2 er[kEPerThread];
  auto fetch = [&](int f0) {
#pragma unroll
    for (int q = 0; q < kCPerThread; ++q) {
      const int e = threadIdx.x + q * kThreads, f = f0 + e / kAngT, t = t0 + e % kAngT;
      xa[q] = xb[q] = float2{0.f, 0.f};
      if (f < F && t < T) {
        xa[q] = X[(int64_t)f * T + t];
        if (!x_is_coherence) xb[q] = X[((int64_t)F + f) * T + t];
      }
    }
    if (accumulate) {
#pragma unroll
      for (int q = 0; q < kEPerThread; ++q) {
        const int e = threadIdx.x + q * kThreads, ff = e / (32 * DPL), d = e % (32 * DPL);
        er[q] = (f0 + ff < F && d < D) ? E[(int64_t)(f0 + ff) * D + d] : double2{0.0, 0.0};
      }
    }
  };
  auto stash = [&](int f0) {
#pragma unroll
    for (int q = 0; q < kCPerThread; ++q) {
      const int e = threadIdx.x + q * kThreads, ff = e / kAngT, tt = e % kAngT;
      const int f = f0 + ff, t = t0 + tt;
      double2 c = double2{0.0, 0.0};
      if (f < F && t < T) {
        const float2 coh = x_is_coherence ? xa[q] : phat_coherence(xa[q], xb[q]);
        if (coherence) coherence[(int64_t)f * T + t] = coh;
        c = double2{(double)coh.x, (double)coh.y};
      }
      Cs[ff][tt] = c;
    }
    if (accumulate) {
#pragma unroll
      for (int q = 0; q < kEPerThread; ++q) {
        const int e = threadIdx.x + q * kThreads;
        Es[e / (32 * DPL)][e % (32 * DPL)] = er[q];
      }
    }
  };

  fetch(0);
  for (int f0 = 0; f0 < F; f0 += BF) {
    stash(f0);
    __syncthreads();
    if (f0 + BF < F) fetch(f0 + BF);
    if (accumulate) {
#pragma unroll
      for (int i = 0; i < BF / kAngWarps; ++i) {
        const int ff = w + kAngWarps * i;
        double2 e[DPL];
#pragma unroll
        for (int j = 0; j < DPL; ++j) e[j] = Es[ff][lane + 32 * j];
#pragma unroll
        for (int tt = 0; tt < kAngT; ++tt) {
          const double2 c = Cs[ff][tt];
#pragma unroll
          for (int j = 0; j < DPL; ++j) acc[tt][j] += c.x * e[j].x - c.y * e[j].y;   // Re(C * E)
        }
      }
    }
    __syncthreads();
  }
  if (!accumulate) return;
  double (*red)[32 * DPL] = reinterpret_cast<double (*)[32 * DPL]>(&Es[0][0]);
  for (int r = 0; r < kAngWarps; ++r) {
    if (w == r) {
#pragma unroll
      for (int tt = 0; tt < kAngT; ++tt)
#pragma unroll
        for (int j = 0; j < DPL; ++j) {
          const int d = lane + 32 * j;
          red[tt][d] = r == 0 ? acc[tt][j] : red[tt][d] + acc[tt][j];
        }
    }
    __syncthreads();
  }
  const int t_valid = min(kAngT, T - t0);
  if (angular)
    for (int e = threadIdx.x; e < kAngT * D; e += blockDim.x) {
      const int d = e / kAngT, tt = e % kAngT;
      if (tt < t_valid) angular[(int64_t)d * T + t0 + tt] = red[tt][d];
    }
  if (tile_sums)
    for (int d = threadIdx.x; d < D; d += blockDim.x) {
      double sum = 0.0;
      for (int tt = 0; tt < t_valid; ++tt) sum += red[tt][d];
      tile_sums[(int64_t)blockIdx.x * D + d] = sum;
    }
}

// phat_angspec_kernel for a steering bank (gccnmf_llbank_*): a CTA takes 16 columns of one entry in sorted order (steer_tile), so
// it stages one table's rows as the plain kernel stages E, and every column's sums are the plain kernel's, term for term and in the
// same order.  Always a spectrogram pair in, coherence and angular spectrum out.
template <int DPL, int BF>
__global__ void __launch_bounds__(kAngWarps * 32)
phat_angspec_bank_kernel(const float2* __restrict__ X, int F, int T, SteerBank bank, int D, float2* __restrict__ coherence,
                         double* __restrict__ angular) {
  constexpr int kThreads = kAngWarps * 32;
  constexpr int kCPerThread = BF * kAngT / kThreads;
  constexpr int kEPerThread = BF * 32 * DPL / kThreads;
  static_assert(BF * kAngT % kThreads == 0 && BF % kAngWarps == 0, "chunk shape");
  __shared__ double2 Cs[BF][kAngT];
  __shared__ double2 Es[(BF > kAngT / 2 ? BF : kAngT / 2)][32 * DPL];
  __shared__ int col_s[kAngT];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int u0, u1;
  const int entry = steer_tile(bank, kAngT, blockIdx.x, u0, u1);
  if (entry < 0) return;
  if (threadIdx.x < kAngT) col_s[threadIdx.x] = u0 + (int)threadIdx.x < u1 ? bank.column(u0 + threadIdx.x) : -1;
  __syncthreads();
  const double2* __restrict__ E = bank.E + (int64_t)entry * F * D;
  double acc[kAngT][DPL];
#pragma unroll
  for (int tt = 0; tt < kAngT; ++tt)
#pragma unroll
    for (int j = 0; j < DPL; ++j) acc[tt][j] = 0.0;

  float2 xa[kCPerThread], xb[kCPerThread];
  double2 er[kEPerThread];
  auto fetch = [&](int f0) {
#pragma unroll
    for (int q = 0; q < kCPerThread; ++q) {
      const int e = threadIdx.x + q * kThreads, f = f0 + e / kAngT, t = col_s[e % kAngT];
      xa[q] = xb[q] = float2{0.f, 0.f};
      if (f < F && t >= 0) {
        xa[q] = X[(int64_t)f * T + t];
        xb[q] = X[((int64_t)F + f) * T + t];
      }
    }
#pragma unroll
    for (int q = 0; q < kEPerThread; ++q) {
      const int e = threadIdx.x + q * kThreads, ff = e / (32 * DPL), d = e % (32 * DPL);
      er[q] = (f0 + ff < F && d < D) ? E[(int64_t)(f0 + ff) * D + d] : double2{0.0, 0.0};
    }
  };
  auto stash = [&](int f0) {
#pragma unroll
    for (int q = 0; q < kCPerThread; ++q) {
      const int e = threadIdx.x + q * kThreads, ff = e / kAngT, tt = e % kAngT;
      const int f = f0 + ff, t = col_s[tt];
      double2 c = double2{0.0, 0.0};
      if (f < F && t >= 0) {
        const float2 coh = phat_coherence(xa[q], xb[q]);
        coherence[(int64_t)f * T + t] = coh;
        c = double2{(double)coh.x, (double)coh.y};
      }
      Cs[ff][tt] = c;
    }
#pragma unroll
    for (int q = 0; q < kEPerThread; ++q) {
      const int e = threadIdx.x + q * kThreads;
      Es[e / (32 * DPL)][e % (32 * DPL)] = er[q];
    }
  };

  fetch(0);
  for (int f0 = 0; f0 < F; f0 += BF) {
    stash(f0);
    __syncthreads();
    if (f0 + BF < F) fetch(f0 + BF);
#pragma unroll
    for (int i = 0; i < BF / kAngWarps; ++i) {
      const int ff = w + kAngWarps * i;
      double2 e[DPL];
#pragma unroll
      for (int j = 0; j < DPL; ++j) e[j] = Es[ff][lane + 32 * j];
#pragma unroll
      for (int tt = 0; tt < kAngT; ++tt) {
        const double2 c = Cs[ff][tt];
#pragma unroll
        for (int j = 0; j < DPL; ++j) acc[tt][j] += c.x * e[j].x - c.y * e[j].y;   // Re(C * E)
      }
    }
    __syncthreads();
  }
  double (*red)[32 * DPL] = reinterpret_cast<double (*)[32 * DPL]>(&Es[0][0]);
  for (int r = 0; r < kAngWarps; ++r) {
    if (w == r) {
#pragma unroll
      for (int tt = 0; tt < kAngT; ++tt)
#pragma unroll
        for (int j = 0; j < DPL; ++j) {
          const int d = lane + 32 * j;
          red[tt][d] = r == 0 ? acc[tt][j] : red[tt][d] + acc[tt][j];
        }
    }
    __syncthreads();
  }
  for (int e = threadIdx.x; e < kAngT * D; e += blockDim.x) {
    const int d = e / kAngT, tt = e % kAngT;
    if (col_s[tt] >= 0) angular[(int64_t)d * T + col_s[tt]] = red[tt][d];
  }
}

__global__ void mean_tiles_kernel(const double* __restrict__ tile_sums, int tiles, int D, int T, double* __restrict__ mean) {
  const int d = blockIdx.x * blockDim.x + threadIdx.x;
  if (d >= D) return;
  double s = 0.0;
  for (int i = 0; i < tiles; ++i) s += tile_sums[(int64_t)i * D + d];
  mean[d] = s / (double)T;
}

// ------------------------------------------------------------------ a6 / a10 / a11: GCC-NMF per TDOA (float64 GEMM)
constexpr int GM = 128, GN = 128, GK = 8, GTM = 8, GTN = 8;
constexpr int kGccThreads = (GM / GTM) * (GN / GTN);

struct LoadWAtoms {  // A(m = atom, k = f) = W[f][atom]
  static constexpr bool kContigK = false;
  const float* W; int K, F;
  __device__ double operator()(int m, int f) const { return (m < K && f < F) ? (double)__ldg(W + (int64_t)f * K + m) : 0.0; }
};
// Re(c * e) of a coherence value and a steering value, the B operand of every GCC-NMF contraction.  One function for all the
// loaders below, so that the compiler cannot contract the expression differently in one of them: a target value then has the
// bits of the all-TDOA value at the same (TDOA, atom, frame).
__device__ __forceinline__ double re_coh_steer(float2 c, double2 e) { return (double)c.x * e.x - (double)c.y * e.y; }

struct LoadRealGCC {  // B(n = t * D + d, k = f) = Re(coherence[f][t] * E[f][d])
  static constexpr bool kContigK = false;
  const float2* coh; const double2* E; int F, T, D, N;
  __device__ double operator()(int n, int f) const {
    if (n >= N || f >= F) return 0.0;
    const int t = n / D, d = n - t * D;
    return re_coh_steer(__ldg(coh + (int64_t)f * T + t), __ldg(E + (int64_t)f * D + d));
  }
};
struct LoadTargetGCC {  // B(n = t * P + q, k = f) = Re(coherence[f][t] * E[f][targets[t * P + q]]): P targets per frame
  static constexpr bool kContigK = false;
  const float2* coh; const double2* E; const int32_t* targets; int F, T, D, P, N;
  __device__ double operator()(int n, int f) const {
    if (n >= N || f >= F) return 0.0;
    const int t = n / P;
    return re_coh_steer(__ldg(coh + (int64_t)f * T + t), __ldg(E + (int64_t)f * D + __ldg(targets + n)));
  }
};

// The two loaders above for a steering bank: column t reads the table of its stream's entry.
struct LoadRealGCCBank {
  static constexpr bool kContigK = false;
  const float2* coh; SteerBank bank; int F, T, D, N;
  __device__ double operator()(int n, int f) const {
    if (n >= N || f >= F) return 0.0;
    const int t = n / D, d = n - t * D;
    return re_coh_steer(__ldg(coh + (int64_t)f * T + t), __ldg(bank.E + ((int64_t)bank.entry(t) * F + f) * D + d));
  }
};
struct LoadTargetGCCBank {
  static constexpr bool kContigK = false;
  const float2* coh; SteerBank bank; const int32_t* targets; int F, T, D, P, N;
  __device__ double operator()(int n, int f) const {
    if (n >= N || f >= F) return 0.0;
    const int t = n / P;
    return re_coh_steer(__ldg(coh + (int64_t)f * T + t), __ldg(bank.E + ((int64_t)bank.entry(t) * F + f) * D + __ldg(targets + n)));
  }
};

// numpy.argmax ordering: NaN is a maximum, first occurrence wins.
__device__ __forceinline__ bool argmax_better(double v, int i, double bv, int bi) {
  const bool vn = isnan(v), bn = isnan(bv);
  if (vn || bn) return vn && (!bn || i < bi);
  return v > bv || (v == bv && i < bi);
}

template <bool ARGMAX>
__global__ void __launch_bounds__(kGccThreads)
tdoa_gccnmf_kernel(int K, int N, int F, LoadWAtoms aload, LoadRealGCC bload, int T, int D, float* __restrict__ values,
                   int32_t* __restrict__ argmax, const int32_t* __restrict__ gate, int gate_capacity, int32_t* __restrict__ ran) {
  // gated form (the graph-safe fallback of the tensor-core argmax): nothing to do unless its refinement list overflowed
  if (gate) {
    if (*gate <= gate_capacity) return;
    if (ran && blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) *ran = 1;
  }
  double acc[GTM][GTN];
  const int m0 = blockIdx.y * GM, n0 = blockIdx.x * GN;
  gemm_simt_mainloop<double, GM, GN, GK, GTM, GTN>(acc, m0, n0, F, aload, bload);
  constexpr int TX = GN / GTN;
  if (values) {
#pragma unroll
    for (int i = 0; i < GTM; ++i) {
      const int m = gemm_row<GM, GTM, TX>(m0, i);
      if (m >= K) continue;
#pragma unroll
      for (int j = 0; j < GTN; ++j) {
        const int n = gemm_col<GN, GTN, TX>(n0, j);
        if (n >= N) continue;
        const int t = n / D, d = n - t * D;
        values[((int64_t)d * K + m) * T + t] = (float)acc[i][j];
      }
    }
  }
  if (ARGMAX) {
    // D is a power of two in [4, 128] and divides GN, so n0 % D == 0 and every 4-column half-row of the
    // register tile lies inside one frame.  D <= 64: a frame spans D/4 consecutive lanes of one half;
    // D == 128: a frame is the whole tile row (both halves of all 16 lanes).
    const int tx = threadIdx.x % TX;
    const int lanes = min(D / 4, TX);
#pragma unroll
    for (int i = 0; i < GTM; ++i) {
      const int m = gemm_row<GM, GTM, TX>(m0, i);
      double bv[2];
      int bi[2];
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        const int d0 = (half * (GN / 2) + tx * (GTN / 2)) % D;  // TDOA index of this half-row's first column
        bv[half] = acc[i][half * (GTN / 2)];
        bi[half] = d0;
#pragma unroll
        for (int j = 1; j < GTN / 2; ++j) {
          const double v = acc[i][half * (GTN / 2) + j];
          if (argmax_better(v, d0 + j, bv[half], bi[half])) { bv[half] = v; bi[half] = d0 + j; }
        }
      }
      if (D == GN) {  // one frame per tile row: fold half 1 into half 0 before the lane reduction
        if (argmax_better(bv[1], bi[1], bv[0], bi[0])) { bv[0] = bv[1]; bi[0] = bi[1]; }
      }
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        if (D == GN && half == 1) break;
        for (int o = 1; o < lanes; o <<= 1) {
          const double ov = __shfl_xor_sync(0xffffffffu, bv[half], o);
          const int oi = __shfl_xor_sync(0xffffffffu, bi[half], o);
          if (argmax_better(ov, oi, bv[half], bi[half])) { bv[half] = ov; bi[half] = oi; }
        }
        const int n_first = n0 + half * (GN / 2) + tx * (GTN / 2);
        if ((tx % lanes) == 0 && m < K && n_first < N) argmax[(int64_t)m * T + n_first / D] = bi[half];
      }
    }
  }
}

// getTargetTDOAGCCNMFs with P targets per frame: values (P, K, T) f32, values[q][k][t] = float32(sum_f W[f][k] Re(coh[f][t] E[f][tau])),
// tau = targets[t P + q].  The same main loop as tdoa_gccnmf_kernel (an fma chain over f from 0 per output), so every value has the
// bits of the all-TDOA value at (tau, k, t).  BN = 32 is the narrow column tile for small T P; it changes no sum.
template <int BN, int TN>
__global__ void __launch_bounds__((GM / GTM) * (BN / TN))
target_gccnmf_kernel(int K, int N, int F, LoadWAtoms aload, LoadTargetGCC bload, int T, int P, float* __restrict__ values) {
  double acc[GTM][TN];
  const int m0 = blockIdx.y * GM, n0 = blockIdx.x * BN;
  gemm_simt_mainloop<double, GM, BN, GK, GTM, TN>(acc, m0, n0, F, aload, bload);
  constexpr int TX = BN / TN;
#pragma unroll
  for (int i = 0; i < GTM; ++i) {
    const int m = gemm_row<GM, GTM, TX>(m0, i);
    if (m >= K) continue;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      const int n = gemm_col<BN, TN, TX>(n0, j);
      if (n >= N) continue;
      const int t = n / P, q = n - t * P;
      values[((int64_t)q * K + m) * T + t] = (float)acc[i][j];
    }
  }
}

// tdoa_gccnmf_kernel<true> (argmax only, optionally gated) and target_gccnmf_kernel for a steering bank: the same main loop and
// epilogue with LoadRealGCCBank / LoadTargetGCCBank, so a column's values and decisions are the plain kernels' on its table.
__global__ void __launch_bounds__(kGccThreads)
tdoa_argmax_bank_kernel(int K, int N, int F, LoadWAtoms aload, LoadRealGCCBank bload, int T, int D, int32_t* __restrict__ argmax,
                        const int32_t* __restrict__ gate, int gate_capacity, int32_t* __restrict__ ran) {
  if (gate) {
    if (*gate <= gate_capacity) return;
    if (ran && blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) *ran = 1;
  }
  double acc[GTM][GTN];
  const int m0 = blockIdx.y * GM, n0 = blockIdx.x * GN;
  gemm_simt_mainloop<double, GM, GN, GK, GTM, GTN>(acc, m0, n0, F, aload, bload);
  constexpr int TX = GN / GTN;
  const int tx = threadIdx.x % TX;
  const int lanes = min(D / 4, TX);
#pragma unroll
  for (int i = 0; i < GTM; ++i) {
    const int m = gemm_row<GM, GTM, TX>(m0, i);
    double bv[2];
    int bi[2];
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const int d0 = (half * (GN / 2) + tx * (GTN / 2)) % D;
      bv[half] = acc[i][half * (GTN / 2)];
      bi[half] = d0;
#pragma unroll
      for (int j = 1; j < GTN / 2; ++j) {
        const double v = acc[i][half * (GTN / 2) + j];
        if (argmax_better(v, d0 + j, bv[half], bi[half])) { bv[half] = v; bi[half] = d0 + j; }
      }
    }
    if (D == GN) {
      if (argmax_better(bv[1], bi[1], bv[0], bi[0])) { bv[0] = bv[1]; bi[0] = bi[1]; }
    }
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      if (D == GN && half == 1) break;
      for (int o = 1; o < lanes; o <<= 1) {
        const double ov = __shfl_xor_sync(0xffffffffu, bv[half], o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi[half], o);
        if (argmax_better(ov, oi, bv[half], bi[half])) { bv[half] = ov; bi[half] = oi; }
      }
      const int n_first = n0 + half * (GN / 2) + tx * (GTN / 2);
      if ((tx % lanes) == 0 && m < K && n_first < N) argmax[(int64_t)m * T + n_first / D] = bi[half];
    }
  }
}

template <int BN, int TN>
__global__ void __launch_bounds__((GM / GTM) * (BN / TN))
target_gccnmf_bank_kernel(int K, int N, int F, LoadWAtoms aload, LoadTargetGCCBank bload, int T, int P, float* __restrict__ values) {
  double acc[GTM][TN];
  const int m0 = blockIdx.y * GM, n0 = blockIdx.x * BN;
  gemm_simt_mainloop<double, GM, BN, GK, GTM, TN>(acc, m0, n0, F, aload, bload);
  constexpr int TX = BN / TN;
#pragma unroll
  for (int i = 0; i < GTM; ++i) {
    const int m = gemm_row<GM, GTM, TX>(m0, i);
    if (m >= K) continue;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      const int n = gemm_col<BN, TN, TX>(n0, j);
      if (n >= N) continue;
      const int t = n / P, q = n - t * P;
      values[((int64_t)q * K + m) * T + t] = (float)acc[i][j];
    }
  }
}

// ------------------------------------------------------------------ a7: masks
__global__ void coeff_mask_kernel(const float* __restrict__ G, int S, int64_t KT, float* __restrict__ masks, int32_t* all_nan_flag) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= KT) return;
  // numpy.nanargmax: NaN is replaced by -inf, then the first maximum wins (so a NaN before -inf is chosen over it); a column
  // that is all NaN raises in numpy: here it sets the flag and gets no source
  int best = 0;
  float bv = -INFINITY;
  bool any = false;
  for (int s = 0; s < S; ++s) {
    const float v = G[(int64_t)s * KT + i];
    if (isnan(v)) continue;
    any = true;
    if (v > bv) { best = s; bv = v; }
  }
  if (!any) {
    best = -1;
    if (all_nan_flag) *all_nan_flag = 1;
  }
  for (int s = 0; s < S; ++s) masks[(int64_t)s * KT + i] = (s == best) ? 1.f : 0.f;
}

__global__ void argmax_mask_kernel(const int32_t* __restrict__ argmax, int64_t KT, const uint8_t* __restrict__ lut, int D, float* __restrict__ mask) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= KT) return;
  const int a = argmax[i];
  mask[i] = (a >= 0 && a < D && lut[a]) ? 1.f : 0.f;
}

// ------------------------------------------------------------------ a8: masked reconstruction with mixture phase
constexpr int RM = 128, RN = 128, RK = 16, RTM = 8, RTN = 8;
constexpr int kReconThreads = (RM / RTM) * (RN / RTN);

struct LoadWRows {  // A(m = f, k = atom) = W[f][atom]
  static constexpr bool kContigK = true;
  const float* W; int F, K;
  __device__ float operator()(int m, int k) const { return (m < F && k < K) ? __ldg(W + (int64_t)m * K + k) : 0.f; }
};
struct LoadMaskedH {  // B(n = t, k = atom) = H[atom][c*T + t] * mask[atom][t]   (gccNMFFunctions.py:150)
  static constexpr bool kContigK = false;
  const float* H; const float* mask; int K, T; int64_t ldh;
  __device__ float operator()(int n, int k) const {
    return (n < T && k < K) ? __ldg(H + (int64_t)k * ldh + n) * __ldg(mask + (int64_t)k * T + n) : 0.f;
  }
};

__global__ void __launch_bounds__(kReconThreads, 2)
masked_recon_kernel(const float* __restrict__ masks, const float2* __restrict__ X, const float* __restrict__ W,
                    const float* __restrict__ H, int F, int T, int K, float2* __restrict__ out) {
  const int s = blockIdx.z / 2, c = blockIdx.z % 2;
  float acc[RTM][RTN];
  const int m0 = blockIdx.y * RM, n0 = blockIdx.x * RN;
  LoadWRows a{W, F, K};
  LoadMaskedH b{H + (int64_t)c * T, masks + (int64_t)s * K * T, K, T, (int64_t)2 * T};
  gemm_simt_mainloop<float, RM, RN, RK, RTM, RTN>(acc, m0, n0, K, a, b);
  const float2* Xc = X + (int64_t)c * F * T;
  float2* o = out + ((int64_t)s * 2 + c) * F * T;
#pragma unroll
  for (int i = 0; i < RTM; ++i) {
    const int m = gemm_row<RM, RTM, RN / RTN>(m0, i);
    if (m >= F) continue;
#pragma unroll
    for (int j = 0; j < RTN; ++j) {
      const int n = gemm_col<RN, RTN, RN / RTN>(n0, j);
      if (n >= T) continue;
      // exp(1j * angle(X)) (gccNMFFunctions.py:151): unit phasor of the mixture bin; angle(0) = 0.
      const float2 x = Xc[(int64_t)m * T + n];
      const double mag = sqrt((double)x.x * x.x + (double)x.y * x.y);
      float pr = 1.f, pi = 0.f;
      if (mag > 0.0) { pr = (float)((double)x.x / mag); pi = (float)((double)x.y / mag); }
      else if (mag != mag) { pr = pi = __int_as_float(0x7fc00000); }
      o[(int64_t)m * T + n] = float2{acc[i][j] * pr, acc[i][j] * pi};
    }
  }
}

// ------------------------------------------------------------------ a11 / a13: online localisation, atom masks, Wiener-like filter
// acc[tau] = max over frames <= t of A[tau, t'] (onlineSpeechEnhancement.ipynb:416); one thread per TDOA scans time.
__global__ void cummax_time_kernel(const double* __restrict__ A, int D, int T, double* __restrict__ acc) {
  const int d = blockIdx.x * blockDim.x + threadIdx.x;
  if (d >= D) return;
  double m = -INFINITY;
  for (int t = 0; t < T; ++t) {
    const double v = A[(int64_t)d * T + t];
    if (v > m || v != v) m = v;          // numpy.max: NaN propagates (and then sticks: comparisons with NaN are false)
    acc[(int64_t)d * T + t] = m;
  }
}
// target[t] = argmax over TDOA of acc[:, t] (:417), numpy.argmax semantics.
__global__ void argmax_tdoa_kernel(const double* __restrict__ acc, int D, int T, int32_t* __restrict__ target) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T) return;
  double bv = acc[t];
  int bi = 0;
  for (int d = 1; d < D; ++d) {
    const double v = acc[(int64_t)d * T + t];
    if (argmax_better(v, d, bv, bi)) { bv = v; bi = d; }
  }
  target[t] = bi;
}

// mode 0 (boxcar): |argmax - target| < eps -> 1 else 0      (onlineSpeechEnhancement.ipynb:423-425; gccNMFProcessor.py:263)
// mode 1 (window): exp(-(|argmax - target| / eps)^beta) / (1 + floor) + floor     (gccNMFProcessor.py:265)
__global__ void atom_mask_kernel(const int32_t* __restrict__ argmax, int K, int T, const int32_t* __restrict__ target, int target_stride,
                                 float target_scalar, float eps, int mode, float beta, float noise_floor, float* __restrict__ mask) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)K * T) return;
  const int t = (int)(i % T);
  const float mu = target ? (float)target[(int64_t)t * target_stride] : target_scalar;
  const float dist = fabsf((float)argmax[i] - mu);
  float m;
  if (mode == 0) m = dist < eps ? 1.f : 0.f;
  else m = expf(-powf(dist / eps, beta)) / (1.f + noise_floor) + noise_floor;
  mask[i] = m;
}

__global__ void rowsum_w_kernel(const float* __restrict__ W, int F, int K, float* __restrict__ rowsum) {
  const int f = blockIdx.x;
  __shared__ float ws[32];
  float s = 0.f;
  for (int k = threadIdx.x; k < K; k += blockDim.x) s += W[(int64_t)f * K + k];
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    s = threadIdx.x < (blockDim.x >> 5) ? ws[threadIdx.x] : 0.f;
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (threadIdx.x == 0) rowsum[f] = s;
  }
}

struct LoadMaskT {  // B(n = t, k = atom) = mask[atom][t]
  static constexpr bool kContigK = false;
  const float* mask; int K, T;
  __device__ float operator()(int n, int k) const { return (n < T && k < K) ? __ldg(mask + (int64_t)k * T + n) : 0.f; }
};

// Y[c] = ((W . mask) / rowsum(W)) * X[c]     (onlineSpeechEnhancement.ipynb:429-431,440; gccNMFProcessor.py:267-269,209)
__global__ void __launch_bounds__(kReconThreads, 2)
wiener_apply_kernel(const float* __restrict__ mask, const float* __restrict__ W, const float* __restrict__ rowsumW,
                    const float2* __restrict__ X, int F, int T, int K, float2* __restrict__ Y, float* __restrict__ wiener) {
  float acc[RTM][RTN];
  const int m0 = blockIdx.y * RM, n0 = blockIdx.x * RN;
  LoadWRows a{W, F, K};
  LoadMaskT b{mask, K, T};
  gemm_simt_mainloop<float, RM, RN, RK, RTM, RTN>(acc, m0, n0, K, a, b);
#pragma unroll
  for (int i = 0; i < RTM; ++i) {
    const int m = gemm_row<RM, RTM, RN / RTN>(m0, i);
    if (m >= F) continue;
    const float rs = rowsumW[m];
#pragma unroll
    for (int j = 0; j < RTN; ++j) {
      const int n = gemm_col<RN, RTN, RN / RTN>(n0, j);
      if (n >= T) continue;
      const float w = acc[i][j] / rs;
      if (wiener) wiener[(int64_t)m * T + n] = w;
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const float2 x = X[((int64_t)c * F + m) * T + n];
        Y[((int64_t)c * F + m) * T + n] = float2{w * x.x, w * x.y};
      }
    }
  }
}

struct LoadHMaybeMasked {  // B(n = t, k = atom) = H[atom][c*T + t] (* mask[atom][t] when mask != NULL)
  static constexpr bool kContigK = false;
  const float* H; const float* mask; int K, T; int64_t ldh;
  __device__ float operator()(int n, int k) const {
    if (n >= T || k >= K) return 0.f;
    const float hv = __ldg(H + (int64_t)k * ldh + n);
    return mask ? hv * __ldg(mask + (int64_t)k * T + n) : hv;
  }
};

// Wiener-like filter with inferred coefficients (onlineSpeechEnhancement.ipynb:435-440), per channel c = blockIdx.z:
//   wiener[c] = (W . (H_c * mask)) / (W . H_c);   Y[c] = wiener[c] * X[c]          H (K, 2T), column c T + t
__global__ void __launch_bounds__(kReconThreads, 2)
wiener_apply_h_kernel(const float* __restrict__ mask, const float* __restrict__ W, const float* __restrict__ H, const float2* __restrict__ X,
                      int F, int T, int K, float2* __restrict__ Y, float* __restrict__ wiener) {
  const int c = blockIdx.z;
  float num[RTM][RTN], den[RTM][RTN];
  const int m0 = blockIdx.y * RM, n0 = blockIdx.x * RN;
  LoadWRows a{W, F, K};
  LoadHMaybeMasked masked{H + (int64_t)c * T, mask, K, T, (int64_t)2 * T}, plain{H + (int64_t)c * T, nullptr, K, T, (int64_t)2 * T};
  gemm_simt_mainloop<float, RM, RN, RK, RTM, RTN>(num, m0, n0, K, a, masked);
  gemm_simt_mainloop<float, RM, RN, RK, RTM, RTN>(den, m0, n0, K, a, plain);
#pragma unroll
  for (int i = 0; i < RTM; ++i) {
    const int m = gemm_row<RM, RTM, RN / RTN>(m0, i);
    if (m >= F) continue;
#pragma unroll
    for (int j = 0; j < RTN; ++j) {
      const int n = gemm_col<RN, RTN, RN / RTN>(n0, j);
      if (n >= T) continue;
      const float w = num[i][j] / den[i][j];
      const int64_t o = ((int64_t)c * F + m) * T + n;
      if (wiener) wiener[o] = w;
      const float2 x = X[o];
      Y[o] = float2{w * x.x, w * x.y};
    }
  }
}

bool is_pow2(int x) { return x > 0 && (x & (x - 1)) == 0; }

}  // namespace

// gcc_tc.cu
bool gccnmf_masked_recon_tc_supported(int S, int F, int T, int K);
extern "C" int gccnmf_masked_recon_planes(gccnmf_handle* h, const float* masks, const float* X, const float* W, const float* H, int S, int F, int T,
                                          int K, float* out, void* workspace, size_t workspace_bytes, void* stream);

extern "C" {

size_t gccnmf_phat_angspec_workspace_bytes(int F, int T, int D) {
  (void)F;
  if (T <= 0 || D <= 0) return 0;
  return align_up((size_t)((T + kAngT - 1) / kAngT) * D * sizeof(double), 256);
}

int gccnmf_phat_angspec(gccnmf_handle* h, const float* X, int F, int T, int x_is_coherence, const double* expJOmegaTau, int D, float* coherence,
                        double* angular, double* mean_angular, void* workspace, size_t workspace_bytes, void* stream) {
  GCCNMF_ENTER(h);
  GCCNMF_REQUIRE(h, F > 0 && T > 0, "phat_angspec: F and T must be positive");
  GCCNMF_REQUIRE(h, X != nullptr, "phat_angspec: NULL spectrogram");
  const bool need_ang = angular || mean_angular;
  if (need_ang) {
    GCCNMF_REQUIRE(h, expJOmegaTau != nullptr && D > 0, "phat_angspec: TDOA table required");
    if (D > kAngMaxD) return gccnmf_fail(h, GCCNMF_ERR_UNSUPPORTED, "phat_angspec: numTDOAs %d > %d", D, kAngMaxD);
  }
  double* tile_sums = nullptr;
  const int tiles = (T + kAngT - 1) / kAngT;
  if (mean_angular) {
    if (!workspace || workspace_bytes < gccnmf_phat_angspec_workspace_bytes(F, T, D))
      return gccnmf_fail(h, GCCNMF_ERR_WORKSPACE, "phat_angspec workspace too small");
    tile_sums = static_cast<double*>(workspace);
  }
  const int Dk = need_ang ? D : 0;
  const float2* Xc = reinterpret_cast<const float2*>(X);
  const double2* Ec = reinterpret_cast<const double2*>(expJOmegaTau);
  float2* Cc = reinterpret_cast<float2*>(coherence);
  if (Dk <= 32) GCCNMF_LAUNCH(h, (phat_angspec_kernel<1, 32>), tiles, kAngWarps * 32, 0, stream, Xc, F, T, x_is_coherence, Ec, Dk, Cc, angular, tile_sums);
  else if (Dk <= 64) GCCNMF_LAUNCH(h, (phat_angspec_kernel<2, 16>), tiles, kAngWarps * 32, 0, stream, Xc, F, T, x_is_coherence, Ec, Dk, Cc, angular, tile_sums);
  else GCCNMF_LAUNCH(h, (phat_angspec_kernel<4, 8>), tiles, kAngWarps * 32, 0, stream, Xc, F, T, x_is_coherence, Ec, Dk, Cc, angular, tile_sums);
  if (mean_angular) GCCNMF_LAUNCH(h, mean_tiles_kernel, (D + 63) / 64, 64, 0, stream, tile_sums, tiles, D, T, mean_angular);
  return GCCNMF_OK;
}

int gccnmf_tdoa_gccnmf(gccnmf_handle* h, const float* coherence, int F, int T, const double* E, int D, const float* W, int K,
                       float* values, int32_t* argmax, void* stream) {
  GCCNMF_ENTER(h);
  GCCNMF_REQUIRE(h, F > 0 && T > 0 && D > 0 && K > 0, "tdoa_gccnmf: dimensions must be positive");
  GCCNMF_REQUIRE(h, coherence && E && W, "tdoa_gccnmf: NULL pointer");
  GCCNMF_REQUIRE(h, (int64_t)T * D < (int64_t)1 << 31, "tdoa_gccnmf: T * D overflows int32");
  if (!values && !argmax) return GCCNMF_OK;
  if (argmax && !(is_pow2(D) && D >= 4 && D <= GN))
    return gccnmf_fail(h, GCCNMF_ERR_UNSUPPORTED, "tdoa_gccnmf: fused argmax needs numTDOAs a power of two in [4, %d] (got %d)", GN, D);
  const int N = T * D;
  LoadWAtoms a{W, K, F};
  LoadRealGCC b{reinterpret_cast<const float2*>(coherence), reinterpret_cast<const double2*>(E), F, T, D, N};
  dim3 grid((N + GN - 1) / GN, (K + GM - 1) / GM);
  if (argmax) {
    auto k = tdoa_gccnmf_kernel<true>;
    GCCNMF_LAUNCH(h, k, grid, kGccThreads, 0, stream, K, N, F, a, b, T, D, values, argmax, nullptr, 0, nullptr);
  } else {
    auto k = tdoa_gccnmf_kernel<false>;
    GCCNMF_LAUNCH(h, k, grid, kGccThreads, 0, stream, K, N, F, a, b, T, D, values, argmax, nullptr, 0, nullptr);
  }
  return GCCNMF_OK;
}

int gccnmf_coeff_mask(gccnmf_handle* h, const float* gccnmfs, int S, int K, int T, float* masks, int32_t* all_nan_flag, void* stream) {
  GCCNMF_ENTER(h);
  GCCNMF_REQUIRE(h, S > 0 && K > 0 && T > 0 && gccnmfs && masks, "coeff_mask: bad arguments");
  const int64_t KT = (int64_t)K * T;
  GCCNMF_LAUNCH(h, coeff_mask_kernel, (unsigned)((KT + 255) / 256), 256, 0, stream, gccnmfs, S, KT, masks, all_nan_flag);
  return GCCNMF_OK;
}

int gccnmf_argmax_mask(gccnmf_handle* h, const int32_t* argmax, int K, int T, const uint8_t* lut, int D, float* mask, void* stream) {
  GCCNMF_ENTER(h);
  GCCNMF_REQUIRE(h, K > 0 && T > 0 && D > 0 && argmax && lut && mask, "argmax_mask: bad arguments");
  const int64_t KT = (int64_t)K * T;
  GCCNMF_LAUNCH(h, argmax_mask_kernel, (unsigned)((KT + 255) / 256), 256, 0, stream, argmax, KT, lut, D, mask);
  return GCCNMF_OK;
}

int gccnmf_masked_recon_phase(gccnmf_handle* h, const float* masks, const float* X, const float* W, const float* H, int S, int F,
                              int T, int K, float* out, void* workspace, size_t workspace_bytes, void* stream) {
  GCCNMF_ENTER(h);
  GCCNMF_REQUIRE(h, S > 0 && F > 0 && T > 0 && K > 0 && masks && X && W && H && out, "masked_recon_phase: bad arguments");
  // tensor cores (plane GEMM over masked-H planes, gcc_tc.cu) when the caller provides the workspace and the shape is covered;
  // else the float32 SIMT GEMM below
  if (workspace && !h->force_simt_nmf && gccnmf_masked_recon_tc_supported(S, F, T, K))
    return gccnmf_masked_recon_planes(h, masks, X, W, H, S, F, T, K, out, workspace, workspace_bytes, stream);
  dim3 grid((T + RN - 1) / RN, (F + RM - 1) / RM, S * 2);
  GCCNMF_LAUNCH(h, masked_recon_kernel, grid, kReconThreads, 0, stream, masks, reinterpret_cast<const float2*>(X), W, H, F, T, K,
                reinterpret_cast<float2*>(out));
  return GCCNMF_OK;
}

int gccnmf_online_targets(gccnmf_handle* h, const double* angular, int D, int T, double* accumulated_max, int32_t* targets, void* stream) {
  GCCNMF_ENTER(h);
  GCCNMF_REQUIRE(h, angular && accumulated_max && targets && D > 0 && T > 0, "online_targets: bad arguments");
  GCCNMF_LAUNCH(h, cummax_time_kernel, (D + 63) / 64, 64, 0, stream, angular, D, T, accumulated_max);
  GCCNMF_LAUNCH(h, argmax_tdoa_kernel, (T + 127) / 128, 128, 0, stream, accumulated_max, D, T, targets);
  return GCCNMF_OK;
}

int gccnmf_atom_mask(gccnmf_handle* h, const int32_t* argmax, int K, int T, const int32_t* targets, float target_scalar, float epsilon,
                     int mode, float beta, float noise_floor, float* mask, void* stream) {
  GCCNMF_ENTER(h);
  GCCNMF_REQUIRE(h, argmax && mask && K > 0 && T > 0 && (mode == 0 || mode == 1), "atom_mask: bad arguments");
  const int64_t n = (int64_t)K * T;
  GCCNMF_LAUNCH(h, atom_mask_kernel, (unsigned)((n + 255) / 256), 256, 0, stream, argmax, K, T, targets, 1, target_scalar, epsilon, mode,
                beta, noise_floor, mask);
  return GCCNMF_OK;
}

size_t gccnmf_wiener_apply_workspace_bytes(int F) { return F > 0 ? align_up((size_t)F * sizeof(float), 256) : 0; }

int gccnmf_wiener_apply(gccnmf_handle* h, const float* mask, const float* W, const float* X, int F, int T, int K, float* Y,
                        float* wiener, void* workspace, size_t workspace_bytes, void* stream) {
  GCCNMF_ENTER(h);
  GCCNMF_REQUIRE(h, mask && W && X && Y && F > 0 && T > 0 && K > 0, "wiener_apply: bad arguments");
  if (!workspace || workspace_bytes < gccnmf_wiener_apply_workspace_bytes(F)) return gccnmf_fail(h, GCCNMF_ERR_WORKSPACE, "wiener_apply workspace too small");
  float* rowsum = static_cast<float*>(workspace);
  GCCNMF_LAUNCH(h, rowsum_w_kernel, F, 128, 0, stream, W, F, K, rowsum);
  dim3 grid((T + RN - 1) / RN, (F + RM - 1) / RM);
  GCCNMF_LAUNCH(h, wiener_apply_kernel, grid, kReconThreads, 0, stream, mask, W, rowsum, reinterpret_cast<const float2*>(X), F, T, K,
                reinterpret_cast<float2*>(Y), wiener);
  return GCCNMF_OK;
}

// Y (2, F, T) c64 = wiener * X with wiener (2, F, T) f32 = (W . (H_c * mask)) / (W . H_c) per channel (ipynb:435-440):
// the numInferenceIterations > 0 branch; H (K, 2T) holds channel c in columns [c T, (c + 1) T).
int gccnmf_wiener_apply_h(gccnmf_handle* h, const float* mask, const float* W, const float* H, const float* X, int F, int T, int K, float* Y,
                          float* wiener, void* stream) {
  GCCNMF_ENTER(h);
  GCCNMF_REQUIRE(h, mask && W && H && X && Y && F > 0 && T > 0 && K > 0, "wiener_apply_h: bad arguments");
  dim3 grid((T + RN - 1) / RN, (F + RM - 1) / RM, 2);
  GCCNMF_LAUNCH(h, wiener_apply_h_kernel, grid, kReconThreads, 0, stream, mask, W, H, reinterpret_cast<const float2*>(X), F, T, K,
                reinterpret_cast<float2*>(Y), wiener);
  return GCCNMF_OK;
}

}  // extern "C"

// The argmax of gccnmf_tdoa_gccnmf as a launch that reads the refinement count of gccnmf_tdoa_argmax on the device and returns at
// once unless it exceeds `capacity`; then it overwrites every decision with the float64 one and sets *ran = 1.  No host
// synchronisation, so it can follow the tensor-core argmax inside a captured graph.
int gccnmf_tdoa_gccnmf_gated(gccnmf_handle* h, const float* coherence, int F, int T, const double* E, int D, const float* W, int K,
                             int32_t* argmax, const int32_t* gate, int capacity, int32_t* ran, void* stream) {
  GCCNMF_REQUIRE(h, F > 0 && T > 0 && D > 0 && K > 0 && coherence && E && W && argmax && gate, "tdoa_gccnmf_gated: bad arguments");
  GCCNMF_REQUIRE(h, (int64_t)T * D < (int64_t)1 << 31, "tdoa_gccnmf_gated: T * D overflows int32");
  if (!(is_pow2(D) && D >= 4 && D <= GN))
    return gccnmf_fail(h, GCCNMF_ERR_UNSUPPORTED, "tdoa_gccnmf_gated: numTDOAs must be a power of two in [4, %d] (got %d)", GN, D);
  const int N = T * D;
  LoadWAtoms a{W, K, F};
  LoadRealGCC b{reinterpret_cast<const float2*>(coherence), reinterpret_cast<const double2*>(E), F, T, D, N};
  dim3 grid((N + GN - 1) / GN, (K + GM - 1) / GM);
  auto k = tdoa_gccnmf_kernel<true>;
  GCCNMF_LAUNCH(h, k, grid, kGccThreads, 0, stream, K, N, F, a, b, T, D, nullptr, argmax, gate, capacity, ran);
  return GCCNMF_OK;
}

// values (P, K, T) f32 = the float64 GCC-NMF contraction at P target TDOAs per frame, targets (T, P) i32 on the device (each in
// [0, D)).  Bit for bit the values gccnmf_tdoa_gccnmf writes at those (TDOA, atom, frame).  Column tiles of 128, or 32 when the
// wide tiles would leave SMs idle.
int gccnmf_target_gccnmf(gccnmf_handle* h, const float* coherence, int F, int T, const double* E, int D, const float* W, int K,
                         const int32_t* targets, int P, float* values, void* stream) {
  GCCNMF_ENTER(h);
  GCCNMF_REQUIRE(h, F > 0 && T > 0 && D > 0 && K > 0 && P > 0 && coherence && E && W && targets && values, "target_gccnmf: bad arguments");
  GCCNMF_REQUIRE(h, (int64_t)T * P < (int64_t)1 << 31 && (int64_t)P * K * T < (int64_t)1 << 31, "target_gccnmf: T x P or P x K x T overflows int32");
  const int N = T * P;
  LoadWAtoms a{W, K, F};
  LoadTargetGCC b{reinterpret_cast<const float2*>(coherence), reinterpret_cast<const double2*>(E), targets, F, T, D, P, N};
  const int mt = (K + GM - 1) / GM;
  if ((int64_t)((N + GN - 1) / GN) * mt >= h->sm_count) {
    auto k = target_gccnmf_kernel<GN, GTN>;
    GCCNMF_LAUNCH(h, k, dim3((N + GN - 1) / GN, mt), (GM / GTM) * (GN / GTN), 0, stream, K, N, F, a, b, T, P, values);
  } else {
    constexpr int kBN = 32, kTN = 4;
    auto k = target_gccnmf_kernel<kBN, kTN>;
    GCCNMF_LAUNCH(h, k, dim3((N + kBN - 1) / kBN, mt), (GM / GTM) * (kBN / kTN), 0, stream, K, N, F, a, b, T, P, values);
  }
  return GCCNMF_OK;
}

// ---- steering banks (gccnmf_llbank_*): the forms above whose column t reads table bank.entry(t)
// gccnmf_phat_angspec of a spectrogram pair into coherence and angular spectrum; the grid covers the most tiles the entries can
// cut (fixed for a configuration, so the launch can sit in a graph whatever the assignment).
int gccnmf_phat_angspec_bank(gccnmf_handle* h, const float* X, int F, int T, const SteerBank& bank, int D, float* coherence, double* angular,
                             void* stream) {
  GCCNMF_REQUIRE(h, F > 0 && T > 0 && D > 0 && X && coherence && angular && bank.Qe >= 1, "phat_angspec_bank: bad arguments");
  if (D > kAngMaxD) return gccnmf_fail(h, GCCNMF_ERR_UNSUPPORTED, "phat_angspec_bank: numTDOAs %d > %d", D, kAngMaxD);
  const int tiles = steer_tiles_max(T, kAngT, bank.Qe);
  const float2* Xc = reinterpret_cast<const float2*>(X);
  float2* Cc = reinterpret_cast<float2*>(coherence);
  if (D <= 32) GCCNMF_LAUNCH(h, (phat_angspec_bank_kernel<1, 32>), tiles, kAngWarps * 32, 0, stream, Xc, F, T, bank, D, Cc, angular);
  else if (D <= 64) GCCNMF_LAUNCH(h, (phat_angspec_bank_kernel<2, 16>), tiles, kAngWarps * 32, 0, stream, Xc, F, T, bank, D, Cc, angular);
  else GCCNMF_LAUNCH(h, (phat_angspec_bank_kernel<4, 8>), tiles, kAngWarps * 32, 0, stream, Xc, F, T, bank, D, Cc, angular);
  return GCCNMF_OK;
}

// The float64 all-TDOA argmax (gccnmf_tdoa_gccnmf's, argmax only); with `gate` the graph-safe fallback of gccnmf_tdoa_gccnmf_gated.
int gccnmf_tdoa_gccnmf_bank(gccnmf_handle* h, const float* coherence, int F, int T, const SteerBank& bank, int D, const float* W, int K,
                            int32_t* argmax, const int32_t* gate, int capacity, int32_t* ran, void* stream) {
  GCCNMF_REQUIRE(h, F > 0 && T > 0 && D > 0 && K > 0 && coherence && W && argmax && bank.Qe >= 1, "tdoa_gccnmf_bank: bad arguments");
  GCCNMF_REQUIRE(h, (int64_t)T * D < (int64_t)1 << 31, "tdoa_gccnmf_bank: T * D overflows int32");
  if (!(is_pow2(D) && D >= 4 && D <= GN))
    return gccnmf_fail(h, GCCNMF_ERR_UNSUPPORTED, "tdoa_gccnmf_bank: numTDOAs must be a power of two in [4, %d] (got %d)", GN, D);
  const int N = T * D;
  LoadWAtoms a{W, K, F};
  LoadRealGCCBank b{reinterpret_cast<const float2*>(coherence), bank, F, T, D, N};
  GCCNMF_LAUNCH(h, tdoa_argmax_bank_kernel, dim3((N + GN - 1) / GN, (K + GM - 1) / GM), kGccThreads, 0, stream, K, N, F, a, b, T, D, argmax, gate,
                capacity, ran);
  return GCCNMF_OK;
}

int gccnmf_target_gccnmf_bank(gccnmf_handle* h, const float* coherence, int F, int T, const SteerBank& bank, int D, const float* W, int K,
                              const int32_t* targets, int P, float* values, void* stream) {
  GCCNMF_REQUIRE(h, F > 0 && T > 0 && D > 0 && K > 0 && P > 0 && coherence && W && targets && values && bank.Qe >= 1,
                 "target_gccnmf_bank: bad arguments");
  GCCNMF_REQUIRE(h, (int64_t)T * P < (int64_t)1 << 31 && (int64_t)P * K * T < (int64_t)1 << 31, "target_gccnmf_bank: T x P or P x K x T overflows int32");
  const int N = T * P;
  LoadWAtoms a{W, K, F};
  LoadTargetGCCBank b{reinterpret_cast<const float2*>(coherence), bank, targets, F, T, D, P, N};
  const int mt = (K + GM - 1) / GM;
  if ((int64_t)((N + GN - 1) / GN) * mt >= h->sm_count) {
    auto k = target_gccnmf_bank_kernel<GN, GTN>;
    GCCNMF_LAUNCH(h, k, dim3((N + GN - 1) / GN, mt), (GM / GTM) * (GN / GTN), 0, stream, K, N, F, a, b, T, P, values);
  } else {
    constexpr int kBN = 32, kTN = 4;
    auto k = target_gccnmf_bank_kernel<kBN, kTN>;
    GCCNMF_LAUNCH(h, k, dim3((N + kBN - 1) / kBN, mt), (GM / GTM) * (kBN / kTN), 0, stream, K, N, F, a, b, T, P, values);
  }
  return GCCNMF_OK;
}

// ---- dictionary banks (gccnmf_lldict_*): the forms above whose CTA takes its columns from one dictionary's segment (steer_tile on the
// dictionary sort) and contracts over that entry's W and K, so every value is the same fma chain a plain kernel over (W_e, K_e) runs.
namespace {

// B(n = j D + d, k = f) = Re(coherence[f][t] E_t[f][d]) for frame j of the tile, t = its column, E_t the table of t's stream
struct LoadRealGCCDict {
  static constexpr bool kContigK = false;
  const float2* coh; SteerBank bank; DictBank dict; int F, T, D, u0, N;
  __device__ double operator()(int n, int f) const {
    if (n >= N || f >= F) return 0.0;
    const int j = n / D, d = n - j * D, t = dict.column(u0 + j);
    return re_coh_steer(__ldg(coh + (int64_t)f * T + t), __ldg(bank.E + ((int64_t)bank.entry(t) * F + f) * D + d));
  }
};
struct LoadTargetGCCDict {
  static constexpr bool kContigK = false;
  const float2* coh; SteerBank bank; DictBank dict; const int32_t* targets; int F, T, D, P, u0, N;
  __device__ double operator()(int n, int f) const {
    if (n >= N || f >= F) return 0.0;
    const int j = n / P, q = n - j * P, t = dict.column(u0 + j);
    return re_coh_steer(__ldg(coh + (int64_t)f * T + t), __ldg(bank.E + ((int64_t)bank.entry(t) * F + f) * D + __ldg(targets + (int64_t)t * P + q)));
  }
};

__global__ void __launch_bounds__(kGccThreads)
tdoa_argmax_dict_kernel(int F, SteerBank bank, DictBank dict, const float2* __restrict__ coh, int T, int D, int32_t* __restrict__ argmax,
                        const int32_t* __restrict__ gate, int gate_capacity, int32_t* __restrict__ ran) {
  if (gate) {
    if (*gate <= gate_capacity) return;
    if (ran && blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) *ran = 1;
  }
  int u0, u1;
  const int e = steer_tile(dict.segments(), GN / D, blockIdx.x, u0, u1);
  if (e < 0) return;
  const int K = __ldg(dict.K + e), m0 = blockIdx.y * GM;
  if (m0 >= K) return;
  const int N = (u1 - u0) * D;
  LoadWAtoms a{dict.W + e * dict.wstride, K, F};
  LoadRealGCCDict b{coh, bank, dict, F, T, D, u0, N};
  double acc[GTM][GTN];
  gemm_simt_mainloop<double, GM, GN, GK, GTM, GTN>(acc, m0, 0, F, a, b);
  constexpr int TX = GN / GTN;
  const int tx = threadIdx.x % TX;
  const int lanes = min(D / 4, TX);
#pragma unroll
  for (int i = 0; i < GTM; ++i) {
    const int m = gemm_row<GM, GTM, TX>(m0, i);
    double bv[2];
    int bi[2];
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const int d0 = (half * (GN / 2) + tx * (GTN / 2)) % D;
      bv[half] = acc[i][half * (GTN / 2)];
      bi[half] = d0;
#pragma unroll
      for (int j = 1; j < GTN / 2; ++j) {
        const double v = acc[i][half * (GTN / 2) + j];
        if (argmax_better(v, d0 + j, bv[half], bi[half])) { bv[half] = v; bi[half] = d0 + j; }
      }
    }
    if (D == GN) {
      if (argmax_better(bv[1], bi[1], bv[0], bi[0])) { bv[0] = bv[1]; bi[0] = bi[1]; }
    }
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      if (D == GN && half == 1) break;
      for (int o = 1; o < lanes; o <<= 1) {
        const double ov = __shfl_xor_sync(0xffffffffu, bv[half], o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi[half], o);
        if (argmax_better(ov, oi, bv[half], bi[half])) { bv[half] = ov; bi[half] = oi; }
      }
      const int n_first = half * (GN / 2) + tx * (GTN / 2);
      if ((tx % lanes) == 0 && m < K && n_first < N) argmax[(int64_t)m * T + dict.column(u0 + n_first / D)] = bi[half];
    }
  }
}

// values (P, Kmax, T): rows < K_e of each column; the rows above are the caller's to fill
__global__ void __launch_bounds__(kGccThreads)
target_gccnmf_dict_kernel(int F, SteerBank bank, DictBank dict, const float2* __restrict__ coh, const int32_t* __restrict__ targets, int T, int D,
                          int P, float* __restrict__ values) {
  int u0, u1;
  const int e = steer_tile(dict.segments(), GN / P, blockIdx.x, u0, u1);
  if (e < 0) return;
  const int K = __ldg(dict.K + e), m0 = blockIdx.y * GM;
  if (m0 >= K) return;
  const int N = (u1 - u0) * P;
  LoadWAtoms a{dict.W + e * dict.wstride, K, F};
  LoadTargetGCCDict b{coh, bank, dict, targets, F, T, D, P, u0, N};
  double acc[GTM][GTN];
  gemm_simt_mainloop<double, GM, GN, GK, GTM, GTN>(acc, m0, 0, F, a, b);
  constexpr int TX = GN / GTN;
#pragma unroll
  for (int i = 0; i < GTM; ++i) {
    const int m = gemm_row<GM, GTM, TX>(m0, i);
    if (m >= K) continue;
#pragma unroll
    for (int j = 0; j < GTN; ++j) {
      const int n = gemm_col<GN, GTN, TX>(0, j);
      if (n >= N) continue;
      const int jj = n / P, q = n - jj * P;
      values[((int64_t)q * dict.Kmax + m) * T + dict.column(u0 + jj)] = (float)acc[i][j];
    }
  }
}

// B(n, k) of the Wiener filters for tile column n (sorted position u0 + n): mask[k][t] (H == NULL) or H[k][c T + t] (* mask[k][t])
struct LoadDictCols {
  static constexpr bool kContigK = false;
  const float* H; const float* mask; DictBank dict; int K, T, u0, N; int64_t ldh;
  __device__ float operator()(int n, int k) const {
    if (n >= N || k >= K) return 0.f;
    const int t = dict.column(u0 + n);
    if (!H) return __ldg(mask + (int64_t)k * T + t);
    const float hv = __ldg(H + (int64_t)k * ldh + t);
    return mask ? hv * __ldg(mask + (int64_t)k * T + t) : hv;
  }
};

// wiener_apply_kernel (H == NULL, rowsum(W_e) from the bank) and wiener_apply_h_kernel (channel c = blockIdx.z) over RN columns of
// one dictionary segment
template <bool WITH_H>
__global__ void __launch_bounds__(kReconThreads, 2)
wiener_dict_kernel(const float* __restrict__ mask, DictBank dict, const float* __restrict__ H, const float2* __restrict__ X, int F, int T,
                   float2* __restrict__ Y, float* __restrict__ wiener) {
  int u0, u1;
  const int e = steer_tile(dict.segments(), RN, blockIdx.x, u0, u1);
  if (e < 0) return;
  const int K = __ldg(dict.K + e), c = blockIdx.z, N = u1 - u0;
  const int m0 = blockIdx.y * RM;
  LoadWRows a{dict.W + e * dict.wstride, F, K};
  float num[RTM][RTN], den[WITH_H ? RTM : 1][WITH_H ? RTN : 1];
  if constexpr (WITH_H) {
    LoadDictCols masked{H + (int64_t)c * T, mask, dict, K, T, u0, N, (int64_t)2 * T}, plain{H + (int64_t)c * T, nullptr, dict, K, T, u0, N, (int64_t)2 * T};
    gemm_simt_mainloop<float, RM, RN, RK, RTM, RTN>(num, m0, 0, K, a, masked);
    gemm_simt_mainloop<float, RM, RN, RK, RTM, RTN>(den, m0, 0, K, a, plain);
  } else {
    LoadDictCols b{nullptr, mask, dict, K, T, u0, N, 0};
    gemm_simt_mainloop<float, RM, RN, RK, RTM, RTN>(num, m0, 0, K, a, b);
  }
#pragma unroll
  for (int i = 0; i < RTM; ++i) {
    const int m = gemm_row<RM, RTM, RN / RTN>(m0, i);
    if (m >= F) continue;
    const float rs = WITH_H ? 0.f : __ldg(dict.rowsum + (int64_t)e * F + m);
#pragma unroll
    for (int j = 0; j < RTN; ++j) {
      const int n = gemm_col<RN, RTN, RN / RTN>(0, j);
      if (n >= N) continue;
      const int t = dict.column(u0 + n);
      if constexpr (WITH_H) {
        const float w = num[i][j] / den[i][j];
        const int64_t o = ((int64_t)c * F + m) * T + t;
        if (wiener) wiener[o] = w;
        const float2 x = X[o];
        Y[o] = float2{w * x.x, w * x.y};
      } else {
        const float w = num[i][j] / rs;
        if (wiener) wiener[(int64_t)m * T + t] = w;
#pragma unroll
        for (int cc = 0; cc < 2; ++cc) {
          const float2 x = X[((int64_t)cc * F + m) * T + t];
          Y[((int64_t)cc * F + m) * T + t] = float2{w * x.x, w * x.y};
        }
      }
    }
  }
}

}  // namespace

int gccnmf_tdoa_gccnmf_dict(gccnmf_handle* h, const float* coherence, int F, int T, const SteerBank& bank, const DictBank& dict, int D,
                            int32_t* argmax, const int32_t* gate, int capacity, int32_t* ran, void* stream) {
  GCCNMF_REQUIRE(h, F > 0 && T > 0 && coherence && argmax && bank.Qe >= 1 && dict.Qd >= 1, "tdoa_gccnmf_dict: bad arguments");
  GCCNMF_REQUIRE(h, (int64_t)T * D < (int64_t)1 << 31, "tdoa_gccnmf_dict: T * D overflows int32");
  if (!(is_pow2(D) && D >= 4 && D <= GN))
    return gccnmf_fail(h, GCCNMF_ERR_UNSUPPORTED, "tdoa_gccnmf_dict: numTDOAs must be a power of two in [4, %d] (got %d)", GN, D);
  GCCNMF_LAUNCH(h, tdoa_argmax_dict_kernel, dim3(steer_tiles_max(T, GN / D, dict.Qd), (dict.Kmax + GM - 1) / GM), kGccThreads, 0, stream, F, bank,
                dict, reinterpret_cast<const float2*>(coherence), T, D, argmax, gate, capacity, ran);
  return GCCNMF_OK;
}

int gccnmf_target_gccnmf_dict(gccnmf_handle* h, const float* coherence, int F, int T, const SteerBank& bank, const DictBank& dict, int D,
                              const int32_t* targets, int P, float* values, void* stream) {
  GCCNMF_REQUIRE(h, F > 0 && T > 0 && P > 0 && P <= GN && coherence && targets && values && bank.Qe >= 1 && dict.Qd >= 1,
                 "target_gccnmf_dict: bad arguments");
  GCCNMF_LAUNCH(h, target_gccnmf_dict_kernel, dim3(steer_tiles_max(T, GN / P, dict.Qd), (dict.Kmax + GM - 1) / GM), kGccThreads, 0, stream, F, bank,
                dict, reinterpret_cast<const float2*>(coherence), targets, T, D, P, values);
  return GCCNMF_OK;
}

// H == NULL: gccnmf_wiener_apply's filter; else gccnmf_wiener_apply_h's, per column on its dictionary
int gccnmf_wiener_dict(gccnmf_handle* h, const float* mask, const DictBank& dict, const float* H, const float* X, int F, int T, float* Y, float* wiener,
                       void* stream) {
  GCCNMF_REQUIRE(h, mask && X && Y && F > 0 && T > 0 && dict.Qd >= 1, "wiener_dict: bad arguments");
  const dim3 grid(steer_tiles_max(T, RN, dict.Qd), (F + RM - 1) / RM, H ? 2 : 1);
  if (H)
    GCCNMF_LAUNCH(h, wiener_dict_kernel<true>, grid, kReconThreads, 0, stream, mask, dict, H, reinterpret_cast<const float2*>(X), F, T,
                  reinterpret_cast<float2*>(Y), wiener);
  else
    GCCNMF_LAUNCH(h, wiener_dict_kernel<false>, grid, kReconThreads, 0, stream, mask, dict, H, reinterpret_cast<const float2*>(X), F, T,
                  reinterpret_cast<float2*>(Y), wiener);
  return GCCNMF_OK;
}

// rowsum(W) (F) as gccnmf_wiener_apply computes it
int gccnmf_rowsum_w(gccnmf_handle* h, const float* W, int F, int K, float* rowsum, void* stream) {
  GCCNMF_LAUNCH(h, rowsum_w_kernel, F, 128, 0, stream, W, F, K, rowsum);
  return GCCNMF_OK;
}
