// All-TDOA GCC-NMF argmax on the tensor cores with exact float64 refinement
// (reference: notebooks/offlineSpeechEnhancement.ipynb cells 27+29, :444-467; online :422-423), and the masked reconstruction
// (gccNMF/gccNMFFunctions.py:145-151) on the same TMA-fed plane GEMM (tma_gemm.cuh) the KL-NMF loop runs on.
//
//   gccNMF[k, tau, t] = sum_f W[f, k] * Re(C[f, t] E[f, tau])        argmax over tau per (k, t)
//
// The reference evaluates this in float64 and the argmax must be the reference's, bit for bit.  A
// float64 contraction is 126 GFLOP at the headline shape (10.9 ms on the SIMT float64 kernel), so:
//   1. build  G[(t, tau), f] = Re(C E)  once: float64 product, rounded to float32, split into bf16 hi / lo planes  (HBM-bound)
//   2. W^T . G^T  on the plane GEMM (3 bf16 products per algorithmic product; M = atoms: W is consumed MN-major as it lies,
//      N = (t, tau) in 256-column tiles = 256 / D whole frames, over f; m-fastest grid + TMA multicast of the G tile to the pair of
//      m tiles that share it, so G streams from HBM once); the whole-tile epilogue keeps, per (atom, frame), the best and
//      second-best value and the index of the best;
//   3. every (atom, frame) whose margin best - second is below the worst-case error of step 2
//      (margin_factor(F) * sum_f |W[f, atom]|, since |G| <= 1) is appended to a list and recomputed EXACTLY in
//      float64 from C, E and W by a warp (the same arithmetic as the float64 kernel in gcc.cu).
// Decisions with a safe margin cannot differ from the float64 ones; the others are the float64 ones.
#include <algorithm>

#include "common.cuh"
#include "tma_gemm_host.cuh"

namespace {

using namespace tgemm_host;

// Error budget of step 2 relative to sum_f |W| (|G| <= 1): the bf16 hi / lo split leaves 2^-18 of each operand and drops the
// lo.lo term (2^-18): <= 3 x 2^-18 per product, worst case all coherent; float32 rounding of G 2^-24; the float32 tensor-core
// accumulator <= 2^-24 per accumulation over 3 F / 16 accumulations (measured 1.2e-5 at 384 accumulations,
// tests/test_gpu_tma.py).  The margin is twice that (two values, each off by the bound) plus 25 % slack; it grows with F.
inline float margin_factor(int F) {
  const double per_value = 3.0 / 262144.0 + (1.0 + 3.0 * F / 16.0) / 16777216.0;
  return (float)(2.5 * per_value);
}

// ------------------------------------------------------------------ step 1: planes of G[(t, tau)][f]
// CTA = 64 bins x 32 frames x all TDOAs.  Warp w owns the TDOAs d = w, w + 8, ... ; lane = bins 2 l, 2 l + 1, so every store is one
// 128-byte row segment of a plane.  E[f][d] is loaded once per (thread, d) -- its rows are D * 16 bytes apart, so a warp's load
// touches 32 lines: doing it inside the frame loop made the first version L1-wavefront-bound -- and reused for the 32 frames of
// the tile, whose coherence values sit in shared memory.
__global__ void __launch_bounds__(256)
build_gcc_planes_kernel(const float2* __restrict__ coh, int F, int T, const double2* __restrict__ E, int D, bf16* __restrict__ G, int64_t pitch,
                        int64_t plane) {
  __shared__ float2 Cs[64][33];   // [f][t]
  const int f0 = blockIdx.x * 64, t0 = blockIdx.y * 32;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (int i = w; i < 64; i += 8) {
    const int f = f0 + i, t = t0 + lane;
    Cs[i][lane] = (f < F && t < T) ? coh[(int64_t)f * T + t] : float2{0.f, 0.f};
  }
  __syncthreads();
  const int f = f0 + 2 * lane;
  if (f >= pitch) return;
  const int t_end = min(32, T - t0);
  for (int d0 = w; d0 < D; d0 += 16) {            // 2 TDOAs per pass: d0, d0 + 8
    double2 e[2][2];
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const int d = d0 + 8 * j;
        e[j][q] = (f + q < F && d < D) ? __ldg(E + (int64_t)(f + q) * D + d) : double2{0.0, 0.0};
      }
    for (int tt = 0; tt < t_end; ++tt) {
      const float2 c0 = Cs[2 * lane][tt], c1 = Cs[2 * lane + 1][tt];
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        if (d0 + 8 * j >= D) break;
        // float64 product rounded to float32 (what the float64 contraction sees to 2^-24), then the hi / lo split
        const float g0 = (float)((double)c0.x * e[j][0].x - (double)c0.y * e[j][0].y);
        const float g1 = (float)((double)c1.x * e[j][1].x - (double)c1.y * e[j][1].y);
        bf16 h0, l0, h1, l1;
        split_bf16(g0, h0, l0);
        split_bf16(g1, h1, l1);
        bf16* row = G + ((int64_t)(t0 + tt) * D + d0 + 8 * j) * pitch + f;
        *reinterpret_cast<__nv_bfloat162*>(row) = __nv_bfloat162(h0, h1);
        *reinterpret_cast<__nv_bfloat162*>(row + plane) = __nv_bfloat162(l0, l1);
      }
    }
  }
}

// build_gcc_planes_kernel for a steering bank: a CTA takes 32 columns of one entry in sorted order (steer_tile) and reuses that
// table's rows across them, writing each column's rows where the plain kernel writes them.
__global__ void __launch_bounds__(256)
build_gcc_planes_bank_kernel(const float2* __restrict__ coh, int F, int T, SteerBank bank, int D, bf16* __restrict__ G, int64_t pitch, int64_t plane) {
  __shared__ float2 Cs[64][33];   // [f][tile column]
  __shared__ int col_s[32];
  int u0, u1;
  const int entry = steer_tile(bank, 32, blockIdx.y, u0, u1);
  if (entry < 0) return;
  const double2* __restrict__ E = bank.E + (int64_t)entry * F * D;
  const int f0 = blockIdx.x * 64;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (threadIdx.x < 32) col_s[lane] = u0 + lane < u1 ? bank.column(u0 + lane) : -1;
  __syncthreads();
  for (int i = w; i < 64; i += 8) {
    const int f = f0 + i, t = col_s[lane];
    Cs[i][lane] = (f < F && t >= 0) ? coh[(int64_t)f * T + t] : float2{0.f, 0.f};
  }
  __syncthreads();
  const int f = f0 + 2 * lane;
  if (f >= pitch) return;
  const int t_end = u1 - u0;
  for (int d0 = w; d0 < D; d0 += 16) {
    double2 e[2][2];
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const int d = d0 + 8 * j;
        e[j][q] = (f + q < F && d < D) ? __ldg(E + (int64_t)(f + q) * D + d) : double2{0.0, 0.0};
      }
    for (int tt = 0; tt < t_end; ++tt) {
      const float2 c0 = Cs[2 * lane][tt], c1 = Cs[2 * lane + 1][tt];
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        if (d0 + 8 * j >= D) break;
        const float g0 = (float)((double)c0.x * e[j][0].x - (double)c0.y * e[j][0].y);
        const float g1 = (float)((double)c1.x * e[j][1].x - (double)c1.y * e[j][1].y);
        bf16 h0, l0, h1, l1;
        split_bf16(g0, h0, l0);
        split_bf16(g1, h1, l1);
        bf16* row = G + ((int64_t)col_s[tt] * D + d0 + 8 * j) * pitch + f;
        *reinterpret_cast<__nv_bfloat162*>(row) = __nv_bfloat162(h0, h1);
        *reinterpret_cast<__nv_bfloat162*>(row + plane) = __nv_bfloat162(l0, l1);
      }
    }
  }
}

// planes[p][i] = split(src[i])  (W as it lies: (F, K) row-major = MN-major operand of the argmax GEMM, K-major of the reconstruction)
__global__ void split_to_planes_kernel(const float* __restrict__ src, int64_t n, bf16* __restrict__ planes, int64_t plane) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  bf16 hi, lo;
  split_bf16(src[i], hi, lo);
  planes[i] = hi;
  planes[plane + i] = lo;
}

// ------------------------------------------------------------------ step 2: whole-tile epilogue of the plane GEMM
// tile[n][m]: m = atom (128 per tile), n = (frame, TDOA) with BN / D whole frames per tile.  One thread per (atom, frame) scans the
// D columns of its frame (consecutive atoms = consecutive shared-memory words: no bank conflicts).
struct EpiArgmaxTile {
  static constexpr bool kTileEpilogue = true;
  static constexpr bool kRowReduce = false;
  static constexpr int kRowValues = 0;
  static constexpr bool kPrefetch = false;
  struct State {};
  struct Loaded {};
  int32_t* __restrict__ argmax;        // (K, T)
  const float* __restrict__ colsumW;   // (K) sum_f |W[f,k]|
  int2* __restrict__ list; uint4* __restrict__ candidates; int* __restrict__ count; int capacity;
  int K, T, D; float margin_factor;
  __device__ void prefetch(int, int) const {}
  __device__ void row_values(int, float*) const {}
  __device__ void elem(int, int, float, int) const {}
  __device__ void tile_epilogue(const float* __restrict__ tile, int m0, int n0, int n_valid, int) const {
    const int frames = n_valid / D;                         // N = T D and the tile width is a multiple of D
    for (int p = threadIdx.x; p < tgemm::kBM * frames; p += blockDim.x) {
      const int ml = p & (tgemm::kBM - 1), j = p / tgemm::kBM;
      const int m = m0 + ml;
      if (m >= K) continue;
      const float* col = tile + (size_t)(j * D) * tgemm::kTileLd + ml;
      float best = -INFINITY, second = -INFINITY;
      int idx = 0, nan = 0;
#pragma unroll 8
      for (int d = 0; d < D; ++d) {
        const float x = col[(size_t)d * tgemm::kTileLd];
        if (x != x) nan = 1;                 // NaN anywhere: let float64 decide with numpy's NaN rules
        if (x > best) { second = best; best = x; idx = d; }
        else if (x > second) second = x;
      }
      const int t = n0 / D + j;
      argmax[(int64_t)m * T + t] = idx;
      const float margin = margin_factor * colsumW[m];
      if (nan || !(best - second > margin)) {
        // the TDOAs that can still be the float64 maximum: every value within the margin of the best (all of them after a NaN)
        uint32_t bits[4] = {0u, 0u, 0u, 0u};
        for (int d = 0; d < D; ++d) {
          const float x = col[(size_t)d * tgemm::kTileLd];
          if (nan || !(best - x > margin)) bits[d >> 5] |= 1u << (d & 31);
        }
        const int slot = atomicAdd(count, 1);
        if (slot < capacity) {
          list[slot] = make_int2(m, t);
          candidates[slot] = make_uint4(bits[0], bits[1], bits[2], bits[3]);
        }
      }
    }
  }
};

// ------------------------------------------------------------------ step 2, persistent form
// The argmax GEMM has many tiles per SM (8 m tiles x T D / 256 n tiles = 3744 at the headline shape, 28 per SM) and no dependency
// between them, so it runs as ONE persistent CTA per SM that walks the tiles m-fastest (the 8 CTAs working on the same B tile are
// neighbours: it is read from HBM once and from the L2 seven times), with the shared-memory pipeline running across tile
// boundaries: the producer fills the stages of tile j + 1 while the MMA warpgroups reduce tile j straight from their registers
// (no shared-memory staging), and the per-CTA prologue is paid once instead of 28 times.  Same arithmetic as
// plane_gemm_kernel<256, 32, true, false> + EpiArgmaxTile (three bf16 products per k-step into one float32 accumulator, k tail
// included): identical values, identical decisions.
constexpr int kPersBN = 256, kPersKB = 32, kPersStages = 4;
constexpr int kPersABytes = 2 * tgemm::kBM * kPersKB * 2;            // MN-major A: 2 atoms of 64 atoms x 32 k-rows x 2 planes = 16 KB
constexpr int kPersBBytes = 2 * kPersBN * kPersKB * 2;               // K-major B: 2 planes x 256 rows x 64 B = 32 KB
constexpr int kPersStageBytes = kPersABytes + kPersBBytes;
constexpr int kPersSmem = kPersStages * kPersStageBytes + 256 + 1024;
constexpr int kPersAtomBytes = 2 * kPersKB * 128;

// (best, second, index of best, NaN seen) of a thread's share of a frame, merged with the lanes that hold the rest of its columns
struct ArgmaxPartial {
  float best, second;
  int idx, nan;
  __device__ void scan(float x, int d) {     // d ascending within a thread: the first of equal maxima wins
    if (x != x) nan = 1;
    if (x > best) { second = best; best = x; idx = d; }
    else if (x > second) second = x;
  }
  __device__ void merge_xor(int o) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o), os = __shfl_xor_sync(0xffffffffu, second, o);
    const int oi = __shfl_xor_sync(0xffffffffu, idx, o), on = __shfl_xor_sync(0xffffffffu, nan, o);
    const bool take = ob > best || (ob == best && oi < idx);
    const float loser = take ? best : ob;
    if (take) { best = ob; idx = oi; }
    second = fmaxf(fmaxf(second, os), loser);         // (scan never stores a NaN: NaN frames are flagged through `nan`)
    nan |= on;
  }
};

template <int D>
__global__ void __launch_bounds__(tgemm::kThreads, 1)
argmax_gemm_persistent_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, int K, int N, int Kc, int m_tiles,
                              int n_tiles, EpiArgmaxTile epi) {
  using namespace tgemm;
  static_assert(D >= 32 && D <= 128 && kPersBN % D == 0, "whole frames of at most 128 TDOAs per tile");
  extern __shared__ unsigned char smem_dyn[];
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~uintptr_t(1023));
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kPersStages * kPersStageBytes);
  uint64_t* full = bars;                         // [stages]  TMA -> MMA
  uint64_t* empty = bars + kPersStages;          // [stages]  MMA warpgroups -> TMA
  if (tid == 0) {
    for (int s = 0; s < kPersStages; ++s) { mbar_init(smem_u32(&full[s]), 1); mbar_init(smem_u32(&empty[s]), kMmaWarpgroups); }
    gmma::fence_barrier_init();
    tma_prefetch_descriptor(&map_a);
    tma_prefetch_descriptor(&map_b);
  }
  __syncthreads();
  const int total_tiles = m_tiles * n_tiles;
  const int num_kb = (Kc + kPersKB - 1) / kPersKB;

  if (warp == 0) {
    if (lane == 0) {
      uint32_t g = 0;                                                  // k-blocks produced so far (all tiles)
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int m0 = (tile % m_tiles) * kBM, n0 = (tile / m_tiles) * kPersBN;
        for (int i = 0; i < num_kb; ++i, ++g) {
          const int s = g % kPersStages;
          const uint32_t use = g / kPersStages;
          if (use > 0) mbar_wait(smem_u32(&empty[s]), (use - 1) & 1);
          const uint32_t bar = smem_u32(&full[s]);
          const uint32_t a_dst = smem_u32(smem + (size_t)s * kPersStageBytes), b_dst = a_dst + kPersABytes;
          mbar_arrive_expect_tx(bar, kPersStageBytes);
          const int k0 = i * kPersKB;
#pragma unroll
          for (int a = 0; a < 2; ++a) tma_load_3d(a_dst + a * kPersAtomBytes, &map_a, bar, m0 + 64 * a, k0, 0);
#pragma unroll
          for (int p = 0; p < 2; ++p) tma_load_3d(b_dst + p * (kPersBN * kPersKB * 2), &map_b, bar, k0, n0, p);
        }
      }
    }
    __syncwarp();
  } else if (warp >= 4) {
    // ---------------------------------------------------------------- MMA warpgroups: 64 atoms each, then argmax per (atom, frame)
    const int g = (warp >> 2) - 1, wt = tid & 127;
    const int c0 = 2 * (wt & 3);                                       // this thread's columns: 8 q + c0, 8 q + c0 + 1
    constexpr int kFrames = kPersBN / D, kGroups = D / 8, kWords = (D + 31) / 32;
    uint32_t gk = 0;                                                   // k-blocks consumed (all tiles)
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const int m0 = (tile % m_tiles) * kBM, n0 = (tile / m_tiles) * kPersBN;
      float acc[kPersBN / 2];
#pragma unroll
      for (int j = 0; j < kPersBN / 2; ++j) acc[j] = 0.f;
      for (int i = 0; i < num_kb; ++i, ++gk) {
        const int s = gk % kPersStages;
        mbar_wait(smem_u32(&full[s]), (gk / kPersStages) & 1);
        const uint32_t a_base = smem_u32(smem + (size_t)s * kPersStageBytes), b_base = a_base + kPersABytes;
        gmma::fence_regs(acc);
        gmma::wgmma_fence();
        mma_kblock<kPersBN, kPersKB, true, false, false>(acc, a_base + g * kPersAtomBytes, b_base, kPersBN * kPersKB * 2);
        gmma::wgmma_commit();
        gmma::fence_regs(acc);
        gmma::wgmma_wait<1>();
        if (i > 0 && wt == 0) gmma::mbar_arrive(smem_u32(&empty[(gk - 1) % kPersStages]));
      }
      gmma::wgmma_wait<0>();
      gmma::fence_regs(acc);
      if (num_kb > 0 && wt == 0) gmma::mbar_arrive(smem_u32(&empty[(gk - 1) % kPersStages]));

      const int frames = min(kPersBN, N - n0) / D;
#pragma unroll
      for (int h = 0; h < 2; ++h) {                                    // rows r and r + 8 of the thread
        const int m = m0 + 64 * g + 16 * (wt >> 5) + ((wt & 31) >> 2) + 8 * h;
        const float margin = m < K ? epi.margin_factor * epi.colsumW[m] : 0.f;
#pragma unroll
        for (int fr = 0; fr < kFrames; ++fr) {
          ArgmaxPartial p{-INFINITY, -INFINITY, 0, 0};
#pragma unroll
          for (int q = 0; q < kGroups; ++q) {
            p.scan(acc[4 * (fr * kGroups + q) + 2 * h], 8 * q + c0);
            p.scan(acc[4 * (fr * kGroups + q) + 2 * h + 1], 8 * q + c0 + 1);
          }
          p.merge_xor(1);
          p.merge_xor(2);
          const bool valid = m < K && fr < frames;
          const int t = n0 / D + fr;
          if (valid && (wt & 3) == 0) epi.argmax[(int64_t)m * epi.T + t] = p.idx;
          const bool near_tie = valid && (p.nan || !(p.best - p.second > margin));
          if (__any_sync(0xffffffffu, near_tie)) {
            uint32_t bits[kWords];                                     // the candidates within the margin
#pragma unroll
            for (int w = 0; w < kWords; ++w) bits[w] = 0u;
#pragma unroll
            for (int q = 0; q < kGroups; ++q)
#pragma unroll
              for (int b = 0; b < 2; ++b) {
                const int d = 8 * q + c0 + b;
                const float x = acc[4 * (fr * kGroups + q) + 2 * h + b];
                if (p.nan || !(p.best - x > margin)) bits[d >> 5] |= 1u << (d & 31);
              }
#pragma unroll
            for (int w = 0; w < kWords; ++w) {
              bits[w] |= __shfl_xor_sync(0xffffffffu, bits[w], 1);
              bits[w] |= __shfl_xor_sync(0xffffffffu, bits[w], 2);
            }
            if (near_tie && (wt & 3) == 0) {
              const int slot = atomicAdd(epi.count, 1);
              if (slot < epi.capacity) {
                uint32_t b4[4] = {0u, 0u, 0u, 0u};
#pragma unroll
                for (int w = 0; w < kWords; ++w) b4[w] = bits[w];
                epi.list[slot] = make_int2(m, t);
                epi.candidates[slot] = make_uint4(b4[0], b4[1], b4[2], b4[3]);
              }
            }
          }
        }
      }
    }
  }
}

template <int D>
int launch_argmax_persistent(gccnmf_handle* h, const CUtensorMap& map_a, const CUtensorMap& map_b, int K, int N, int F, int m_tiles, int n_tiles,
                             const EpiArgmaxTile& epi, void* stream) {
  static DeviceFlags configured;
  if (!configured(h)) {
    GCCNMF_CHECK_CUDA(h, cudaFuncSetAttribute(argmax_gemm_persistent_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, kPersSmem));
    configured(h) = true;
  }
  const int ctas = std::min(h->sm_count, m_tiles * n_tiles);
  return launch_ex(h, "argmax_gemm_persistent_kernel", argmax_gemm_persistent_kernel<D>, dim3(ctas), dim3(tgemm::kThreads), (size_t)kPersSmem, stream,
                   false, dim3(1, 1, 1), map_a, map_b, K, N, F, m_tiles, n_tiles, epi);
}

// ------------------------------------------------------------------ step 2 for a dictionary bank (gccnmf_lldict_*)
// argmax_gemm_persistent_kernel over Qd dictionaries in one launch.  An n tile holds up to 256 / D frames of ONE entry's segment in
// sorted order (steer_tile), an m tile 128 of that entry's atoms; tiles past the last segment or at or above K[e] are skipped by
// the producer and the consumers alike.  A is the stacked (F, Qd Kp) planes, so entry e's tile starts at column e Kp + m0.  B is
// gathered: 256 / D boxes of D rows (one frame each) per plane and k-block from G as the plain build lays it out; every box starts
// on a swizzle-atom boundary (D x 64 bytes), so the stage holds the image one 256-row box would, and the MMA code is the plain
// kernel's.  A short tile repeats its first frame in the unused slots (the transaction count stays fixed); the epilogue drops them.
struct EpiArgmaxDict {
  int32_t* __restrict__ argmax;        // (Kmax, T)
  int2* __restrict__ list; uint4* __restrict__ candidates; int* __restrict__ count; int capacity;
  int T; float margin_factor;
};

template <int D>
__global__ void __launch_bounds__(tgemm::kThreads, 1)
argmax_gemm_dict_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, int Kc, int m_tiles, int n_tiles,
                        DictBank dict, EpiArgmaxDict epi) {
  using namespace tgemm;
  static_assert(D >= 32 && D <= 128 && kPersBN % D == 0, "whole frames of at most 128 TDOAs per tile");
  constexpr int kFrames = kPersBN / D;
  extern __shared__ unsigned char smem_dyn[];
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~uintptr_t(1023));
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kPersStages * kPersStageBytes);
  uint64_t* full = bars;
  uint64_t* empty = bars + kPersStages;
  if (tid == 0) {
    for (int s = 0; s < kPersStages; ++s) { mbar_init(smem_u32(&full[s]), 1); mbar_init(smem_u32(&empty[s]), kMmaWarpgroups); }
    gmma::fence_barrier_init();
    tma_prefetch_descriptor(&map_a);
    tma_prefetch_descriptor(&map_b);
  }
  __syncthreads();
  const int total_tiles = m_tiles * n_tiles;
  const int num_kb = (Kc + kPersKB - 1) / kPersKB;
  const SteerBank segs = dict.segments();
  // the tile's entry (-1: skipped), first atom and sorted positions [u0, u1)
  auto decode = [&](int tile, int& m0, int& u0, int& u1) {
    m0 = (tile % m_tiles) * kBM;
    const int e = steer_tile(segs, kFrames, tile / m_tiles, u0, u1);
    return (e >= 0 && m0 < __ldg(dict.K + e)) ? e : -1;
  };

  if (warp == 0) {
    if (lane == 0) {
      uint32_t g = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        int m0, u0, u1;
        const int e = decode(tile, m0, u0, u1);
        if (e < 0) continue;
        int rows[kFrames];
#pragma unroll
        for (int j = 0; j < kFrames; ++j) rows[j] = dict.column(u0 + j < u1 ? u0 + j : u0) * D;
        const int ma = e * dict.Kp + m0;
        for (int i = 0; i < num_kb; ++i, ++g) {
          const int s = g % kPersStages;
          const uint32_t use = g / kPersStages;
          if (use > 0) mbar_wait(smem_u32(&empty[s]), (use - 1) & 1);
          const uint32_t bar = smem_u32(&full[s]);
          const uint32_t a_dst = smem_u32(smem + (size_t)s * kPersStageBytes), b_dst = a_dst + kPersABytes;
          mbar_arrive_expect_tx(bar, kPersStageBytes);
          const int k0 = i * kPersKB;
#pragma unroll
          for (int a = 0; a < 2; ++a) tma_load_3d(a_dst + a * kPersAtomBytes, &map_a, bar, ma + 64 * a, k0, 0);
#pragma unroll
          for (int p = 0; p < 2; ++p)
#pragma unroll
            for (int j = 0; j < kFrames; ++j) tma_load_3d(b_dst + p * (kPersBN * kPersKB * 2) + j * (D * kPersKB * 2), &map_b, bar, k0, rows[j], p);
        }
      }
    }
    __syncwarp();
  } else if (warp >= 4) {
    const int g = (warp >> 2) - 1, wt = tid & 127;
    const int c0 = 2 * (wt & 3);
    constexpr int kGroups = D / 8, kWords = (D + 31) / 32;
    uint32_t gk = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      int m0, u0, u1;
      const int e = decode(tile, m0, u0, u1);
      if (e < 0) continue;
      const int K = __ldg(dict.K + e);
      float acc[kPersBN / 2];
#pragma unroll
      for (int j = 0; j < kPersBN / 2; ++j) acc[j] = 0.f;
      for (int i = 0; i < num_kb; ++i, ++gk) {
        const int s = gk % kPersStages;
        mbar_wait(smem_u32(&full[s]), (gk / kPersStages) & 1);
        const uint32_t a_base = smem_u32(smem + (size_t)s * kPersStageBytes), b_base = a_base + kPersABytes;
        gmma::fence_regs(acc);
        gmma::wgmma_fence();
        mma_kblock<kPersBN, kPersKB, true, false, false>(acc, a_base + g * kPersAtomBytes, b_base, kPersBN * kPersKB * 2);
        gmma::wgmma_commit();
        gmma::fence_regs(acc);
        gmma::wgmma_wait<1>();
        if (i > 0 && wt == 0) gmma::mbar_arrive(smem_u32(&empty[(gk - 1) % kPersStages]));
      }
      gmma::wgmma_wait<0>();
      gmma::fence_regs(acc);
      if (num_kb > 0 && wt == 0) gmma::mbar_arrive(smem_u32(&empty[(gk - 1) % kPersStages]));

      const int frames = u1 - u0;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int m = m0 + 64 * g + 16 * (wt >> 5) + ((wt & 31) >> 2) + 8 * h;
        const float margin = m < K ? epi.margin_factor * __ldg(dict.colsum + (int64_t)e * dict.Kp + m) : 0.f;
#pragma unroll
        for (int fr = 0; fr < kFrames; ++fr) {
          ArgmaxPartial p{-INFINITY, -INFINITY, 0, 0};
#pragma unroll
          for (int q = 0; q < kGroups; ++q) {
            p.scan(acc[4 * (fr * kGroups + q) + 2 * h], 8 * q + c0);
            p.scan(acc[4 * (fr * kGroups + q) + 2 * h + 1], 8 * q + c0 + 1);
          }
          p.merge_xor(1);
          p.merge_xor(2);
          const bool valid = m < K && fr < frames;
          const int t = valid ? dict.column(u0 + fr) : 0;
          if (valid && (wt & 3) == 0) epi.argmax[(int64_t)m * epi.T + t] = p.idx;
          const bool near_tie = valid && (p.nan || !(p.best - p.second > margin));
          if (__any_sync(0xffffffffu, near_tie)) {
            uint32_t bits[kWords];
#pragma unroll
            for (int w = 0; w < kWords; ++w) bits[w] = 0u;
#pragma unroll
            for (int q = 0; q < kGroups; ++q)
#pragma unroll
              for (int b = 0; b < 2; ++b) {
                const int d = 8 * q + c0 + b;
                const float x = acc[4 * (fr * kGroups + q) + 2 * h + b];
                if (p.nan || !(p.best - x > margin)) bits[d >> 5] |= 1u << (d & 31);
              }
#pragma unroll
            for (int w = 0; w < kWords; ++w) {
              bits[w] |= __shfl_xor_sync(0xffffffffu, bits[w], 1);
              bits[w] |= __shfl_xor_sync(0xffffffffu, bits[w], 2);
            }
            if (near_tie && (wt & 3) == 0) {
              const int slot = atomicAdd(epi.count, 1);
              if (slot < epi.capacity) {
                uint32_t b4[4] = {0u, 0u, 0u, 0u};
#pragma unroll
                for (int w = 0; w < kWords; ++w) b4[w] = bits[w];
                epi.list[slot] = make_int2(m, t);
                epi.candidates[slot] = make_uint4(b4[0], b4[1], b4[2], b4[3]);
              }
            }
          }
        }
      }
    }
  }
}

template <int D>
int launch_argmax_dict(gccnmf_handle* h, const CUtensorMap& map_a, const CUtensorMap& map_b, int F, int m_tiles, int n_tiles, const DictBank& dict,
                       const EpiArgmaxDict& epi, void* stream) {
  static DeviceFlags configured;
  if (!configured(h)) {
    GCCNMF_CHECK_CUDA(h, cudaFuncSetAttribute(argmax_gemm_dict_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, kPersSmem));
    configured(h) = true;
  }
  const int ctas = std::min(h->sm_count, m_tiles * n_tiles);
  return launch_ex(h, "argmax_gemm_dict_kernel", argmax_gemm_dict_kernel<D>, dim3(ctas), dim3(tgemm::kThreads), (size_t)kPersSmem, stream, false,
                   dim3(1, 1, 1), map_a, map_b, F, m_tiles, n_tiles, dict, epi);
}

// ------------------------------------------------------------------ step 3: exact float64 recomputation of flagged (atom, frame) pairs
__device__ __forceinline__ bool argmax_better64(double v, int i, double bv, int bi) {   // numpy.argmax: NaN is a maximum, first wins
  const bool vn = v != v, bn = bv != bv;
  if (vn || bn) return vn && (!bn || i < bi);
  return v > bv || (v == bv && i < bi);
}

// Reference version: one warp per flagged (atom, frame), lane = TDOA (+ 32 j), every bin's row of E read from L2 by every
// warp (13 485 pairs x 513 rows x 1 KB = 7 GB of L2 reads at the headline shape: L2-bandwidth bound, 0.8 ms).
__global__ void __launch_bounds__(256)
refine_argmax_kernel(const int2* __restrict__ list, const int* __restrict__ count, int capacity, const float2* __restrict__ coh,
                     int F, int T, const double2* __restrict__ E, int D, const float* __restrict__ W, int K, int32_t* __restrict__ argmax) {
  const int lane = threadIdx.x & 31;
  const int warps = gridDim.x * (blockDim.x >> 5);
  const int n = min(*count, capacity);
  for (int p = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); p < n; p += warps) {
    const int k = list[p].x, t = list[p].y;
    double acc[4] = {0.0, 0.0, 0.0, 0.0};   // TDOAs lane, lane + 32, lane + 64, lane + 96 (D <= 128)
    for (int f = 0; f < F; ++f) {
      const float2 c = __ldg(coh + (int64_t)f * T + t);
      const double w = (double)__ldg(W + (int64_t)f * K + k);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int d = lane + 32 * j;
        if (d < D) {
          const double2 e = __ldg(E + (int64_t)f * D + d);
          acc[j] = fma((double)c.x * e.x - (double)c.y * e.y, w, acc[j]);
        }
      }
    }
    double bv = acc[0];
    int bi = lane;
#pragma unroll
    for (int j = 1; j < 4; ++j)
      if (lane + 32 * j < D && argmax_better64(acc[j], lane + 32 * j, bv, bi)) { bv = acc[j]; bi = lane + 32 * j; }
    if (lane >= D) { bv = -INFINITY; bi = 1 << 30; }
    for (int o = 16; o > 0; o >>= 1) {
      const double ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (argmax_better64(ov, oi, bv, bi)) { bv = ov; bi = oi; }
    }
    if (lane == 0) argmax[(int64_t)k * T + t] = bi;
  }
}


// Same arithmetic (bin order, one fma per bin: the float64 kernel's), with E staged through shared memory in chunks of
// kRefineChunk bins and shared by the CTA's 8 warps x 4 pairs per warp: 32 x less L2 traffic for E.  The (strided)
// coherence and W values of a chunk are fetched by the lanes -- lane l < 16: coherence of bin l for the warp's 4 pairs,
// lane 16 + l: W -- and broadcast with shuffles.
constexpr int kRefineChunk = 16, kRefinePairs = 4;
__global__ void __launch_bounds__(256)
refine_argmax_shared_kernel(const int2* __restrict__ list, const int* __restrict__ count, int capacity, const float2* __restrict__ coh,
                            int F, int T, const double2* __restrict__ E, int D, const float* __restrict__ W, int K, int32_t* __restrict__ argmax) {
  __shared__ double2 Es[kRefineChunk][64];        // D <= 64
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n = min(*count, capacity);
  const int per_cta = 8 * kRefinePairs;
  for (int base = blockIdx.x * per_cta; base < n; base += gridDim.x * per_cta) {      // (uniform per CTA: the barriers below are safe)
    int pk[kRefinePairs], pt[kRefinePairs];
#pragma unroll
    for (int p = 0; p < kRefinePairs; ++p) {
      const int idx = base + warp * kRefinePairs + p;
      const int2 kt = idx < n ? list[idx] : make_int2(0, 0);
      pk[p] = kt.x; pt[p] = kt.y;
    }
    double acc[kRefinePairs][2];
#pragma unroll
    for (int p = 0; p < kRefinePairs; ++p) { acc[p][0] = 0.0; acc[p][1] = 0.0; }
    for (int f0 = 0; f0 < F; f0 += kRefineChunk) {
      __syncthreads();                            // the previous chunk has been consumed
      for (int i = threadIdx.x; i < kRefineChunk * 64; i += 256) {
        const int fl = i >> 6, d = i & 63, f = f0 + fl;
        Es[fl][d] = (f < F && d < D) ? __ldg(E + (int64_t)f * D + d) : double2{0.0, 0.0};
      }
      // lane l < 16: coherence of bin f0 + l; lane >= 16: W of bin f0 + l - 16 (both for the warp's 4 pairs)
      const int fm = min(f0 + (lane & 15), F - 1);
      float cx[kRefinePairs], cy[kRefinePairs];   // (for lanes >= 16, cx carries W)
#pragma unroll
      for (int p = 0; p < kRefinePairs; ++p) {
        if (lane < 16) {
          const float2 c = __ldg(coh + (int64_t)fm * T + pt[p]);
          cx[p] = c.x; cy[p] = c.y;
        } else {
          cx[p] = __ldg(W + (int64_t)fm * K + pk[p]);
          cy[p] = 0.f;
        }
      }
      __syncthreads();
      const int fcount = min(kRefineChunk, F - f0);
      for (int fl = 0; fl < fcount; ++fl) {
        const double2 e0 = Es[fl][lane], e1 = Es[fl][lane + 32];
#pragma unroll
        for (int p = 0; p < kRefinePairs; ++p) {
          const double c_re = (double)__shfl_sync(0xffffffffu, cx[p], fl), c_im = (double)__shfl_sync(0xffffffffu, cy[p], fl);
          const double wd = (double)__shfl_sync(0xffffffffu, cx[p], 16 + fl);
          acc[p][0] = fma(c_re * e0.x - c_im * e0.y, wd, acc[p][0]);
          acc[p][1] = fma(c_re * e1.x - c_im * e1.y, wd, acc[p][1]);
        }
      }
    }
#pragma unroll
    for (int p = 0; p < kRefinePairs; ++p) {
      double bv = acc[p][0];
      int bi = lane;
      if (lane + 32 < D && argmax_better64(acc[p][1], lane + 32, bv, bi)) { bv = acc[p][1]; bi = lane + 32; }
      if (lane >= D) { bv = -INFINITY; bi = 1 << 30; }
      for (int o = 16; o > 0; o >>= 1) {
        const double ov = __shfl_xor_sync(0xffffffffu, bv, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (argmax_better64(ov, oi, bv, bi)) { bv = ov; bi = oi; }
      }
      const int idx = base + warp * kRefinePairs + p;
      if (lane == 0 && idx < n) argmax[(int64_t)pk[p] * T + pt[p]] = bi;
    }
  }
}

__global__ void abs_colsum_kernel(const float* __restrict__ W, int F, int K, float* __restrict__ colsum) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= K) return;
  float s = 0.f;
  for (int f = 0; f < F; ++f) s += fabsf(W[(int64_t)f * K + k]);
  colsum[k] = s;
}

// Candidate refinement (the default): the GEMM epilogue leaves, per flagged (atom, frame), the set of TDOAs whose value lies within
// the margin of the best -- 2 or 3 of D as a rule -- and only those are recomputed in float64.  One warp per pair.  The lanes load
// 32 consecutive bins of TRANSPOSED copies of the coherence (T, F), W (K, F) and E (D, F), so every load of a warp is one contiguous
// row segment (the first version gathered: 700 MB of 32-byte sectors at the headline shape), form Re(C E) of their bin for each
// candidate and stage it in shared memory; lane j then adds the 32 bins into candidate j's sum, one fma per bin in bin order.  So
// every candidate is ONE fma chain over f = 0 .. F - 1, the float64 kernel's summation order (tdoa_gccnmf_kernel, gcc.cu): values
// that differ only at float64 rounding level -- the two central TDOAs of mono input -- are ordered exactly as it orders them.
// (Lane-strided partial sums added by a shuffle tree, the previous form, round differently and flipped such decisions.)  The next
// 32 bins are loaded while the chains run.
constexpr int kRefineGroup = 8;        // candidates per pass over the bins
__global__ void __launch_bounds__(256)
refine_candidates_kernel(const int2* __restrict__ list, const uint4* __restrict__ candidates, const int* __restrict__ count, int capacity,
                         const float2* __restrict__ cohT, const float* __restrict__ WT, const double2* __restrict__ ET, int F, int64_t Fp, int D,
                         int T, int32_t* __restrict__ argmax) {
  __shared__ double re_s[8][kRefineGroup][33];     // per warp: Re(C E) of 32 bins per candidate (row padded: conflict-free reads)
  __shared__ double w_s[8][32];                    // per warp: W of the 32 bins
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  double (*re)[33] = re_s[wib];
  double* wv = w_s[wib];
  const int warps = gridDim.x * (blockDim.x >> 5);
  const int n = min(*count, capacity);
  for (int p = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); p < n; p += warps) {
    const int k = list[p].x, t = list[p].y;
    const uint4 c4 = candidates[p];
    uint32_t bits[4] = {c4.x, c4.y, c4.z, c4.w};
    const float2* crow = cohT + (int64_t)t * Fp;
    const float* wrow = WT + (int64_t)k * Fp;
    double bv = 0.0;
    int bi = -1;
    int word = 0;
    while (true) {
      int ds[kRefineGroup], nd = 0;                       // the next <= 8 candidate TDOAs, ascending (warp-uniform)
      while (nd < kRefineGroup && word < 4) {
        if (bits[word] == 0u) { ++word; continue; }
        const int b = __ffs(bits[word]) - 1;
        bits[word] &= bits[word] - 1;
        ds[nd++] = word * 32 + b;
      }
      if (nd == 0) break;
      double g[kRefineGroup], w = 0.0;                    // this lane's bin of the chunk: Re(C E) per candidate, W
      auto load = [&](int f0) {
        const int f = f0 + lane;
        if (f >= F) return;
        const float2 c = crow[f];
        w = (double)wrow[f];
#pragma unroll
        for (int j = 0; j < kRefineGroup; ++j)
          if (j < nd) {
            const double2 e = ET[(int64_t)ds[j] * Fp + f];
            g[j] = (double)c.x * e.x - (double)c.y * e.y;
          }
      };
      load(0);
      double acc = 0.0;                                   // lane j < nd: candidate ds[j]
      for (int f0 = 0; f0 < F; f0 += 32) {
#pragma unroll
        for (int j = 0; j < kRefineGroup; ++j)
          if (j < nd) re[j][lane] = g[j];
        wv[lane] = w;
        __syncwarp();
        if (f0 + 32 < F) load(f0 + 32);
        if (lane < nd) {
          const double* r = re[lane];
          if (F - f0 >= 32) {
#pragma unroll 8
            for (int s = 0; s < 32; ++s) acc = fma(r[s], wv[s], acc);
          } else {
            for (int s = 0; s < F - f0; ++s) acc = fma(r[s], wv[s], acc);
          }
        }
        __syncwarp();
      }
#pragma unroll
      for (int j = 0; j < kRefineGroup; ++j) {            // ascending TDOAs: numpy's first-maximum rule
        if (j < nd) {
          const double v = __shfl_sync(0xffffffffu, acc, j);
          if (bi < 0 || argmax_better64(v, ds[j], bv, bi)) { bv = v; bi = ds[j]; }
        }
      }
    }
    if (lane == 0 && bi >= 0) argmax[(int64_t)k * T + t] = bi;
  }
}

// refine_candidates_kernel for a steering bank: a pair reads the transposed table of its column's entry.
__global__ void __launch_bounds__(256)
refine_candidates_bank_kernel(const int2* __restrict__ list, const uint4* __restrict__ candidates, const int* __restrict__ count, int capacity,
                              const float2* __restrict__ cohT, const float* __restrict__ WT, SteerBank bank, int F, int64_t Fp, int D,
                              int T, int32_t* __restrict__ argmax) {
  __shared__ double re_s[8][kRefineGroup][33];     // per warp: Re(C E) of 32 bins per candidate (row padded: conflict-free reads)
  __shared__ double w_s[8][32];                    // per warp: W of the 32 bins
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  double (*re)[33] = re_s[wib];
  double* wv = w_s[wib];
  const int warps = gridDim.x * (blockDim.x >> 5);
  const int n = min(*count, capacity);
  for (int p = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); p < n; p += warps) {
    const int k = list[p].x, t = list[p].y;
    const uint4 c4 = candidates[p];
    uint32_t bits[4] = {c4.x, c4.y, c4.z, c4.w};
    const float2* crow = cohT + (int64_t)t * Fp;
    const float* wrow = WT + (int64_t)k * Fp;
    const double2* ET = bank.ET + (int64_t)bank.entry(t) * D * Fp;      // the pair's table, transposed
    double bv = 0.0;
    int bi = -1;
    int word = 0;
    while (true) {
      int ds[kRefineGroup], nd = 0;                       // the next <= 8 candidate TDOAs, ascending (warp-uniform)
      while (nd < kRefineGroup && word < 4) {
        if (bits[word] == 0u) { ++word; continue; }
        const int b = __ffs(bits[word]) - 1;
        bits[word] &= bits[word] - 1;
        ds[nd++] = word * 32 + b;
      }
      if (nd == 0) break;
      double g[kRefineGroup], w = 0.0;                    // this lane's bin of the chunk: Re(C E) per candidate, W
      auto load = [&](int f0) {
        const int f = f0 + lane;
        if (f >= F) return;
        const float2 c = crow[f];
        w = (double)wrow[f];
#pragma unroll
        for (int j = 0; j < kRefineGroup; ++j)
          if (j < nd) {
            const double2 e = ET[(int64_t)ds[j] * Fp + f];
            g[j] = (double)c.x * e.x - (double)c.y * e.y;
          }
      };
      load(0);
      double acc = 0.0;                                   // lane j < nd: candidate ds[j]
      for (int f0 = 0; f0 < F; f0 += 32) {
#pragma unroll
        for (int j = 0; j < kRefineGroup; ++j)
          if (j < nd) re[j][lane] = g[j];
        wv[lane] = w;
        __syncwarp();
        if (f0 + 32 < F) load(f0 + 32);
        if (lane < nd) {
          const double* r = re[lane];
          if (F - f0 >= 32) {
#pragma unroll 8
            for (int s = 0; s < 32; ++s) acc = fma(r[s], wv[s], acc);
          } else {
            for (int s = 0; s < F - f0; ++s) acc = fma(r[s], wv[s], acc);
          }
        }
        __syncwarp();
      }
#pragma unroll
      for (int j = 0; j < kRefineGroup; ++j) {            // ascending TDOAs: numpy's first-maximum rule
        if (j < nd) {
          const double v = __shfl_sync(0xffffffffu, acc, j);
          if (bi < 0 || argmax_better64(v, ds[j], bv, bi)) { bv = v; bi = ds[j]; }
        }
      }
    }
    if (lane == 0 && bi >= 0) argmax[(int64_t)k * T + t] = bi;
  }
}

// refine_candidates_bank_kernel for a dictionary bank: a pair also reads the transposed W of its column's dictionary.
__global__ void __launch_bounds__(256)
refine_candidates_dict_kernel(const int2* __restrict__ list, const uint4* __restrict__ candidates, const int* __restrict__ count, int capacity,
                              const float2* __restrict__ cohT, DictBank dict, SteerBank bank, int F, int64_t Fp, int D, int T,
                              int32_t* __restrict__ argmax) {
  __shared__ double re_s[8][kRefineGroup][33];
  __shared__ double w_s[8][32];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  double (*re)[33] = re_s[wib];
  double* wv = w_s[wib];
  const int warps = gridDim.x * (blockDim.x >> 5);
  const int n = min(*count, capacity);
  for (int p = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); p < n; p += warps) {
    const int k = list[p].x, t = list[p].y;
    const uint4 c4 = candidates[p];
    uint32_t bits[4] = {c4.x, c4.y, c4.z, c4.w};
    const float2* crow = cohT + (int64_t)t * Fp;
    const float* wrow = dict.WT + ((int64_t)dict.entry(t) * dict.Kp + k) * Fp;
    const double2* ET = bank.ET + (int64_t)bank.entry(t) * D * Fp;
    double bv = 0.0;
    int bi = -1;
    int word = 0;
    while (true) {
      int ds[kRefineGroup], nd = 0;
      while (nd < kRefineGroup && word < 4) {
        if (bits[word] == 0u) { ++word; continue; }
        const int b = __ffs(bits[word]) - 1;
        bits[word] &= bits[word] - 1;
        ds[nd++] = word * 32 + b;
      }
      if (nd == 0) break;
      double g[kRefineGroup], w = 0.0;
      auto load = [&](int f0) {
        const int f = f0 + lane;
        if (f >= F) return;
        const float2 c = crow[f];
        w = (double)wrow[f];
#pragma unroll
        for (int j = 0; j < kRefineGroup; ++j)
          if (j < nd) {
            const double2 e = ET[(int64_t)ds[j] * Fp + f];
            g[j] = (double)c.x * e.x - (double)c.y * e.y;
          }
      };
      load(0);
      double acc = 0.0;
      for (int f0 = 0; f0 < F; f0 += 32) {
#pragma unroll
        for (int j = 0; j < kRefineGroup; ++j)
          if (j < nd) re[j][lane] = g[j];
        wv[lane] = w;
        __syncwarp();
        if (f0 + 32 < F) load(f0 + 32);
        if (lane < nd) {
          const double* r = re[lane];
          if (F - f0 >= 32) {
#pragma unroll 8
            for (int s = 0; s < 32; ++s) acc = fma(r[s], wv[s], acc);
          } else {
            for (int s = 0; s < F - f0; ++s) acc = fma(r[s], wv[s], acc);
          }
        }
        __syncwarp();
      }
#pragma unroll
      for (int j = 0; j < kRefineGroup; ++j) {
        if (j < nd) {
          const double v = __shfl_sync(0xffffffffu, acc, j);
          if (bi < 0 || argmax_better64(v, ds[j], bv, bi)) { bv = v; bi = ds[j]; }
        }
      }
    }
    if (lane == 0 && bi >= 0) argmax[(int64_t)k * T + t] = bi;
  }
}

// A dictionary's bf16 planes: columns [e Kp, e Kp + Kp) of the (F, Qd Kp) planes, W (F, K) as it lies, zero past K.
__global__ void split_dict_planes_kernel(const float* __restrict__ W, int F, int K, int Kp, int64_t ld, bf16* __restrict__ planes, int64_t plane) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)F * Kp) return;
  const int f = (int)(i / Kp), k = (int)(i - (int64_t)f * Kp);
  bf16 hi, lo;
  split_bf16(k < K ? W[(int64_t)f * K + k] : 0.f, hi, lo);
  planes[(int64_t)f * ld + k] = hi;
  planes[plane + (int64_t)f * ld + k] = lo;
}

// dst (cols, ld) = src (rows, cols)^T for 4-, 8- and 16-byte elements (zero in the pad columns [rows, ld))
template <typename E>
__global__ void transpose_pad_kernel(const E* __restrict__ src, int rows, int cols, E* __restrict__ dst, int64_t ld) {
  __shared__ E tile[32][33];
  const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int r = r0 + i, c = c0 + threadIdx.x;
    tile[i][threadIdx.x] = (r < rows && c < cols) ? src[(int64_t)r * cols + c] : E{};
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, r = r0 + threadIdx.x;
    if (c < cols && r < ld) dst[(int64_t)c * ld + r] = tile[threadIdx.x][i];
  }
}

constexpr int kArgmaxTile = 256;       // columns (frame, TDOA) per tile: 256 / D whole frames

struct ArgmaxWorkspace {
  bf16 *Gp, *Wp;
  float *colsum, *WT;
  float2* cohT;
  double2* ET;
  int2* list;
  uint4* cand;
  int* count;
  int64_t Fp, plane_g, plane_w;
  int capacity;
  bool ok;
};

int list_capacity(int K, int T) { return (int)std::min<int64_t>((int64_t)K * T, std::max<int64_t>(1 << 16, (int64_t)K * T / 8)); }

ArgmaxWorkspace carve_argmax(void* ws, size_t bytes, int F, int T, int D, int K) {
  WorkspaceCarver c(ws ? ws : reinterpret_cast<void*>(256), ws ? bytes : ~size_t(0) >> 1);
  ArgmaxWorkspace w;
  w.Fp = (F + 7) & ~7;
  w.plane_g = (int64_t)T * D * w.Fp;
  w.plane_w = (int64_t)F * K;
  w.capacity = list_capacity(K, T);
  w.Gp = c.take<bf16>((size_t)2 * w.plane_g);
  w.Wp = c.take<bf16>((size_t)2 * w.plane_w);
  w.colsum = c.take<float>(K);
  w.ET = c.take<double2>((size_t)D * w.Fp);
  w.cand = c.take<uint4>(w.capacity);
  w.cohT = c.take<float2>((size_t)T * w.Fp);
  w.WT = c.take<float>((size_t)K * w.Fp);
  w.list = c.take<int2>(w.capacity);
  w.count = c.take<int>(4);
  w.ok = ws != nullptr && c.ok();
  w.plane_g = (int64_t)T * D * w.Fp;
  return w;
}
size_t argmax_workspace_bytes(int F, int T, int D, int K) {
  WorkspaceCarver c(reinterpret_cast<void*>(256), ~size_t(0) >> 1);
  const size_t Fp = (F + 7) & ~7;
  c.take<bf16>((size_t)2 * T * D * Fp); c.take<bf16>((size_t)2 * F * K); c.take<float>(K); c.take<double2>((size_t)D * Fp);
  c.take<uint4>(list_capacity(K, T)); c.take<float2>((size_t)T * Fp); c.take<float>((size_t)K * Fp); c.take<int2>(list_capacity(K, T)); c.take<int>(4);
  return align_up(c.used, 256);
}

// ------------------------------------------------------------------ a8: masked reconstruction on the plane GEMM
// est[s][c] (F, T) = (W . (H_c * M_s)) * exp(j angle(X_c))  (gccNMFFunctions.py:150-151), computed transposed so that every operand
// is consumed as it lies:  D[m = (batch b = 2 s + c, t), n = f] = sum_k A(m, k) B(f, k),  A = masked H planes (K rows, frames
// contiguous: MN-major; the batches are stacked along m, each padded to whole 128-frame tiles), B = W planes (F, K): K-major.
// The by-column epilogue owns 4 consecutive frames of one bin: one 32-byte complex64 segment of est per lane.
__global__ void masked_h_planes_kernel(const float* __restrict__ H, const float* __restrict__ masks, int S, int K, int T, int Tpad,
                                       bf16* __restrict__ planes, int64_t pitch, int64_t plane) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)K * pitch) return;
  const int k = (int)(i / pitch), col = (int)(i - (int64_t)k * pitch);
  const int b = col / Tpad, t = col - b * Tpad;
  float v = 0.f;
  if (t < T) v = H[(int64_t)k * (2 * T) + (int64_t)(b & 1) * T + t] * masks[((int64_t)(b >> 1) * K + k) * T + t];   // H_c * M_s
  bf16 hi, lo;
  split_bf16(v, hi, lo);
  planes[i] = hi;
  planes[plane + i] = lo;
  (void)S;
}

struct EpiReconPhase {
  struct State {};
  struct Loaded { float4 x01, x23; };
  static constexpr bool kRowReduce = false;
  static constexpr int kRowValues = 0;
  static constexpr bool kPrefetch = false;
  const float2* __restrict__ X;    // (2, F, T)
  float2* __restrict__ out;        // (S, 2, F, T)
  int F, T, Tpad, M; bool vec;     // M = batches * Tpad
  __device__ void prefetch(int, int) const {}
  __device__ void row_values(int, float*) const {}
  __device__ void init(State&, int, const float*) const {}
  __device__ float4 row_partial(const State&) const { return make_float4(0.f, 0.f, 0.f, 0.f); }
  __device__ void row_total(int, int, float) const {}
  __device__ void elem(int, int, float, int) const {}
  // exp(1j * angle(X)) (gccNMFFunctions.py:151): unit phasor of the mixture bin; angle(0) = 0
  __device__ static float2 phase_times(float a, float2 x) {
    const double mag = sqrt((double)x.x * x.x + (double)x.y * x.y);
    float pr = 1.f, pi = 0.f;
    if (mag > 0.0) { pr = (float)((double)x.x / mag); pi = (float)((double)x.y / mag); }
    else if (mag != mag) { pr = pi = __int_as_float(0x7fc00000); }
    return float2{a * pr, a * pi};
  }
  __device__ Loaded load(int m, int n) const {
    Loaded l;
    l.x01 = l.x23 = make_float4(0.f, 0.f, 0.f, 0.f);
    if (m >= M) return l;
    const int b = m / Tpad, t = m - b * Tpad;
    const float2* src = X + ((int64_t)(b & 1) * F + n) * T + t;
    if (vec && t + 4 <= T) {
      l.x01 = *reinterpret_cast<const float4*>(src);
      l.x23 = *reinterpret_cast<const float4*>(src + 2);
    } else {
      float2 v[4] = {{0.f, 0.f}, {0.f, 0.f}, {0.f, 0.f}, {0.f, 0.f}};
      for (int i = 0; i < 4; ++i)
        if (t + i < T) v[i] = src[i];
      l.x01 = make_float4(v[0].x, v[0].y, v[1].x, v[1].y);
      l.x23 = make_float4(v[2].x, v[2].y, v[3].x, v[3].y);
    }
    return l;
  }
  __device__ void store(int m, int n, const float4& acc, const Loaded& l, int, State&) const {
    if (m >= M) return;
    const int b = m / Tpad, t = m - b * Tpad;      // (Tpad is a multiple of 4: the 4 rows of a lane lie in one batch)
    if (t >= T) return;
    float2* dst = out + ((int64_t)b * F + n) * T + t;
    const float2 r0 = phase_times(acc.x, float2{l.x01.x, l.x01.y}), r1 = phase_times(acc.y, float2{l.x01.z, l.x01.w});
    const float2 r2 = phase_times(acc.z, float2{l.x23.x, l.x23.y}), r3 = phase_times(acc.w, float2{l.x23.z, l.x23.w});
    if (vec && t + 4 <= T) {
      *reinterpret_cast<float4*>(dst) = make_float4(r0.x, r0.y, r1.x, r1.y);
      *reinterpret_cast<float4*>(dst + 2) = make_float4(r2.x, r2.y, r3.x, r3.y);
    } else {
      const float2 r[4] = {r0, r1, r2, r3};
      for (int i = 0; i < 4; ++i)
        if (t + i < T) dst[i] = r[i];
    }
  }
};

struct ReconWorkspace {
  bf16 *Ap, *Wp;
  int64_t pitch, plane_a, plane_w;
  int Tpad;
  size_t bytes;
  bool ok;
};
ReconWorkspace carve_recon(void* ws, size_t bytes, int S, int F, int T, int K) {
  WorkspaceCarver c(ws ? ws : reinterpret_cast<void*>(256), ws ? bytes : ~size_t(0) >> 1);
  ReconWorkspace w;
  w.Tpad = (T + tgemm::kBM - 1) / tgemm::kBM * tgemm::kBM;
  w.pitch = (int64_t)2 * S * w.Tpad;
  w.plane_a = (int64_t)K * w.pitch;
  w.plane_w = (int64_t)F * K;
  w.Ap = c.take<bf16>((size_t)2 * w.plane_a);
  w.Wp = c.take<bf16>((size_t)2 * w.plane_w);
  w.bytes = align_up(c.used, 256);
  w.ok = ws != nullptr && c.ok();
  return w;
}

}  // namespace

// gcc.cu
int gccnmf_tdoa_gccnmf_bank(gccnmf_handle* h, const float* coherence, int F, int T, const SteerBank& bank, int D, const float* W, int K,
                            int32_t* argmax, const int32_t* gate, int capacity, int32_t* ran, void* stream);

bool gccnmf_tdoa_argmax_tc_supported(int F, int T, int D, int K) {
  const bool d_ok = D >= 8 && D <= 128 && (D & (D - 1)) == 0;          // whole frames per 256-column tile; refinement kernels: D <= 128
  return d_ok && K % 8 == 0 && K >= 64 && F >= 32 && (int64_t)T * D >= kArgmaxTile && (int64_t)T * D < ((int64_t)1 << 31);
}
bool gccnmf_masked_recon_tc_supported(int S, int F, int T, int K) { return S >= 1 && K % 8 == 0 && K >= 64 && F >= 64 && T >= 64; }

extern "C" {

int gccnmf_tdoa_argmax_refine_capacity(int K, int T) { return (K > 0 && T > 0) ? list_capacity(K, T) : 0; }

size_t gccnmf_tdoa_argmax_workspace_bytes(int F, int T, int D, int K) {
  if (F <= 0 || T <= 0 || D <= 0 || K <= 0) return 0;
  if (!gccnmf_tdoa_argmax_tc_supported(F, T, D, K)) return 256;
  return argmax_workspace_bytes(F, T, D, K);
}

}  // extern "C"

// gccnmf_tdoa_argmax, or with `bank` its form for a steering bank (E unused): only the plane build, the refinement and the float64
// fallback read the tables; the GEMM and its epilogue see G alone.  A bank always takes the candidate refinement, over the
// transposed tables it keeps (every refinement form gives the float64 decision).
static int tdoa_argmax(gccnmf_handle* h, const float* coherence, int F, int T, const double* E, const SteerBank* bank, int D, const float* W, int K,
                       int32_t* argmax, int32_t* overflow_flag, void* workspace, size_t workspace_bytes, void* stream) {
  GCCNMF_ENTER(h);
  GCCNMF_REQUIRE(h, F > 0 && T > 0 && D > 0 && K > 0 && coherence && (E || bank) && W && argmax, "tdoa_argmax: bad arguments");
  if (h->force_simt_nmf || !gccnmf_tdoa_argmax_tc_supported(F, T, D, K)) {
    // exact float64 SIMT kernel: nothing to refine, and the caller must not read an unwritten counter
    if (overflow_flag) GCCNMF_CHECK_CUDA(h, cudaMemsetAsync(overflow_flag, 0, sizeof(int32_t), (cudaStream_t)stream));
    if (bank) return gccnmf_tdoa_gccnmf_bank(h, coherence, F, T, *bank, D, W, K, argmax, nullptr, 0, nullptr, stream);
    return gccnmf_tdoa_gccnmf(h, coherence, F, T, E, D, W, K, nullptr, argmax, stream);
  }
  ArgmaxWorkspace w = carve_argmax(workspace, workspace_bytes, F, T, D, K);
  if (!w.ok) return gccnmf_fail(h, GCCNMF_ERR_WORKSPACE, "tdoa_argmax workspace too small: need %zu bytes", gccnmf_tdoa_argmax_workspace_bytes(F, T, D, K));
  GCCNMF_REQUIRE(h, !bank || bank->Fp == w.Fp, "tdoa_argmax: the bank's transposed tables have %lld bins, the workspace %lld",
                 (long long)(bank ? bank->Fp : 0), (long long)w.Fp);
  GCCNMF_CHECK_CUDA(h, cudaMemsetAsync(w.count, 0, 16, (cudaStream_t)stream));
  if (bank)
    GCCNMF_LAUNCH(h, build_gcc_planes_bank_kernel, dim3((int)((w.Fp + 63) / 64), steer_tiles_max(T, 32, bank->Qe)), 256, 0, stream,
                  reinterpret_cast<const float2*>(coherence), F, T, *bank, D, w.Gp, w.Fp, w.plane_g);
  else
    GCCNMF_LAUNCH(h, build_gcc_planes_kernel, dim3((int)((w.Fp + 63) / 64), (T + 31) / 32), 256, 0, stream,
                  reinterpret_cast<const float2*>(coherence), F, T, reinterpret_cast<const double2*>(E), D, w.Gp, w.Fp, w.plane_g);
  const int64_t nw = (int64_t)F * K;
  GCCNMF_LAUNCH(h, split_to_planes_kernel, (unsigned)((nw + 255) / 256), 256, 0, stream, W, nw, w.Wp, w.plane_w);
  GCCNMF_LAUNCH(h, abs_colsum_kernel, (K + 127) / 128, 128, 0, stream, W, F, K, w.colsum);
  const int N = T * D;
  const Operand Wmn{w.Wp, (int64_t)K, w.plane_w, true};          // A(m = atom, k = f): (F, K) as it lies
  const Operand Gk{w.Gp, w.Fp, w.plane_g, false};                // B(n = (t, tau), k = f)
  EpiArgmaxTile epi{argmax, w.colsum, w.list, w.cand, w.count, w.capacity, K, T, D, margin_factor(F)};
  if (h->argmax_persistent && D >= 32) {
    CUtensorMap map_a, map_b;
    if (int st = tmap_mnmajor(h, Wmn.planes, K, F, Wmn.pitch, Wmn.plane, &map_a)) return st;
    if (int st = tmap_kmajor(h, Gk.planes, N, F, Gk.pitch, Gk.plane, kPersBN, &map_b)) return st;
    const int m_tiles = (K + tgemm::kBM - 1) / tgemm::kBM, n_tiles = (N + kPersBN - 1) / kPersBN;
    const int st = D == 32 ? launch_argmax_persistent<32>(h, map_a, map_b, K, N, F, m_tiles, n_tiles, epi, stream)
                 : D == 64 ? launch_argmax_persistent<64>(h, map_a, map_b, K, N, F, m_tiles, n_tiles, epi, stream)
                           : launch_argmax_persistent<128>(h, map_a, map_b, K, N, F, m_tiles, n_tiles, epi, stream);
    if (st) return st;
  } else if (int st = plane_gemm<true, false>(h, kArgmaxTile, Wmn, Gk, K, N, F, 1, false, epi, nullptr, stream, true)) {
    return st;
  }
  if (bank) {
    const dim3 tb(32, 8);
    GCCNMF_LAUNCH(h, transpose_pad_kernel<float2>, dim3((T + 31) / 32, (int)((w.Fp + 31) / 32)), tb, 0, stream, reinterpret_cast<const float2*>(coherence), F,
                  T, w.cohT, w.Fp);
    GCCNMF_LAUNCH(h, transpose_pad_kernel<float>, dim3((K + 31) / 32, (int)((w.Fp + 31) / 32)), tb, 0, stream, W, F, K, w.WT, w.Fp);
    GCCNMF_LAUNCH(h, refine_candidates_bank_kernel, h->sm_count * 8, 256, 0, stream, w.list, w.cand, w.count, w.capacity, w.cohT, w.WT, *bank, F, w.Fp, D,
                  T, argmax);
  } else if (h->argmax_refine_shared) {
    // candidate refinement over transposed copies (contiguous loads); argmax_refine_shared = 0 selects the all-TDOA kernels below
    const dim3 tb(32, 8);
    GCCNMF_LAUNCH(h, transpose_pad_kernel<float2>, dim3((T + 31) / 32, (int)((w.Fp + 31) / 32)), tb, 0, stream, reinterpret_cast<const float2*>(coherence), F,
                  T, w.cohT, w.Fp);
    GCCNMF_LAUNCH(h, transpose_pad_kernel<float>, dim3((K + 31) / 32, (int)((w.Fp + 31) / 32)), tb, 0, stream, W, F, K, w.WT, w.Fp);
    GCCNMF_LAUNCH(h, transpose_pad_kernel<double2>, dim3((D + 31) / 32, (int)((w.Fp + 31) / 32)), tb, 0, stream, reinterpret_cast<const double2*>(E), F, D,
                  w.ET, w.Fp);
    GCCNMF_LAUNCH(h, refine_candidates_kernel, h->sm_count * 8, 256, 0, stream, w.list, w.cand, w.count, w.capacity, w.cohT, w.WT, w.ET, F, w.Fp, D, T,
                  argmax);
  } else if (D <= 64) {
    GCCNMF_LAUNCH(h, refine_argmax_shared_kernel, h->sm_count * 4, 256, 0, stream, w.list, w.count, w.capacity,
                  reinterpret_cast<const float2*>(coherence), F, T, reinterpret_cast<const double2*>(E), D, W, K, argmax);
  } else {
    GCCNMF_LAUNCH(h, refine_argmax_kernel, h->sm_count * 4, 256, 0, stream, w.list, w.count, w.capacity,
                  reinterpret_cast<const float2*>(coherence), F, T, reinterpret_cast<const double2*>(E), D, W, K, argmax);
  }
  // more near-ties than the list holds (at least 1/8 of all decisions): the caller must fall back to the float64 kernel.  Mono input
  // (identical channels) gets there: the two central TDOAs of the symmetric grid tie in nearly every decision.
  if (overflow_flag) GCCNMF_CHECK_CUDA(h, cudaMemcpyAsync(overflow_flag, w.count, sizeof(int), cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return GCCNMF_OK;
}

extern "C" {

int gccnmf_tdoa_argmax(gccnmf_handle* h, const float* coherence, int F, int T, const double* E, int D, const float* W, int K,
                       int32_t* argmax, int32_t* overflow_flag, void* workspace, size_t workspace_bytes, void* stream) {
  return tdoa_argmax(h, coherence, F, T, E, nullptr, D, W, K, argmax, overflow_flag, workspace, workspace_bytes, stream);
}

size_t gccnmf_masked_recon_workspace_bytes(int S, int F, int T, int K) {
  if (S <= 0 || F <= 0 || T <= 0 || K <= 0 || !gccnmf_masked_recon_tc_supported(S, F, T, K)) return 256;
  return carve_recon(nullptr, 0, S, F, T, K).bytes;
}

// Tensor-core masked reconstruction (gccnmf_masked_recon_phase routes here when the shape is covered and a workspace is given).
int gccnmf_masked_recon_planes(gccnmf_handle* h, const float* masks, const float* X, const float* W, const float* H, int S, int F, int T, int K,
                               float* out, void* workspace, size_t workspace_bytes, void* stream) {
  ReconWorkspace w = carve_recon(workspace, workspace_bytes, S, F, T, K);
  if (!w.ok) return gccnmf_fail(h, GCCNMF_ERR_WORKSPACE, "masked_recon workspace too small: need %zu bytes", w.bytes);
  const int64_t na = (int64_t)K * w.pitch, nw = (int64_t)F * K;
  GCCNMF_LAUNCH(h, masked_h_planes_kernel, (unsigned)((na + 255) / 256), 256, 0, stream, H, masks, S, K, T, w.Tpad, w.Ap, w.pitch, w.plane_a);
  GCCNMF_LAUNCH(h, split_to_planes_kernel, (unsigned)((nw + 255) / 256), 256, 0, stream, W, nw, w.Wp, w.plane_w);
  const int M = 2 * S * w.Tpad;
  const Operand Amn{w.Ap, w.pitch, w.plane_a, true};             // A(m = (batch, t), k = atom): (K, batches x Tpad) as built
  const Operand Wk{w.Wp, (int64_t)K, w.plane_w, false};          // B(n = f, k = atom)
  EpiReconPhase epi{reinterpret_cast<const float2*>(X), reinterpret_cast<float2*>(out), F, T, w.Tpad, M,
                    T % 4 == 0 && (reinterpret_cast<uintptr_t>(X) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0};
  // tile width over the F bins: the smallest of the instantiated widths whose tiles waste the fewest columns
  const int widths[4] = {128, 176, 208, 256};
  int bn = 128, best = 1 << 30;
  for (int i = 0; i < 4; ++i) {
    const int waste = (F + widths[i] - 1) / widths[i] * widths[i] - F;
    if (waste < best) { best = waste; bn = widths[i]; }
  }
  return plane_gemm<true, false>(h, bn, Amn, Wk, M, F, K, 1, false, epi, nullptr, stream, false, bn > tgemm::kBM);   // pairs for wide tiles
}

}  // extern "C"

// gccnmf_tdoa_argmax for a steering bank (gccnmf_llbank_*): the same workspace, bank.Fp = (F + 7) & ~7.
int gccnmf_tdoa_argmax_bank(gccnmf_handle* h, const float* coherence, int F, int T, const SteerBank& bank, int D, const float* W, int K,
                            int32_t* argmax, int32_t* overflow_flag, void* workspace, size_t workspace_bytes, void* stream) {
  return tdoa_argmax(h, coherence, F, T, nullptr, &bank, D, W, K, argmax, overflow_flag, workspace, workspace_bytes, stream);
}

// ET (D, Fp) = E (F, D)^T, complex128, bins F .. Fp - 1 zero: the transposed table a bank's refinement reads.
int gccnmf_steering_transpose(gccnmf_handle* h, const double* E, int F, int D, double* ET, int64_t Fp, void* stream) {
  GCCNMF_LAUNCH(h, transpose_pad_kernel<double2>, dim3((D + 31) / 32, (int)((Fp + 31) / 32)), dim3(32, 8), 0, stream, reinterpret_cast<const double2*>(E), F,
                D, reinterpret_cast<double2*>(ET), Fp);
  return GCCNMF_OK;
}

// ---- dictionary banks (gccnmf_lldict_*)
// Entry e's derived forms from its W (F, K) f32 on the device: the bf16 planes (zero past K), the |W| column sums and the transpose
// (K, Fp) the refinement reads.  abs_colsum_kernel and transpose_pad_kernel are the plain argmax's, so the values are its values.
int gccnmf_lldict_prepare(gccnmf_handle* h, const DictBank& dict, int entry, const float* W, int F, int K, void* stream) {
  const int64_t ld = (int64_t)dict.Qd * dict.Kp, n = (int64_t)F * dict.Kp;
  bf16* planes = reinterpret_cast<bf16*>(const_cast<void*>(dict.planes)) + (int64_t)entry * dict.Kp;
  GCCNMF_LAUNCH(h, split_dict_planes_kernel, (unsigned)((n + 255) / 256), 256, 0, stream, W, F, K, dict.Kp, ld, planes, (int64_t)F * ld);
  GCCNMF_LAUNCH(h, abs_colsum_kernel, (K + 127) / 128, 128, 0, stream, W, F, K, const_cast<float*>(dict.colsum) + (int64_t)entry * dict.Kp);
  GCCNMF_LAUNCH(h, transpose_pad_kernel<float>, dim3((K + 31) / 32, (int)((dict.Fp + 31) / 32)), dim3(32, 8), 0, stream, W, F, K,
                const_cast<float*>(dict.WT) + (int64_t)entry * dict.Kp * dict.Fp, dict.Fp);
  return GCCNMF_OK;
}

// gcc.cu
int gccnmf_tdoa_gccnmf_dict(gccnmf_handle* h, const float* coherence, int F, int T, const SteerBank& bank, const DictBank& dict, int D,
                            int32_t* argmax, const int32_t* gate, int capacity, int32_t* ran, void* stream);

size_t gccnmf_tdoa_argmax_dict_workspace_bytes(int F, int T, int D, int K) { return argmax_workspace_bytes(F, T, D, K); }

// The tensor-core argmax for a dictionary bank: the plane build of the steering bank, ONE grouped GEMM launch over every entry
// (argmax_gemm_dict_kernel), then the candidate refinement over the column's table and dictionary.  The workspace is
// gccnmf_tdoa_argmax's at K = Kmax (its W planes and sums go unused: the bank keeps its own).  Without the tensor path (D < 32,
// F < 32 or the SIMT option) the float64 SIMT form decides every pair.
int gccnmf_tdoa_argmax_dict(gccnmf_handle* h, const float* coherence, int F, int T, const SteerBank& bank, const DictBank& dict, int D,
                            int32_t* argmax, int32_t* overflow_flag, void* workspace, size_t workspace_bytes, void* stream) {
  GCCNMF_ENTER(h);
  GCCNMF_REQUIRE(h, F > 0 && T > 0 && D > 0 && coherence && argmax && bank.Qe >= 1 && dict.Qd >= 1, "tdoa_argmax_dict: bad arguments");
  if (h->force_simt_nmf || D < 32 || D > 128 || F < 32 || (int64_t)T * D >= ((int64_t)1 << 31)) {
    if (overflow_flag) GCCNMF_CHECK_CUDA(h, cudaMemsetAsync(overflow_flag, 0, sizeof(int32_t), (cudaStream_t)stream));
    return gccnmf_tdoa_gccnmf_dict(h, coherence, F, T, bank, dict, D, argmax, nullptr, 0, nullptr, stream);
  }
  const int K = dict.Kmax;
  const size_t need = argmax_workspace_bytes(F, T, D, K);
  ArgmaxWorkspace w = carve_argmax(workspace, workspace_bytes, F, T, D, K);
  if (!w.ok || workspace_bytes < need) return gccnmf_fail(h, GCCNMF_ERR_WORKSPACE, "tdoa_argmax_dict workspace too small: need %zu bytes", need);
  GCCNMF_REQUIRE(h, bank.Fp == w.Fp && dict.Fp == w.Fp, "tdoa_argmax_dict: the banks' transposed tables have %lld bins, the workspace %lld",
                 (long long)bank.Fp, (long long)w.Fp);
  GCCNMF_CHECK_CUDA(h, cudaMemsetAsync(w.count, 0, 16, (cudaStream_t)stream));
  GCCNMF_LAUNCH(h, build_gcc_planes_bank_kernel, dim3((int)((w.Fp + 63) / 64), steer_tiles_max(T, 32, bank.Qe)), 256, 0, stream,
                reinterpret_cast<const float2*>(coherence), F, T, bank, D, w.Gp, w.Fp, w.plane_g);
  const int64_t ld = (int64_t)dict.Qd * dict.Kp;
  const bf16* planes = reinterpret_cast<const bf16*>(dict.planes);
  CUtensorMap map_a, map_b;
  if (int st = tmap_mnmajor(h, planes, (int)ld, F, ld, (int64_t)F * ld, &map_a)) return st;
  if (int st = tmap_kmajor(h, w.Gp, T * D, F, w.Fp, w.plane_g, D, &map_b)) return st;
  const int m_tiles = (K + tgemm::kBM - 1) / tgemm::kBM, n_tiles = steer_tiles_max(T * D, kPersBN, dict.Qd) ;
  const EpiArgmaxDict epi{argmax, w.list, w.cand, w.count, w.capacity, T, margin_factor(F)};
  const int st = D == 32 ? launch_argmax_dict<32>(h, map_a, map_b, F, m_tiles, n_tiles, dict, epi, stream)
               : D == 64 ? launch_argmax_dict<64>(h, map_a, map_b, F, m_tiles, n_tiles, dict, epi, stream)
                         : launch_argmax_dict<128>(h, map_a, map_b, F, m_tiles, n_tiles, dict, epi, stream);
  if (st) return st;
  GCCNMF_LAUNCH(h, transpose_pad_kernel<float2>, dim3((T + 31) / 32, (int)((w.Fp + 31) / 32)), dim3(32, 8), 0, stream,
                reinterpret_cast<const float2*>(coherence), F, T, w.cohT, w.Fp);
  GCCNMF_LAUNCH(h, refine_candidates_dict_kernel, h->sm_count * 8, 256, 0, stream, w.list, w.cand, w.count, w.capacity, w.cohT, dict, bank, F, w.Fp,
                D, T, argmax);
  if (overflow_flag) GCCNMF_CHECK_CUDA(h, cudaMemcpyAsync(overflow_flag, w.count, sizeof(int), cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return GCCNMF_OK;
}
