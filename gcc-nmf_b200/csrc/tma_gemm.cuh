// TMA-fed 3xBF16 GEMM over pre-split operand planes on the Hopper warpgroup tensor cores (wgmma, sm_90a).
//
//   D[m, n] = sum_k A(m, k) * B(n, k)        A = A_hi + A_lo, B = B_hi + B_lo   (bf16 planes, hi = bf16(x), lo = bf16(x - hi))
//
// Each operand lives in global memory as TWO bf16 planes [2][rows][pitch] written by the kernel that produced it
// (the KL-NMF epilogues / the W update), in ONE orientation; the contraction picks the matching shared-memory layout:
//   K-major  : element (r, k) at rows r, k contiguous        TMA boxes {KB, rows / cluster extent, 1 plane}, SWIZZLE_64B rows
//   MN-major : element (r, k) at rows k, r contiguous        TMA boxes {64, KB, 2 planes} = 64-wide atoms, SWIZZLE_128B
// so no matrix is ever transposed or re-split inside the loop.
// Per 16-deep k-step the products lo.hi + hi.lo + hi.hi accumulate in float32 registers: three wgmma of width BN, or -- dual-N
// loop, K-major B with 2 BN <= 256 -- A_lo . B_hi of width BN and A_hi . [B_hi; B_lo] of width 2 BN over the adjacent hi and lo
// planes of the stage; the epilogue adds the two accumulator halves.
//
// CTA = one 128 x BN accumulator tile, three warpgroups (12 warps):
//   warpgroup 0  warp 0 lane 0 is the TMA producer: waits empty[s], arms full[s] with the stage's byte count, issues the boxes;
//                warps 1-3 fetch the epilogue's per-row values, prefetch / preload its operands and compute the SIMT tail rows
//   warpgroups 1, 2  the MMA: each issues the wgmma of 64 accumulator rows (m0 + 64 (g - 1) ..) and releases the stages it read
// then the accumulators go to a shared tile[n][m] and all 12 warps run the functor by columns.
// Rows past the last full 128-row tile (F = 513 = 4 x 128 + 1) are computed in float32 SIMT by warps 1-3 while the main loop
// runs.  A cluster of CN x CM CTAs (n tiles x m tiles) shares operand tiles: each CTA loads 1 / CN of its A tile and 1 / CM of
// its B tile and TMA-multicasts the slice to the CTAs of its cluster row / column.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include <cstdint>
#include <type_traits>

#include "gmma_ptx.cuh"

namespace tgemm {

using gmma::mbar_init;
using gmma::mbar_wait;
using gmma::smem_u32;

constexpr int kBM = 128;
constexpr int kMmaWarpgroups = 2;          // 64 accumulator rows each
constexpr int kAuxWarps = 3;               // warps 1-3 (warp 0 is the producer)
constexpr int kThreads = (1 + kMmaWarpgroups) * 128;
constexpr int kColumnsInFlight = 8;        // epilogue: independent column loads per thread before the first dependent store
constexpr int kMaxRowValues = 4;           // per-row values an epilogue functor may stage in shared memory
constexpr int kSmemBudget = 216 * 1024;    // stages; + barriers + epilogue scratch + alignment slack stays under the 227 KB per-CTA limit
// Leading dimension (floats) of the staged accumulator tile [BN][kTileLd]: the four lanes of a wgmma fragment quad hold one row at
// columns c, c + 2, c + 4, c + 6, and the 4-word pad puts those columns 8 banks apart, so a warp's 32 staging stores hit 32 distinct
// banks (with 128 they all land on the bank of their row: 4-way conflicts); a column stays 16-byte aligned for the float4 reads.
constexpr int kTileLd = kBM + 4;

__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// One 3-D box (inner, rows, planes) -> shared memory; completion is signalled on `bar` as transaction bytes.
// Coordinates outside the tensor are zero-filled (and still counted in the transaction bytes).
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
// One 2-D box (inner, rows) -> shared memory of this CTA, completion signalled on `bar`; out-of-range elements are zero-filled.
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
// One 4-D box (inner, rows, planes, clip) -> shared memory of this CTA: the operand maps of a batched launch (Clips).
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
// Same, delivered to the same shared-memory offset (and signalled on the same barrier offset) of every CTA of the cluster in `mask`.
template <bool MULTICAST>
__device__ __forceinline__ void tma_load_3d_mc(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2, uint16_t mask) {
  if (MULTICAST) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4, %5}], [%2], %6;"
        ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "h"(mask)
        : "memory");
  } else {
    tma_load_3d(dst, map, bar, c0, c1, c2);
  }
}
__device__ __forceinline__ void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// 16 bytes from the shared memory of CTA `rank` of my cluster, at the offset of my own `local` pointer
__device__ __forceinline__ float4 ld_cluster_f32x4(const float* local, uint32_t rank) {
  uint32_t remote;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(gmma::smem_u32(local)), "r"(rank));
  float4 v;
  asm volatile("ld.shared::cluster.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(remote) : "memory");
  return v;
}
__device__ __forceinline__ void tma_prefetch_descriptor(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t) :: "memory");
  return t;
}
// Programmatic dependent launch: both are no-ops for a kernel launched without the attribute.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait_prior_grids() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// hi = bf16(x) (round to nearest even), lo = bf16(x - hi): x = hi + lo up to 2^-17 |x|.
__device__ __forceinline__ void split_bf16(float x, __nv_bfloat16& hi, __nv_bfloat16& lo) {
  hi = __float2bfloat16_rn(x);
  lo = __float2bfloat16_rn(x - __bfloat162float(hi));
}

// 8 consecutive elements of a plane pair (one 16-byte load per plane) as floats hi + lo.
__device__ __forceinline__ void load_planes8(const __nv_bfloat16* hi, const __nv_bfloat16* lo, float (&out)[8]) {
  const uint4 h = __ldg(reinterpret_cast<const uint4*>(hi)), l = __ldg(reinterpret_cast<const uint4*>(lo));
  const uint32_t hw[4] = {h.x, h.y, h.z, h.w}, lw[4] = {l.x, l.y, l.z, l.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    out[2 * i] = __uint_as_float(hw[i] << 16) + __uint_as_float(lw[i] << 16);
    out[2 * i + 1] = __uint_as_float(hw[i] & 0xFFFF0000u) + __uint_as_float(lw[i] & 0xFFFF0000u);
  }
}

// Completion signal of a whole launch to the ranks of a sharded run: the last CTA to finish adds 1 to the arrival counter of every
// rank (peer-mapped addresses).  The data the signal publishes lies in THIS GPU's memory -- peers fetch it over NVLink through this
// GPU's L2 -- so a device-scope fence per CTA is enough and the adds are relaxed (no MEMBAR.SYS: that costs ~5 us).
struct PeerSignal {
  unsigned* counters[8];
  int world;              // 0: no signal
};
__device__ __forceinline__ void signal_peers(const PeerSignal& sig) {
  for (int r = 0; r < sig.world; ++r) asm volatile("red.relaxed.sys.global.add.u32 [%0], %1;" ::"l"(sig.counters[r]), "r"(1u) : "memory");
}

struct PlaneGemmArgs {
  int M, N, Kc;
  int m_tiles;             // 128-row tiles on the tensor cores (= gridDim.y)
  int tail_rows;           // rows [128 m_tiles, M) computed in float32 SIMT by the epilogue warps while the main loop runs (K-major operands)
  int tail_cols;           // columns of the n tile each m tile's CTA takes for those rows (multiple of 2)
  int kblocks_per_split;   // k-blocks of KB handled by one blockIdx.z
  int preload;             // 1: the by-column epilogue's global operands are fetched into registers while the main loop runs
  int m_fastest;           // 0: grid (n tiles, m tiles, splits); 1: grid (m tiles, n tiles, splits) -- the CTAs that share a B tile are
                           // launched together, so a large B operand is read from HBM once (cluster shapes with CN == 1 only)
  int z_cluster;           // S > 1: the S k-splits of a tile form a (1, 1, S) cluster and are summed through distributed shared memory
                           // (CTA z finishes the z-th slice of the tile's columns, rank order 0 .. S - 1); the functor sees z = 0
  // SIMT tail rows (both operands K-major only): element (r, k) of plane p at ptr[p * plane + r * ld + k]
  const __nv_bfloat16* A; int64_t a_plane, lda;
  const __nv_bfloat16* B; int64_t b_plane, ldb;
  unsigned* done_counter;       // with `signal`: CTA completion count of this launch (zero before and after)
  PeerSignal signal;
  unsigned long long* timing;   // optional diagnostics, 8 slots per CTA: [0] / [7] globaltimer (ns) at CTA start / end (tail CTAs too),
                                // [1..6] clock64: start, first stage full, last MMA issued, producer done, accumulators retired, epilogue end
};


// WANT_OPERAND: the epilogue takes its float32 operand tile [BN][128] in shared memory (see wants_smem_operand); it gets it when
// at least kMinStagesWithOperand pipeline stages remain beside it, else the operand is read from global memory as before.
constexpr int kMinStagesWithOperand = 4;
template <int BN, int KB, bool A_MN, bool B_MN, int NACC = 1, bool WANT_OPERAND = false>   // NACC = 2: dual-N mode, two BN-column accumulator halves
struct Config {
  static_assert(KB == 32 || KB == 64, "k-block of 32 (SWIZZLE_64B K-major rows) or 64 (SWIZZLE_128B)");
  static_assert(BN % 8 == 0 && BN >= 16 && BN * NACC <= 256, "wgmma N (= BN, or 2 BN in the dual-N loop)");
  static constexpr int kAAtoms = kBM / 64;
  static constexpr int kBAtoms = (BN + 63) / 64;
  static constexpr int kAtomBytes = 2 * KB * 128;                 // one MN-major atom: 64 elements x KB k-rows x 2 planes
  static constexpr int kABytes = 2 * kBM * KB * 2;
  static constexpr int kBBytes = B_MN ? kBAtoms * kAtomBytes : 2 * BN * KB * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static_assert(kABytes % 1024 == 0 && kBBytes % 1024 == 0, "operand blocks must keep 1024-byte alignment");
  static constexpr int kOperandWant = BN * kBM * 4;
  static constexpr bool kOperandFits = (kSmemBudget - kOperandWant) / kStageBytes >= kMinStagesWithOperand &&
                                       ((kSmemBudget - kOperandWant) / kStageBytes) * kStageBytes >= BN * kTileLd * 4;
  static constexpr int kOperandBytes = (WANT_OPERAND && kOperandFits) ? kOperandWant : 0;   // behind the stages, never aliased
  static constexpr int kStagesRaw = (kSmemBudget - kOperandBytes) / kStageBytes;
  static constexpr int kStages = kStagesRaw > 8 ? 8 : kStagesRaw;
  static_assert(kStages >= 2, "tile too large for a 2-stage pipeline");
  static constexpr int kAccCols = BN * NACC;                      // wgmma N; each thread holds kAccCols / 2 floats
  static constexpr int kBarrierBytes = 256;
  static constexpr int kScratchBytes = kMaxRowValues * kBM * 4 + (kThreads / 32) * 32 * 16;
  static constexpr int kTotal = kStages * kStageBytes + kOperandBytes + kBarrierBytes + kScratchBytes + 1024;   // + alignment slack
  static_assert(kStages * kStageBytes >= BN * kTileLd * 4, "the epilogue stages the accumulator tile in the pipeline buffers");
  static_assert(kTotal <= 227 * 1024, "shared memory per CTA");
};

// One k-block (KB deep) of the 3xBF16 contraction for the 64 accumulator rows of one warpgroup, issued asynchronously.
//   a_base: this warpgroup's rows of the A hi plane in the stage; b_base: the B hi plane; b_lo_off: B lo plane - B hi plane
// Products in the order lo.hi, hi.lo, hi.hi (dual-N: A_lo . B_hi, then A_hi . [B_hi; B_lo]).  The k tail needs no
// special case: TMA zero-fills the k-rows past the end of both operands, so their products add exact zeros (and an issue that
// depends on the data would make ptxas serialise the wgmma).
template <int N, int KB, bool A_MN, bool B_MN, bool DUAL>
__device__ __forceinline__ void mma_kblock(float (&acc)[N / 2], uint32_t a_base, uint32_t b_base, uint32_t b_lo_off) {
  constexpr uint32_t kAtom = 2 * KB * 128;
  constexpr uint32_t a_lo_off = A_MN ? KB * 128 : kBM * KB * 2;
  constexpr uint32_t a_step = A_MN ? 2048u : 32u, b_step = B_MN ? 2048u : 32u;
  constexpr uint32_t kKSbo = 8 * KB * 2;
  constexpr uint32_t kKSwizzle = (KB == 32) ? gmma::kSwizzle64B : gmma::kSwizzle128B;
  auto desc = [&](uint32_t addr, bool mn) {
    return mn ? gmma::make_desc(addr, kAtom, 1024, gmma::kSwizzle128B) : gmma::make_desc(addr, 16, kKSbo, kKSwizzle);
  };
#pragma unroll
  for (int kk = 0; kk < KB / 16; ++kk) {
    const uint32_t a_addr = a_base + kk * a_step, b_addr = b_base + kk * b_step;
    const uint64_t a_hi = desc(a_addr, A_MN), a_lo = desc(a_addr + a_lo_off, A_MN);
    const uint64_t b_hi = desc(b_addr, B_MN), b_lo = desc(b_addr + b_lo_off, B_MN);
    if constexpr (DUAL) {
      // N = BN into the first half of the accumulator: the column of a fragment element depends on its register index and the
      // lane only, so acc[0 .. N / 4) of the N = 2 BN fragment are exactly the N = BN fragment.  lo.lo is not computed: it is
      // below 2^-18 |a| |b|, under the 2^-17 to which each plane pair represents its value.
      // Ordering: the PTX ISA orders accumulator accesses of successive wgmma.mma_async by default only when they have the same
      // shape.  These two MMAs differ in N and share registers, so each is preceded by wgmma.fence (for kk = 0 the caller's
      // fence before the k-block is the first one).
      if (kk > 0) gmma::wgmma_fence();
      gmma::Wgmma<N / 2>::template mma<A_MN, B_MN>(reinterpret_cast<float(&)[N / 4]>(acc), a_lo, b_hi);
      gmma::wgmma_fence();
      // N = 2 BN: the descriptor at b_hi walks the BN rows of the hi plane and on into the lo plane behind it
      gmma::Wgmma<N>::template mma<A_MN, B_MN>(acc, a_hi, b_hi);
      (void)b_lo;
    } else {
      gmma::Wgmma<N>::template mma<A_MN, B_MN>(acc, a_lo, b_hi);
      gmma::Wgmma<N>::template mma<A_MN, B_MN>(acc, a_hi, b_lo);
      gmma::Wgmma<N>::template mma<A_MN, B_MN>(acc, a_hi, b_hi);
    }
  }
}

// Epilogues with `static constexpr bool kTileEpilogue = true` take the whole staged tile:
//   __device__ void tile_epilogue(const float* tile /* [n][kTileLd] */, int m0, int n0, int n_valid, int z) const;   (all threads)
template <class E, class = void>
struct has_tile_epilogue { static constexpr bool value = false; };
template <class E>
struct has_tile_epilogue<E, decltype((void)E::kTileEpilogue)> { static constexpr bool value = E::kTileEpilogue; };

// Epilogues with `static constexpr bool kDualN = true` ask for the dual-N main loop where the shape allows it (K-major B, 2 BN <= 256).
// The hi and lo planes of a K-major B tile are adjacent in the stage, so ONE MMA with N = 2 BN multiplies A_hi with [B_hi ; B_lo]
// into two accumulator halves, and one of N = BN adds A_lo . B_hi to the first half: 2 MMAs per k-step compute the three products
// lo.hi + hi.hi | hi.lo over 3 BN columns, as the plain loop does in three MMAs of BN, and the epilogue adds the two halves.
// Epilogues with `static constexpr bool kPreloadOperands = true` have their by-column global operands fetched into registers while
// the main loop runs (opt-in: measured to pay for the ratio epilogue of the W.H contractions, to cost for the H update; not used
// where the operand comes into shared memory instead, see wants_smem_operand).
template <class E, class = void>
struct wants_preload { static constexpr bool value = false; };
template <class E>
struct wants_preload<E, decltype((void)E::kPreloadOperands)> { static constexpr bool value = E::kPreloadOperands; };

// Epilogues with `static constexpr bool kSmemOperand = true` have a by-column operand that is one float32 element per output
// element, in the output's layout (`Loaded` is that float4):  CUtensorMap operand_map;  const float* operand() const;
// int64_t operand_ld() const;  int operand_cols() const  (element (m, n) at operand()[n * operand_ld() + m], n < operand_cols()).
// The launcher encodes operand_map with a box of 128 m x BN n; the producer thread loads the CTA's box with one TMA copy when it
// has issued its last stage, into shared memory beside the stages, and the epilogue reads its columns from there.
template <class E, class = void>
struct wants_smem_operand { static constexpr bool value = false; };
template <class E>
struct wants_smem_operand<E, decltype((void)E::kSmemOperand)> { static constexpr bool value = E::kSmemOperand; };

template <class E, class = void>
struct wants_dual_n { static constexpr bool value = false; };
template <class E>
struct wants_dual_n<E, decltype((void)E::kDualN)> { static constexpr bool value = E::kDualN; };

// Batched launch of a by-column epilogue E over C clips of one shape: blockIdx.z = clip * splits + split, so the (1, 1, splits)
// extent of a clip's k-splits never mixes clips, and clip c's operand planes, epilogue buffers and SIMT-tail operands all lie
// c * clip_bytes past clip 0's (one per-clip workspace carve repeated C times).  The operand maps carry a fourth, clip dimension
// with that stride, so TMA zero-fills each clip's ragged edges exactly as in a launch on that clip alone, and the functor a CTA
// runs is E::at_offset(c * clip_bytes): E with every pointer moved to clip c.  Every tile therefore computes what the same tile of
// a solo launch computes.  A batched launch runs 1 x 1 clusters and takes the epilogue operand from global memory (no operand
// map), neither of which changes a result.  The trait makes it a separate instantiation of plane_gemm_kernel.
template <class E>
struct Clips {
  static constexpr bool kBatched = true;
  static constexpr bool kRowReduce = E::kRowReduce;
  static constexpr int kRowValues = E::kRowValues;
  static constexpr bool kPrefetch = E::kPrefetch;
  static constexpr bool kDualN = wants_dual_n<E>::value;
  static constexpr bool kPreloadOperands = wants_preload<E>::value;
  using State = typename E::State;
  using Loaded = typename E::Loaded;
  E e;                 // clip 0
  int64_t clip_bytes;
  int splits;
};
template <class E>
struct is_batched { static constexpr bool value = false; };
template <class E>
struct is_batched<Clips<E>> { static constexpr bool value = true; };

// The functor of this CTA's clip (the launch's own functor when not batched), its clip and its k-split.
template <class E> __device__ __forceinline__ const E& clip_epilogue(const E& e, int) { return e; }
template <class E> __device__ __forceinline__ E clip_epilogue(const Clips<E>& c, int clip) { return c.e.at_offset(c.clip_bytes * clip); }
template <class E> __device__ __forceinline__ int clip_of(const E&) { return 0; }
template <class E> __device__ __forceinline__ int clip_of(const Clips<E>& c) { return (int)blockIdx.z / c.splits; }
template <class E> __device__ __forceinline__ int split_of(const E&) { return blockIdx.z; }
template <class E> __device__ __forceinline__ int split_of(const Clips<E>& c) { return (int)blockIdx.z % c.splits; }
template <class E> __device__ __forceinline__ int64_t clip_offset(const E&, int) { return 0; }
template <class E> __device__ __forceinline__ int64_t clip_offset(const Clips<E>& c, int clip) { return c.clip_bytes * clip; }
// Ragged launch of a by-column epilogue E over clips of different lengths that share one tile width: the grid is flat, the
// concatenation of each clip's own (n tiles x m tiles x splits) CTAs, so a short clip launches only its own tiles.  A CTA finds its
// clip in `tiles` (sorted by cta_begin) and takes from it everything that differs between clips: the extents N and Kc, the k-split
// ranges, the clip's own operand tensor maps (encoded on the host with the clip's exact extents, so TMA zero-fills its edges exactly as
// in a solo launch, and read through their global address) and the SIMT-tail operands.  The functor it runs is
// E::at_clip(clips, clip): E with the clip's buffers and lengths from the functor's per-clip table.  1 x 1 clusters, k-splits as
// slabs, epilogue operands from global memory, as in Clips.  A separate instantiation of plane_gemm_kernel.
struct RaggedTile {
  int cta_begin;                 // first CTA of the clip in the flat grid
  int clip;                      // index into the functor's per-clip table
  int N, Kc, n_tiles, kblocks_per_split;
  const CUtensorMap* map_a;      // in global memory
  const CUtensorMap* map_b;
  const __nv_bfloat16* tail_a;   // SIMT tail rows: the clip's A and B planes and plane strides (lda, ldb are the launch's)
  const __nv_bfloat16* tail_b;
  int64_t a_plane, b_plane;
};
template <class E>
struct Ragged {
  static constexpr bool kRowReduce = E::kRowReduce;
  static constexpr int kRowValues = E::kRowValues;
  static constexpr bool kPrefetch = E::kPrefetch;
  static constexpr bool kDualN = wants_dual_n<E>::value;
  static constexpr bool kPreloadOperands = wants_preload<E>::value;
  using State = typename E::State;
  using Loaded = typename E::Loaded;
  E e;                           // the fields every clip shares
  const RaggedTile* tiles;
  int count;
  const void* clips;             // the functor's per-clip table
};
template <class E>
struct is_ragged { static constexpr bool value = false; };
template <class E>
struct is_ragged<Ragged<E>> { static constexpr bool value = true; };

// Index of the entry of `tiles` that holds this CTA: a 32-way search by warp 0 (three rounds of loads for 8191 clips), published
// to the CTA through shared memory.  Called by every thread.
__device__ __forceinline__ int ragged_find(const RaggedTile* tiles, int count) {
  __shared__ int found;
  if (threadIdx.x < 32) {
    const int me = (int)blockIdx.x;
    int lo = 0, hi = count;                   // tiles[lo].cta_begin <= me < tiles[hi].cta_begin
    while (hi - lo > 1) {
      const int step = (hi - lo + 31) / 32;
      const int i = lo + (int)threadIdx.x * step;
      const unsigned le = __ballot_sync(0xffffffffu, i < hi && tiles[i].cta_begin <= me);
      lo += (31 - __clz(le)) * step;          // (lane 0 always qualifies)
      hi = min(hi, lo + step);
    }
    if (threadIdx.x == 0) found = lo;
  }
  __syncthreads();
  return found;
}
// A tensor map written to global memory by a copy before the launch is read by the tensormap proxy: acquire it first.
__device__ __forceinline__ void tensormap_acquire(const CUtensorMap* map) {
  asm volatile("fence.proxy.tensormap::generic.acquire.sys [%0], 128;" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
template <class E> __device__ __forceinline__ E clip_epilogue(const Ragged<E>& r, int clip) { return r.e.at_clip(r.clips, clip); }

template <bool BATCHED, bool MULTICAST>
__device__ __forceinline__ void tma_load_operand(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2, int clip, uint16_t mask) {
  if constexpr (BATCHED) tma_load_4d(dst, map, bar, c0, c1, c2, clip);
  else tma_load_3d_mc<MULTICAST>(dst, map, bar, c0, c1, c2, mask);
}

// Epilogue concept (functors in klnmf_tma.cu).  The kernel stages the accumulator tile in shared memory and hands it out by
// columns: a warp owns column n, lane l rows m .. m + 3 with m = m0 + 4 l (contiguous in every output of the KL-NMF loop).
//   static constexpr int kRowValues (<= kMaxRowValues);  __device__ void row_values(int m, float* v) const;
//       per-row constants, fetched by one thread per row while the main loop runs and staged in shared memory
//   struct State;   __device__ void init(State&, int m, const float* rowvals) const;    rowvals[i * 128 + 0..3] = value i of rows m .. m + 3
//   struct Loaded;  __device__ Loaded load(int m, int n) const;          the column's global operands (issued kColumnsInFlight deep)
//   static constexpr bool kPrefetch;  __device__ void prefetch(int m, int n) const;     L2 prefetch of the line load(m, n) will read
//   __device__ void store(int m, int n, float4 acc, const Loaded&, int z, State&) const;
//   static constexpr bool kRowReduce;  __device__ float4 row_partial(const State&) const;  __device__ void row_total(int m, int tile_n, float) const;
//   __device__ void elem(int m, int n, float acc, int z) const;          SIMT tail rows (one column per lane)
template <int BN, int KB, bool A_MN, bool B_MN, int CN, int CM, class Epilogue>
__global__ void __launch_bounds__(kThreads, 1)
plane_gemm_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, PlaneGemmArgs args,
                  const __grid_constant__ Epilogue epi) {
  constexpr bool DUAL = wants_dual_n<Epilogue>::value && !B_MN && 2 * BN <= 256;
  using C = Config<BN, KB, A_MN, B_MN, DUAL ? 2 : 1, wants_smem_operand<Epilogue>::value && !has_tile_epilogue<Epilogue>::value>;
  constexpr bool OPERAND = C::kOperandBytes > 0;     // the epilogue's operand tile comes into shared memory by TMA
  constexpr int kCluster = CN * CM;
  constexpr bool BATCHED = is_batched<Epilogue>::value;
  constexpr bool RAGGED = is_ragged<Epilogue>::value;
  static_assert((!BATCHED && !RAGGED) || kCluster == 1, "a batched or ragged launch runs 1 x 1 clusters");
  static_assert((CN == 1 || CN == 2) && (CM == 1 || CM == 2), "cluster of CN n-tiles x CM m-tiles");
  static_assert(A_MN || (kBM / CN) % 8 == 0, "A row slices keep the swizzle atoms whole");
  static_assert(B_MN || (BN / CM) % 8 == 0, "B row slices keep the swizzle atoms whole");
  extern __shared__ unsigned char smem_dyn[];
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~uintptr_t(1023));

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const bool mf = args.m_fastest != 0;
  // my tile, k-split and clip, and the extents, k-split length and operand maps of my clip
  int tile_n, tile_m, z, clip, N = args.N, Kc = args.Kc, kblocks_per_split = args.kblocks_per_split;
  const CUtensorMap* tmap_a = &map_a;
  const CUtensorMap* tmap_b = &map_b;
  const RaggedTile* rt = nullptr;
  if constexpr (RAGGED) {
    rt = epi.tiles + ragged_find(epi.tiles, epi.count);
    const int local = (int)blockIdx.x - rt->cta_begin, per_split = rt->n_tiles * args.m_tiles;
    tile_n = local % rt->n_tiles;
    tile_m = (local % per_split) / rt->n_tiles;
    z = local / per_split;
    clip = rt->clip;
    N = rt->N; Kc = rt->Kc; kblocks_per_split = rt->kblocks_per_split;
    tmap_a = rt->map_a; tmap_b = rt->map_b;
  } else {
    tile_n = mf ? (int)blockIdx.y : (int)blockIdx.x;
    tile_m = mf ? (int)blockIdx.x : (int)blockIdx.y;
    z = split_of(epi);
    clip = clip_of(epi);
  }
  auto&& ep = clip_epilogue(epi, clip);     // the functor of my clip
  const int n0 = tile_n * BN;
  const int total_kblocks = (Kc + KB - 1) / KB;
  const int kb_begin = z * kblocks_per_split;
  const int kb_end = min(total_kblocks, kb_begin + kblocks_per_split);
  const int num_kb = max(0, kb_end - kb_begin);
  // position inside the cluster (x = n tile, y = m tile); rank = x + CN y (%cluster_ctarank)
  const int cx = (!mf && CN > 1) ? (int)(blockIdx.x % CN) : 0;     // (the m-fastest grid is used with CN == 1 only)
  const int cy = (CM > 1) ? tile_m % CM : 0;
  // CTAs that receive my slice of A (same m tile: my cluster row) / of B (same n tile: my cluster column)
  const uint16_t mask_row = (uint16_t)(((1u << CN) - 1u) << (CN * cy));
  const uint16_t mask_col = (uint16_t)((CM > 1 ? ((1u << cx) | (1u << (cx + CN))) : (1u << cx)));

  const float* operand = reinterpret_cast<const float*>(smem + C::kStages * C::kStageBytes);   // [BN][128] when OPERAND
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + C::kStages * C::kStageBytes + C::kOperandBytes);
  uint64_t* full = bars;                    // [kStages]  TMA -> MMA
  uint64_t* empty = bars + C::kStages;      // [kStages]  MMA warpgroups (of every CTA that shares a slice with me) -> TMA
  uint64_t* operand_full = bars + 2 * C::kStages;   // TMA -> epilogue (OPERAND)
  // epilogue scratch behind the barriers (never touched by TMA): per-row functor values, row-sum partials of the 12 warps
  float* rowvals = reinterpret_cast<float*>(reinterpret_cast<unsigned char*>(bars) + C::kBarrierBytes);   // [kMaxRowValues][128]
  float4* red = reinterpret_cast<float4*>(rowvals + kMaxRowValues * kBM);                             // [12 warps][32 lanes]
  float* tile = reinterpret_cast<float*>(smem);        // epilogue: [BN][kTileLd] float32, aliases the pipeline stages
  const int m0 = tile_m * kBM;

  const int cta_linear = blockIdx.x + gridDim.x * (blockIdx.y + gridDim.y * blockIdx.z);
  if (args.timing && tid == 0) {
    args.timing[cta_linear * 8 + 0] = globaltimer_ns();
    args.timing[cta_linear * 8 + 1] = clock64();
  }
  if (tid == 0) {
    for (int s = 0; s < C::kStages; ++s) {
      mbar_init(smem_u32(&full[s]), 1);
      // one release per MMA warpgroup of every CTA whose multicast lands in this stage (incl. myself)
      mbar_init(smem_u32(&empty[s]), kMmaWarpgroups * (CN + CM - 1));
    }
    if constexpr (OPERAND) mbar_init(smem_u32(operand_full), 1);
    gmma::fence_barrier_init();
    if constexpr (RAGGED) {
      tensormap_acquire(tmap_a);
      tensormap_acquire(tmap_b);
    }
    tma_prefetch_descriptor(tmap_a);
    tma_prefetch_descriptor(tmap_b);
    if constexpr (OPERAND) tma_prefetch_descriptor(&epi.operand_map);
  }
  if (kCluster > 1) cluster_sync();     // no peer may signal my barriers or write my stages before they are initialised
  else __syncthreads();
  // Everything above overlaps the previous kernel's tail under programmatic dependent launch; nothing below may
  // touch global memory before the prior grids have completed.
  pdl_launch_dependents();
  pdl_wait_prior_grids();

  // Early loads of the epilogue's global operands (V^T for the ratio, the old H^T for the H update): the warps of warpgroup 0
  // fetch the values of their first kPre columns into registers while the tensor cores are still busy, so the by-column pass
  // after the main loop starts with its operands already there; the MMA warpgroups issue theirs as soon as the tile is staged.
  constexpr int kWarpsAll = kThreads / 32;
  constexpr int kLoadedWords = (int)((sizeof(typename Epilogue::Loaded) + 3) / 4);
  constexpr bool kPreloads = !OPERAND && wants_preload<Epilogue>::value && !has_tile_epilogue<Epilogue>::value && !std::is_empty<typename Epilogue::Loaded>::value;
  constexpr int kPreCap = 64 / (kLoadedWords > 0 ? kLoadedWords : 1);                      // register budget: 64 words per thread
  constexpr int kPre = kPreloads ? ((BN + kWarpsAll - 1) / kWarpsAll < kPreCap ? (BN + kWarpsAll - 1) / kWarpsAll : kPreCap) : 0;
  typename Epilogue::Loaded pre[kPre > 0 ? kPre : 1];
  auto preload = [&]() {
    if constexpr (kPre > 0) {
      if (!args.preload) return;
      const int n_valid = min(BN, N - n0);
#pragma unroll
      for (int u = 0; u < kPre; ++u) {
        const int cc = warp + kWarpsAll * u;
        if (cc < n_valid) pre[u] = ep.load(m0 + 4 * lane, n0 + cc);
      }
    }
  };

  if (warp == 0) {
    // ------------------------------------------------------------------ TMA producer (one thread)
    if (lane == 0) {
      for (int i = 0; i < num_kb; ++i) {
        const int s = i % C::kStages;
        const uint32_t use = i / C::kStages;
        if (use > 0) mbar_wait(smem_u32(&empty[s]), (use - 1) & 1);   // the MMAs (mine and my peers') that read this stage have retired
        const uint32_t bar = smem_u32(&full[s]);
        const uint32_t a_dst = smem_u32(smem + (size_t)s * C::kStageBytes), b_dst = a_dst + C::kABytes;
        const int k0 = (kb_begin + i) * KB;
        mbar_arrive_expect_tx(bar, C::kStageBytes);                    // my slices + the ones my peers multicast to me
        if (A_MN) {
#pragma unroll
          for (int a = 0; a < C::kAAtoms; ++a)
            if (a % CN == cx) tma_load_operand<BATCHED, (CN > 1)>(a_dst + a * C::kAtomBytes, tmap_a, bar, m0 + 64 * a, k0, 0, clip, mask_row);
        } else {
          constexpr int kRows = kBM / CN;      // my row slice of the A tile, one box per plane
#pragma unroll
          for (int p = 0; p < 2; ++p)
            tma_load_operand<BATCHED, (CN > 1)>(a_dst + p * (kBM * KB * 2) + cx * (kRows * KB * 2), tmap_a, bar, k0, m0 + cx * kRows, p, clip, mask_row);
        }
        if (B_MN) {
#pragma unroll
          for (int a = 0; a < C::kBAtoms; ++a)
            if (a % CM == cy) tma_load_operand<BATCHED, (CM > 1)>(b_dst + a * C::kAtomBytes, tmap_b, bar, n0 + 64 * a, k0, 0, clip, mask_col);
        } else {
          constexpr int kRows = BN / CM;
#pragma unroll
          for (int p = 0; p < 2; ++p)
            tma_load_operand<BATCHED, (CM > 1)>(b_dst + p * (BN * KB * 2) + cy * (kRows * KB * 2), tmap_b, bar, k0, n0 + cy * kRows, p, clip, mask_col);
        }
      }
      if constexpr (OPERAND) {
        // the epilogue operand tile, issued behind the last stage so that it does not delay the main loop's operands; it arrives
        // while the MMAs of the last stages run
        mbar_arrive_expect_tx(smem_u32(operand_full), C::kOperandBytes);
        tma_load_2d(smem_u32(operand), &epi.operand_map, smem_u32(operand_full), m0, n0);
      }
      if (args.timing) args.timing[cta_linear * 8 + 4] = clock64();   // producer done issuing
    }
    __syncwarp();
    preload();
  } else if (warp < 4) {
    // ------------------------------------------------------------------ warps 1-3, while the main loop runs
    const int e = warp - 1;
    if (Epilogue::kRowValues > 0) {                      // the functor's per-row values, one row per thread
      for (int r = e * 32 + lane; r < kBM; r += kAuxWarps * 32) {
        float rv[Epilogue::kRowValues > 0 ? Epilogue::kRowValues : 1];
        ep.row_values(m0 + r, rv);
#pragma unroll
        for (int i = 0; i < Epilogue::kRowValues; ++i) rowvals[i * kBM + r] = rv[i];
      }
    }
    if (Epilogue::kPrefetch) {
      // pull the epilogue's global operands of this tile towards L2 while the main loop runs (they were last touched an
      // iteration ago and have partly been evicted to HBM since): one prefetch per 128-byte line, 4 lines per column
      const int n_valid = min(BN, N - n0);
      if ((lane & 7) == 0)
        for (int c = e; c < n_valid; c += kAuxWarps) ep.prefetch(m0 + 4 * lane, n0 + c);
    }
    if (!A_MN && !B_MN && args.tail_rows > 0) {
      // Rows past the last full 128-row tile (F = 513 = 4 x 128 + 1), float32 SIMT from the K-major planes: the m tiles of
      // this n tile share its columns (tail_cols <= 256 each), each warp takes two columns per step, each lane 8 consecutive k per
      // 16-byte load (hi and lo plane), four k-chunks in flight.  The result of step i of a round stays in lanes 2i / 2i + 1 and
      // the functor runs with one column per lane, so its global loads overlap.
      // (k-splits summed inside a cluster, z_cluster > 1: the functor is not linear in the accumulator, so the tail rows are computed
      // over the WHOLE contraction, each split taking its share of the tile's tail columns)
      const bool z_red = kCluster == 1 && args.z_cluster > 1;
      const int k_begin = z_red ? 0 : kb_begin * KB, k_end = z_red ? Kc : min(Kc, kb_end * KB);
      const int tcols = z_red ? (((args.tail_cols + args.z_cluster - 1) / args.z_cluster) + 1) & ~1 : args.tail_cols;
      const int c_begin = n0 + (z_red ? tile_m * args.z_cluster + z : tile_m) * tcols;
      const int c_end = min(min(N, n0 + BN), c_begin + tcols);
      constexpr int kRound = 32 * kAuxWarps;             // columns per round: 16 steps of 2 columns per warp
      const __nv_bfloat16* tail_a = reinterpret_cast<const __nv_bfloat16*>(reinterpret_cast<const char*>(args.A) + clip_offset(epi, clip));
      const __nv_bfloat16* tail_b = reinterpret_cast<const __nv_bfloat16*>(reinterpret_cast<const char*>(args.B) + clip_offset(epi, clip));
      int64_t a_plane = args.a_plane, b_plane = args.b_plane;
      if constexpr (RAGGED) {
        tail_a = rt->tail_a; tail_b = rt->tail_b;
        a_plane = rt->a_plane; b_plane = rt->b_plane;
      }
      for (int m = args.m_tiles * kBM; m < args.M; ++m) {
        const __nv_bfloat16* a_hi = tail_a + (int64_t)m * args.lda;
        const __nv_bfloat16* a_lo = a_hi + a_plane;
#pragma unroll 1
        for (int c_round = c_begin; c_round < c_end; c_round += kRound) {
          float keep = 0.f;
#pragma unroll 1
          for (int i = 0; i < 16; ++i) {
            const int n = c_round + 2 * (e + i * kAuxWarps);
            if (n >= c_end) break;
            const bool two = n + 1 < c_end;
            const __nv_bfloat16* b_hi = tail_b + (int64_t)n * args.ldb;
            const __nv_bfloat16* b_lo = b_hi + b_plane;
            const int64_t next = two ? args.ldb : 0;
            float acc0 = 0.f, acc1 = 0.f;
#pragma unroll 4
            for (int k = k_begin + 8 * lane; k < k_end; k += 256) {     // pitches are multiples of 8; pad columns hold zeros
              float a[8], b0[8], b1[8];
              load_planes8(a_hi + k, a_lo + k, a);
              load_planes8(b_hi + k, b_lo + k, b0);
              load_planes8(b_hi + next + k, b_lo + next + k, b1);
#pragma unroll
              for (int j = 0; j < 8; ++j) { acc0 = fmaf(a[j], b0[j], acc0); acc1 = fmaf(a[j], b1[j], acc1); }
            }
            for (int o = 16; o > 0; o >>= 1) { acc0 += __shfl_xor_sync(0xffffffffu, acc0, o); acc1 += __shfl_xor_sync(0xffffffffu, acc1, o); }
            if (lane == 2 * i) keep = acc0;
            if (lane == 2 * i + 1) keep = acc1;
          }
          const int n_mine = c_round + 2 * (e + (lane >> 1) * kAuxWarps) + (lane & 1);
          if (n_mine < c_end) ep.elem(m, n_mine, keep, z_red ? 0 : z);
        }
      }
    }
    preload();
  } else {
    // ------------------------------------------------------------------ MMA warpgroups: 64 rows each, float32 accumulators in registers
    const int g = (warp >> 2) - 1;                       // 0 / 1: rows m0 + 64 g ..
    const int wt = tid & 127;                            // thread of the warpgroup
    float acc[C::kAccCols / 2];
#pragma unroll
    for (int j = 0; j < C::kAccCols / 2; ++j) acc[j] = 0.f;
    const uint32_t a_slab = A_MN ? (uint32_t)(g * C::kAtomBytes) : (uint32_t)(g * 64 * KB * 2);
    constexpr uint32_t b_lo_off = B_MN ? KB * 128 : BN * KB * 2;
    const uint16_t mask_release = mask_row | mask_col;
    auto release = [&](int s) {      // this warpgroup has finished reading stage s: tell every CTA whose multicast lands in it
      if (wt == 0) {
        if (kCluster > 1) {
          for (uint32_t r = 0; r < (uint32_t)kCluster; ++r)
            if (mask_release & (1u << r)) gmma::mbar_arrive_cluster(smem_u32(&empty[s]), r);
        } else {
          gmma::mbar_arrive(smem_u32(&empty[s]));
        }
      }
    };
    for (int i = 0; i < num_kb; ++i) {
      const int s = i % C::kStages;
      mbar_wait(smem_u32(&full[s]), (i / C::kStages) & 1);
      if (args.timing && i == 0 && tid == 128) args.timing[cta_linear * 8 + 2] = clock64();
      const uint32_t a_base = smem_u32(smem + (size_t)s * C::kStageBytes), b_base = a_base + C::kABytes;
      gmma::fence_regs(acc);
      gmma::wgmma_fence();
      mma_kblock<C::kAccCols, KB, A_MN, B_MN, DUAL>(acc, a_base + a_slab, b_base, b_lo_off);
      gmma::wgmma_commit();
      gmma::fence_regs(acc);
      // the previous k-block's MMAs have retired once at most this one is in flight: its stage may be refilled
      gmma::wgmma_wait<1>();
      if (i > 0) release((i - 1) % C::kStages);
    }
    gmma::wgmma_wait<0>();
    gmma::fence_regs(acc);
    if (num_kb > 0) release((num_kb - 1) % C::kStages);
    if (args.timing && tid == 128) args.timing[cta_linear * 8 + 3] = clock64();
    // both warpgroups have finished reading the stages (and every TMA box, mine and the ones my peers multicast to me, was
    // consumed by these MMAs): the accumulators may overwrite them
    asm volatile("bar.sync 1, %0;" ::"n"(kMmaWarpgroups * 128) : "memory");
    if (args.timing && tid == 128) args.timing[cta_linear * 8 + 5] = clock64();
    const int r0 = 64 * g + 16 * (wt >> 5) + ((wt & 31) >> 2);
    const int c0 = 2 * (wt & 3);
#pragma unroll
    for (int j = 0; j < BN / 2; ++j) {
      const int col = 8 * (j >> 2) + c0 + (j & 1), row = r0 + 8 * ((j >> 1) & 1);
      float v = acc[j];
      if constexpr (DUAL) v += acc[j + BN / 2];        // + the A_hi . B_lo half: columns BN .. 2 BN - 1
      tile[(size_t)col * kTileLd + row] = v;
    }
    preload();
  }
  // ------------------------------------------------------------------ epilogue (all 12 warps)
  // Each warp owns whole columns n -- 128 consecutive m are contiguous in every output -- one float4 of m per lane, so each
  // global access of a warp is one 512-byte (float32) or 256-byte (bf16 plane) row segment, with kColumnsInFlight
  // independent loads per thread before the first dependent store.
  __syncthreads();
  const int zc = (kCluster == 1 && !has_tile_epilogue<Epilogue>::value) ? args.z_cluster : 0;
  if (zc > 1) cluster_sync();             // every k-split of this tile has staged its partial accumulator
  if constexpr (has_tile_epilogue<Epilogue>::value) {
    // whole-tile epilogue: the functor reads the staged accumulator tile[n][m] itself (reductions ACROSS columns, e.g. the argmax
    // over the TDOAs of a frame, which the by-column hand-out below cannot express)
    epi.tile_epilogue(tile, m0, n0, min(BN, args.N - n0), z);
    if (args.timing && tid == 64) args.timing[cta_linear * 8 + 6] = clock64();
  } else {
    constexpr int kWarps = kThreads / 32;
    const int m_first = m0 + 4 * lane;
    typename Epilogue::State st;
    ep.init(st, m_first, rowvals + 4 * lane);
    int n_valid = min(BN, N - n0);
    constexpr int U = kColumnsInFlight;
    int c_first = warp;
    if constexpr (OPERAND) mbar_wait(smem_u32(operand_full), 0);
    if (zc > 1) {                          // my slice of the tile's columns
      const int per = (n_valid + zc - 1) / zc;
      c_first = z * per + warp;
      n_valid = min(n_valid, (z + 1) * per);
    }
    if constexpr (kPre > 0) {
      if (args.preload && zc <= 1) {
#pragma unroll
        for (int u = 0; u < kPre; ++u) {
          const int cc = warp + kWarps * u;
          if (cc < n_valid) {
            const float4 acc = *reinterpret_cast<const float4*>(tile + (size_t)cc * kTileLd + 4 * lane);
            ep.store(m_first, n0 + cc, acc, pre[u], z, st);
          }
        }
        c_first = warp + kWarps * kPre;
      }
    }
#pragma unroll 1
    for (int c = c_first; c < n_valid; c += kWarps * U) {
      typename Epilogue::Loaded loaded[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int cc = c + kWarps * u;
        if (cc < n_valid) {
          if constexpr (OPERAND) loaded[u] = typename Epilogue::Loaded{*reinterpret_cast<const float4*>(operand + (size_t)cc * kBM + 4 * lane)};
          else loaded[u] = ep.load(m_first, n0 + cc);
        }
      }
      if (zc > 1) {
        // sum of the k-splits in split order (the order the W update used for the slabs): the distributed-shared-memory loads of ALL
        // U columns of a split are issued before the first add (one at a time they cost a remote-SM round trip per column: the
        // epilogue took 15 k cycles instead of 6 k)
        float4 sum[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int cc = c + kWarps * u;
          const float* src = tile + (size_t)(cc < n_valid ? cc : 0) * kTileLd + 4 * lane;
          sum[u] = z == 0 ? *reinterpret_cast<const float4*>(src) : ld_cluster_f32x4(src, 0);
        }
        for (int r = 1; r < zc; ++r) {
          float4 t[U];
#pragma unroll
          for (int u = 0; u < U; ++u) {
            const int cc = c + kWarps * u;
            const float* src = tile + (size_t)(cc < n_valid ? cc : 0) * kTileLd + 4 * lane;
            t[u] = r == z ? *reinterpret_cast<const float4*>(src) : ld_cluster_f32x4(src, (uint32_t)r);
          }
#pragma unroll
          for (int u = 0; u < U; ++u) { sum[u].x += t[u].x; sum[u].y += t[u].y; sum[u].z += t[u].z; sum[u].w += t[u].w; }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int cc = c + kWarps * u;
          if (cc < n_valid) ep.store(m_first, n0 + cc, sum[u], loaded[u], 0, st);
        }
      } else {
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int cc = c + kWarps * u;
          if (cc < n_valid) {
            const float4 acc = *reinterpret_cast<const float4*>(tile + (size_t)cc * kTileLd + 4 * lane);
            ep.store(m_first, n0 + cc, acc, loaded[u], z, st);
          }
        }
      }
    }
    if constexpr (Epilogue::kRowReduce) {   // per-row sums over the tile's columns: 12 warp partials -> one value per row
      red[warp * 32 + lane] = ep.row_partial(st);
      __syncthreads();
      if (tid < kBM) {
        const float* r = reinterpret_cast<const float*>(red);
        float sum = 0.f;
#pragma unroll
        for (int w = 0; w < kWarps; ++w) sum += r[w * kBM + tid];
        ep.row_total(m0 + tid, tile_n, sum);
      }
    }
    if (args.timing && tid == 64) args.timing[cta_linear * 8 + 6] = clock64();
  }
  // No CTA of a cluster may exit while a peer can still signal its barriers (my last releases have been delivered by now:
  // they precede accum_full, which the epilogue waited for).
  if (kCluster > 1 || zc > 1) cluster_sync();          // (z-cluster: no CTA exits while a peer still reads its tile)
  else __syncthreads();
  if (args.signal.world > 0 && tid == 0) {             // every store of this CTA precedes the barrier above
    __threadfence();
    const unsigned prev = atomicAdd(args.done_counter, 1u);
    if (prev == gridDim.x * gridDim.y * gridDim.z - 1) {
      *args.done_counter = 0;
      __threadfence();
      signal_peers(args.signal);
    }
  }
  if (args.timing && tid == 0) args.timing[cta_linear * 8 + 7] = globaltimer_ns();
}

}  // namespace tgemm
