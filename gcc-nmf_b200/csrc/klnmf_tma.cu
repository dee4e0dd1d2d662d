// KL-NMF (reference: gccNMF/gccNMFFunctions.py:69-83) on the TMA-fed wgmma GEMM over pre-split bf16 planes (tma_gemm.cuh).
//
// Every matrix lives in ONE orientation; the four contractions of an iteration pick the wgmma operand layout
// (K-major / MN-major) that matches it, so nothing is transposed or re-split inside the loop:
//   U    (F, K)   float32 master (the caller's W buffer) + bf16 hi/lo planes Up (F, K)
//   G^T  (T2, K)  float32 master HT32 + planes HTp          (the caller's H (K, T2) is read once and written once)
//   V^T  (T2, Fp) float32 (epilogue operand only)
//   R^T  (T2, Fp) planes RTp only, R = V / (U G)            Fp = F rounded up to 8 (16-byte plane rows)
//
// Gauge.  The reference renormalises after every W update: n = ||W'[:, k]||, W = W' / n, H = n H (:79-:81).  W.H, both
// multiplicative updates and the next norms are covariant under that per-atom rescaling, so the loop carries the UNNORMALISED pair
// (U, G) with W_ref = U / c, H_ref = c G, c = column norms of U -- and c enters the arithmetic in exactly one place, the
// sparsity / epsilon term of the H update:
//      G <- G * (U^T R) / (colsum(U) + c (alpha + eps))           (:76 multiplied through by c)
//      U <- U * (R G^T) / rowsum(G)                                (:77; the c's cancel)         c <- ||U[:, k]||
// Nothing is rescaled inside the loop (the reference rewrites W and the 15 MB of H every iteration); the normalisation is applied
// once, when the caller's W and H are written (finish).  Before the first W update c = 1 (the reference's W0 is not normalised).
//
// One iteration, reference order (:76-:77); M = accumulator rows (the coalesced store direction):
//   G1  RTp = split(VT / (U . G^T))       M = f,    N = t,    over atoms   A = Up K-major,   B = HTp K-major
//   G2  HT32, HTp = G * (U^T . R) / (colsum(U) + c (alpha + eps)); row-sum partials
//                                          M = atom, N = t,    over f       A = Up MN-major,  B = RTp K-major
//   G3  RTp = split(VT / (U . G^T))       again with the new G
//   G4  partial[z] = (R . G^T)^T          M = atom, N = f,    over frames  A = HTp MN-major, B = RTp MN-major, split over z
//   A   U *= sum_z partial / rowsum(G); planes Up; per-row-block partial column sums and sums of squares (-> colsum(U), c)
// F = 513 = 4 x 128 + 1: the row past the last full 128-row tile of G1 / G3 is computed in float32 SIMT by the tile CTAs'
// epilogue warps while the main loop runs.
// Tile widths are chosen per contraction by a cost model over the SM count of the device (make_plan).
#include <algorithm>
#include <cstring>
#include <mutex>
#include <utility>
#include <vector>

#include "common.cuh"
#include "tma_gemm_host.cuh"

void gccnmf_tmap_cache_free(gccnmf_handle* h) {
  delete h->tmaps;
  h->tmaps = nullptr;
}

namespace {

using namespace tgemm_host;

constexpr int kApplyTile = 32;

// ------------------------------------------------------------------------------------------------ epilogues
// (concept: tma_gemm.cuh)  A warp owns column n; the lane holds rows m .. m + 3, contiguous in every output below.
// at_offset(bytes): the same functor with every buffer pointer moved `bytes` on (the clip of a batched launch, tgemm::Clips).
// at_clip(table, c): the same functor with clip c's buffers and length from a ragged run's per-clip table (tgemm::Ragged).
template <class T>
__device__ __forceinline__ T* byte_offset(T* p, int64_t bytes) {
  return p ? reinterpret_cast<T*>(reinterpret_cast<typename std::conditional<std::is_const<T>::value, const char, char>::type*>(p) + bytes) : p;
}
// One clip of a ragged run (gccnmf_klnmf_ragged), in the call's workspace table: its V, W and H, its own workspace carve, and the
// k-splits and row-sum slots of its solo plan.
struct RaggedClip {
  const float* V; int64_t ld_v; float* W; float* H;
  float *HT, *VT, *partial, *colsum, *sumsq_part, *rowsum_part;
  bf16 *HTp, *Wp, *RTp;
  int64_t plane_ht, plane_rt;
  int T2, splits, rowsum_slots;
};
struct EpiStoreT {   // DT[z][n][m] = acc.  G4 partials (m = atom, n = f) and the test entry.
  struct State {};
  struct Loaded {};
  static constexpr bool kDualN = true;       // (takes effect for K-major B tiles of <= 128 columns: the test entry covers the dual-N loop,
                                             // whose products are the plain loop's three)
  static constexpr bool kRowReduce = false;
  static constexpr int kRowValues = 0;
  static constexpr bool kPrefetch = false;
  float* __restrict__ DT; int64_t ld, slab; int M, N; bool vec; bool streaming;
  __device__ void prefetch(int, int) const {}
  __device__ void row_values(int, float*) const {}
  __device__ void init(State&, int, const float*) const {}
  __device__ float4 row_partial(const State&) const { return make_float4(0.f, 0.f, 0.f, 0.f); }
  __device__ void row_total(int, int, float) const {}
  __device__ void elem(int m, int n, float acc, int z) const { DT[(int64_t)z * slab + (int64_t)n * ld + m] = acc; }
  __device__ EpiStoreT at_offset(int64_t bytes) const { EpiStoreT e = *this; e.DT = byte_offset(DT, bytes); return e; }
  __device__ EpiStoreT at_clip(const void* table, int c) const { EpiStoreT e = *this; e.DT = static_cast<const RaggedClip*>(table)[c].partial; return e; }
  __device__ Loaded load(int, int) const { return Loaded{}; }
  __device__ void store(int m, int n, const float4& acc, const Loaded&, int z, State&) const {
    const int valid = min(4, M - m);
    if (valid <= 0) return;
    if (streaming) store4_streaming(DT + (int64_t)z * slab + (int64_t)n * ld + m, acc, valid, vec);
    else store4(DT + (int64_t)z * slab + (int64_t)n * ld + m, acc, valid, vec);
  }
};

struct EpiRatioPlanes {   // RT[n][m] = split(VT[n][m] / acc)     G1 / G3 (m = f, n = t)
  struct State {};
  struct Loaded { float4 vt; };
  static constexpr bool kRowReduce = false;
  static constexpr int kRowValues = 0;
  static constexpr bool kPrefetch = false;   // V^T is read twice per iteration and stays in L2 (96 % hit rate measured)
  static constexpr bool kDualN = true;       // 2 MMAs per k-step, N = BN and N = 2 BN (the three hi / lo products), see tma_gemm.cuh
  static constexpr bool kPreloadOperands = true;   // V^T of the thread's columns is fetched while the main loop runs (wide tiles)
  static constexpr bool kSmemOperand = true;       // V^T tile by TMA into shared memory where the tile leaves room for it
  const float* __restrict__ VT; bf16* __restrict__ RT; int64_t ld, plane; int M, N; bool vec;
  CUtensorMap operand_map;                         // (encoded by the launcher)
  const float* operand() const { return VT; }
  __device__ EpiRatioPlanes at_offset(int64_t bytes) const {
    EpiRatioPlanes e;
    e.VT = byte_offset(VT, bytes); e.RT = byte_offset(RT, bytes);
    e.ld = ld; e.plane = plane; e.M = M; e.N = N; e.vec = vec;
    return e;
  }
  __device__ EpiRatioPlanes at_clip(const void* table, int c) const {
    const RaggedClip& r = static_cast<const RaggedClip*>(table)[c];
    EpiRatioPlanes e;
    e.VT = r.VT; e.RT = r.RTp;
    e.ld = ld; e.plane = r.plane_rt; e.M = M; e.N = r.T2; e.vec = vec;
    return e;
  }
  int64_t operand_ld() const { return ld; }
  int operand_cols() const { return N; }
  __device__ void prefetch(int, int) const {}
  __device__ void row_values(int, float*) const {}
  __device__ void init(State&, int, const float*) const {}
  __device__ float4 row_partial(const State&) const { return make_float4(0.f, 0.f, 0.f, 0.f); }
  __device__ void row_total(int, int, float) const {}
  __device__ void elem(int m, int n, float acc, int) const {
    bf16 hi, lo;
    split_bf16(VT[(int64_t)n * ld + m] / acc, hi, lo);
    RT[(int64_t)n * ld + m] = hi;
    RT[plane + (int64_t)n * ld + m] = lo;
  }
  __device__ Loaded load(int m, int n) const { return Loaded{load4(VT + (int64_t)n * ld + m, min(4, M - m), vec, 1.f)}; }
  __device__ void store(int m, int n, const float4& acc, const Loaded& l, int, State&) const {
    const int valid = min(4, M - m);
    if (valid <= 0) return;
    // V / (W H) with the hardware reciprocal (<= 2 ulp; the IEEE division sequence is ~10 instructions per element and made
    // this epilogue instruction-bound)
    const float4 r = make_float4(__fdividef(l.vt.x, acc.x), __fdividef(l.vt.y, acc.y), __fdividef(l.vt.z, acc.z), __fdividef(l.vt.w, acc.w));
    store_planes4(RT + (int64_t)n * ld + m, plane, r, valid, vec);
  }
};

// G2 (m = atom, n = frame): G <- G * acc / (colsum(U)[m] + c[m] (alpha + eps))  (:76 in the (U, G) gauge, see the header).
// G^T is updated in place (float32 master + planes); the per-row sums of the new G over the tile's columns go to
// rowsum_part[tile_n][m] (one writer per value, fixed summation order, no atomics).
struct EpiUpdateH {
  struct State { float4 rden, rsum; };
  struct Loaded { float4 old; };
  static constexpr bool kRowReduce = true;
  static constexpr int kRowValues = 1;   // 1 / (colsum(U)[m] + c[m] (alpha + eps))
  static constexpr bool kPrefetch = true;
  __device__ void prefetch(int m, int n) const {
    if (m < M) tgemm::prefetch_l2(HT + (int64_t)n * ld + m);
  }
  float* __restrict__ HT; bf16* __restrict__ HTp; const float* __restrict__ colsum_part; const float* __restrict__ sumsq_part;
  float* __restrict__ rowsum_part; float alpha, eps; int64_t ld, plane; int M, N; int slots; bool vec;
  __device__ EpiUpdateH at_offset(int64_t bytes) const {
    EpiUpdateH e = *this;
    e.HT = byte_offset(HT, bytes); e.HTp = byte_offset(HTp, bytes); e.colsum_part = byte_offset(colsum_part, bytes);
    e.sumsq_part = byte_offset(sumsq_part, bytes); e.rowsum_part = byte_offset(rowsum_part, bytes);
    return e;
  }
  __device__ EpiUpdateH at_clip(const void* table, int c) const {     // (sumsq_part: non-NULL once the W update has left the clip's)
    const RaggedClip& r = static_cast<const RaggedClip*>(table)[c];
    EpiUpdateH e = *this;
    e.HT = r.HT; e.HTp = r.HTp; e.colsum_part = r.colsum;
    e.sumsq_part = sumsq_part ? r.sumsq_part : nullptr; e.rowsum_part = r.rowsum_part;
    e.plane = r.plane_ht; e.N = r.T2;
    return e;
  }
  __device__ void row_values(int m, float* v) const {
    v[0] = 1.f;
    if (m >= M) return;
    float c = 0.f, q = 0.f;
    for (int b0 = 0; b0 < slots; b0 += 8) {       // the W update's per-row-block partials, 8 (+ 8) loads in flight
      float p[8], r[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        p[j] = (b0 + j < slots) ? colsum_part[(int64_t)(b0 + j) * M + m] : 0.f;
        r[j] = (sumsq_part && b0 + j < slots) ? sumsq_part[(int64_t)(b0 + j) * M + m] : 0.f;
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) { c += p[j]; q += r[j]; }
    }
    const float nrm = sumsq_part ? sqrtf(q) : 1.f;         // c = ||U[:, m]||; 1 before the first W update (W0 is not normalised)
    v[0] = 1.f / ((c + nrm * alpha) + nrm * eps);
  }
  __device__ void init(State& s, int, const float* rowvals) const {
    s.rsum = make_float4(0.f, 0.f, 0.f, 0.f);
    s.rden = *reinterpret_cast<const float4*>(rowvals);
  }
  __device__ float4 row_partial(const State& s) const { return s.rsum; }
  __device__ void row_total(int m, int tile_n, float sum) const {
    if (m < M) rowsum_part[(int64_t)tile_n * M + m] = sum;
  }
  __device__ void elem(int, int, float, int) const {}   // M = atoms is tiled without SIMT tail rows
  __device__ Loaded load(int m, int n) const { return Loaded{load4(HT + (int64_t)n * ld + m, max(0, min(4, M - m)), vec, 0.f)}; }
  __device__ void store(int m, int n, const float4& acc, const Loaded& l, int, State& s) const {
    const int valid = min(4, M - m);
    if (valid <= 0) return;
    const float4 o = l.old;
    // acc / denom as acc * (1 / denom): the reciprocal is one IEEE division per row, shared by the tile's columns
    float4 hv = make_float4(o.x * (acc.x * s.rden.x), o.y * (acc.y * s.rden.y), o.z * (acc.z * s.rden.z), o.w * (acc.w * s.rden.w));
    if (valid < 4) {
      if (valid < 2) hv.y = 0.f;
      if (valid < 3) hv.z = 0.f;
      hv.w = 0.f;
    }
    const int64_t i = (int64_t)n * ld + m;
    store4(HT + i, hv, valid, vec);
    store_planes4(HTp + i, plane, hv, valid, vec);
    s.rsum.x += hv.x; s.rsum.y += hv.y; s.rsum.z += hv.z; s.rsum.w += hv.w;
  }
};

// ------------------------------------------------------------------------------------------------ small kernels
// dst32 (cols, ld32) = src (rows, cols; ld_src)^T, zero in the pad columns [rows, ld32); optional hi/lo planes (cols, ldp).
// Each small kernel below has a `_clips` form for batched runs (gccnmf_klnmf_batched): the clip comes from the last grid index, the
// caller's matrices of clip c lie c clip strides on, and its workspace buffers c * ws_clip_bytes on (one carve per clip).
__device__ __forceinline__ void transpose_split(const float* __restrict__ src, int rows, int cols, int64_t ld_src, float* __restrict__ dst32,
                                                int64_t ld32, bf16* __restrict__ planes, int64_t ldp, int64_t plane) {
  __shared__ float tile[32][33];
  const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int r = r0 + i, c = c0 + threadIdx.x;
    tile[i][threadIdx.x] = (r < rows && c < cols) ? src[(int64_t)r * ld_src + c] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, r = r0 + threadIdx.x;
    if (c >= cols) continue;
    const float x = tile[threadIdx.x][i];
    if (dst32 && r < ld32) dst32[(int64_t)c * ld32 + r] = x;
    if (planes && r < ldp) {
      bf16 hi, lo;
      split_bf16(x, hi, lo);
      planes[(int64_t)c * ldp + r] = hi;
      planes[plane + (int64_t)c * ldp + r] = lo;
    }
  }
}
__global__ void tma_transpose_split_kernel(const float* __restrict__ src, int rows, int cols, int64_t ld_src, float* __restrict__ dst32,
                                           int64_t ld32, bf16* __restrict__ planes, int64_t ldp, int64_t plane) {
  transpose_split(src, rows, cols, ld_src, dst32, ld32, planes, ldp, plane);
}
__global__ void tma_transpose_split_clips_kernel(const float* __restrict__ src, int rows, int cols, int64_t ld_src, int64_t src_clip,
                                                 float* __restrict__ dst32, int64_t ld32, bf16* __restrict__ planes, int64_t ldp, int64_t plane,
                                                 int64_t ws_clip_bytes) {
  const int64_t c = blockIdx.z;
  transpose_split(src + c * src_clip, rows, cols, ld_src, byte_offset(dst32, c * ws_clip_bytes), ld32, byte_offset(planes, c * ws_clip_bytes),
                  ldp, plane);
}

__device__ __forceinline__ void split_planes(const float* __restrict__ src, int64_t n, bf16* __restrict__ planes, int64_t plane) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  bf16 hi, lo;
  split_bf16(src[i], hi, lo);
  planes[i] = hi;
  planes[plane + i] = lo;
}
__global__ void tma_split_kernel(const float* __restrict__ src, int64_t n, bf16* __restrict__ planes, int64_t plane) { split_planes(src, n, planes, plane); }
__global__ void tma_split_clips_kernel(const float* __restrict__ src, int64_t n, bf16* __restrict__ planes, int64_t plane, int64_t ws_clip_bytes) {
  const int64_t c = blockIdx.y;
  split_planes(src + c * n, n, byte_offset(planes, c * ws_clip_bytes), plane);
}

// planes (rows, pitch) = split(src (rows, inner)) row by row (pitch >= inner; pad columns are left as they are).
__global__ void tma_split_rows_kernel(const float* src, int rows, int inner, bf16* planes, int64_t pitch, int64_t plane) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)rows * inner) return;
  const int r = (int)(i / inner), col = (int)(i - (int64_t)r * inner);
  bf16 hi, lo;
  split_bf16(src[i], hi, lo);
  planes[(int64_t)r * pitch + col] = hi;
  planes[plane + (int64_t)r * pitch + col] = lo;
}

__device__ __forceinline__ void column_sums(const float* W, int F, int K, float* colsum) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= K) return;
  float s = 0.f;
  for (int f = 0; f < F; ++f) s += W[(int64_t)f * K + k];   // row order like numpy.sum(W, axis=0)
  colsum[k] = s;
}
__global__ void tma_colsum_kernel(const float* W, int F, int K, float* colsum) { column_sums(W, F, K, colsum); }
__global__ void tma_colsum_clips_kernel(const float* W, int F, int K, float* colsum, int64_t ws_clip_bytes) {
  const int64_t c = blockIdx.y;
  column_sums(W + c * F * K, F, K, byte_offset(colsum, c * ws_clip_bytes));
}

// Cross-rank sum read straight from the NVSwitch: p is the multicast address of a symmetric buffer, every rank's copy of the
// 16 bytes is fetched and added inside the switch (SASS LDGMC.E.ADD.F32x4).
__device__ __forceinline__ float4 multimem_sum_f32x4(const float* p) {
  float4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
  return v;
}

// W update, one fully parallel pass over tiles of 32 rows x 128 atoms (grid: atoms / 128 x rows / 32 = 8 x 17 = 136 CTAs at the
// headline shape: one wave): a thread owns 4 consecutive atoms (one 16-byte access per matrix) of 4 rows, with every load of
// its 4 rows -- 4 x (k-split partials + U) -- in flight before the first use:
//   U <- U * (sum_z partial[z]) / rowsum(G)  (:77 in the (U, G) gauge); planes of U; per-tile column sums and column sums of
//   squares -> colsum_part / sumsq_part[row block][atom] (summed by their consumers: colsum(U) and c = ||U[:, k]||)
constexpr int kApplyAtoms = 128;      // atoms per CTA (32 lanes x 4)
// Where the numerator and the row sums of G come from:
//   kApplyLocal     this GPU's k-split partials / row-sum slots (single-GPU loop, or an all-reduced numerator given by the caller)
//   kApplyMultimem  one-shot in the switch: every word is the multimem.ld_reduce sum over the ranks' symmetric buffers
//   kApplyPull      one-shot pull: every rank's numerator and row-sum slots are read from its own memory over NVLink (peer-mapped
//                   addresses) and added in rank order -- plain loads pipeline where multimem.ld_reduce took ~8 us for 2 MB
//   kApplyPullOwner two-shot pull: the numerator word comes from the rank that owns (and has already summed) its slice
enum { kApplyLocal = 0, kApplyMultimem = 1, kApplyPull = 2, kApplyPullOwner = 3 };
struct PeerSet {
  const float* numer[8];     // each rank's numerator buffer (F*K floats)
  const float* rowsum[8];    // each rank's row-sum slots (rowsum_slots x K)
  const float* reduced[8];   // each rank's slice-owner buffer (two-shot pull)
  int world;
  int64_t chunk4;            // float4 words per owned slice (two-shot pull)
};
__device__ __forceinline__ float4 ld_sys_f32x4(const float* p) {      // strong system-scope load: never served from a stale non-coherent line
  float4 v;
  asm volatile("ld.relaxed.sys.global.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
  return v;
}
template <int MODE>
__device__ __forceinline__ void
apply_w(float* __restrict__ U, bf16* __restrict__ Up, int64_t plane, const float* __restrict__ partial, int splits,
        const float* __restrict__ rowsum, int rowsum_slots, int F, int K, float* __restrict__ sumsq_part, float* __restrict__ colsum_part,
        const unsigned* arrival_counter, unsigned arrivals_expected, unsigned long long* stamp, const PeerSet& peers) {
  constexpr bool MULTIMEM = MODE == kApplyMultimem;
  constexpr bool PULL = MODE == kApplyPull || MODE == kApplyPullOwner;
  __shared__ float4 part[2][8][32];
  tgemm::pdl_launch_dependents();
  tgemm::pdl_wait_prior_grids();
  const int c = threadIdx.x, g = threadIdx.y;          // c: lane (4 atoms), g: row group 0..7
  const bool stamping = stamp != nullptr && blockIdx.x == 0 && blockIdx.y == 0 && c == 0 && g == 0;   // diagnostics (gccnmf_debug_timing)
  if (stamping) stamp[0] = tgemm::globaltimer_ns();
  if (arrival_counter) {
    // every rank's contribution is in place once my copy of the counter has received all arrivals
    if (c == 0 && g == 0) {
      unsigned seen;
      unsigned long long spins = 0;
      do {
        asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(seen) : "l"(arrival_counter) : "memory");
        if (++spins > (1ull << 25)) __trap();   // a lost peer must not hang the box
      } while ((int)(seen - arrivals_expected) < 0);
    }
    __syncthreads();
  }
  if (stamping) stamp[1] = tgemm::globaltimer_ns();
  const int k = blockIdx.x * kApplyAtoms + 4 * c;       // K % 8 == 0 on this path: a thread's 4 atoms are all inside or all outside
  const int64_t slab = (int64_t)F * K;
  const bool active = k < K;
  // every global load of the thread is issued before the first one is used: the row-sum slots (spread over the 8 row groups),
  // the k-split partials and U of its 4 rows
  float4 rs_part = make_float4(0.f, 0.f, 0.f, 0.f);
  float4 numer[kApplyTile / 8], u[kApplyTile / 8];
  float4 p[kApplyTile / 8][kMaxSplits];
  if (active) {
    if (PULL) {
      for (int rank = 0; rank < peers.world; ++rank)
        for (int s = g; s < rowsum_slots; s += 8) {
          const float4 v = ld_sys_f32x4(peers.rowsum[rank] + (int64_t)s * K + k);
          rs_part.x += v.x; rs_part.y += v.y; rs_part.z += v.z; rs_part.w += v.w;
        }
    } else if (!MULTIMEM) {
      for (int s = g; s < rowsum_slots; s += 8) {
        const float4 v = arrival_counter ? __ldcg(reinterpret_cast<const float4*>(rowsum + (int64_t)s * K + k)) : __ldg(reinterpret_cast<const float4*>(rowsum + (int64_t)s * K + k));
        rs_part.x += v.x; rs_part.y += v.y; rs_part.z += v.z; rs_part.w += v.w;
      }
    }
#pragma unroll
    for (int r = 0; r < kApplyTile / 8; ++r) {
      const int f = blockIdx.y * kApplyTile + g + 8 * r;
      numer[r] = u[r] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (f < F) {
        const int64_t i = (int64_t)f * K + k;
        u[r] = *reinterpret_cast<const float4*>(U + i);
        if (MULTIMEM) {
          numer[r] = multimem_sum_f32x4(partial + i);      // sum over ranks, reduced inside the NVSwitch
        } else if (MODE == kApplyPull) {
#pragma unroll
          for (int z = 0; z < kMaxSplits; ++z)              // (z = rank: the ranks' numerators take the place of the k-split slabs)
            p[r][z] = z < splits ? ld_sys_f32x4(peers.numer[z] + i) : make_float4(0.f, 0.f, 0.f, 0.f);
        } else if (MODE == kApplyPullOwner) {
          const int owner = (int)((i >> 2) / peers.chunk4);
#pragma unroll
          for (int z = 1; z < kMaxSplits; ++z) p[r][z] = make_float4(0.f, 0.f, 0.f, 0.f);
          p[r][0] = ld_sys_f32x4(peers.reduced[owner] + i);
        } else {
#pragma unroll
          for (int z = 0; z < kMaxSplits; ++z)
            p[r][z] = z < splits ? (arrival_counter ? __ldcg(reinterpret_cast<const float4*>(partial + (int64_t)z * slab + i))      // written by peers: not through L1
                                                   : __ldg(reinterpret_cast<const float4*>(partial + (int64_t)z * slab + i)))
                                 : make_float4(0.f, 0.f, 0.f, 0.f);
        }
      }
    }
  }
  part[0][g][c] = rs_part;
  __syncthreads();
  float4 rs = make_float4(1.f, 1.f, 1.f, 1.f);
  if (active) {
    if (MULTIMEM) {
      rs = multimem_sum_f32x4(rowsum + k);
    } else {
      rs = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int j = 0; j < 8; ++j) { const float4 v = part[0][j][c]; rs.x += v.x; rs.y += v.y; rs.z += v.z; rs.w += v.w; }
#pragma unroll
      for (int r = 0; r < kApplyTile / 8; ++r) {        // split partials summed in split order
        numer[r] = p[r][0];
#pragma unroll
        for (int z = 1; z < kMaxSplits; ++z)
          if (z < splits) { numer[r].x += p[r][z].x; numer[r].y += p[r][z].y; numer[r].z += p[r][z].z; numer[r].w += p[r][z].w; }
      }
    }
  }
  __syncthreads();                                       // part[] is reused below
  if (stamping) stamp[2] = tgemm::globaltimer_ns();      // (the numerator and row sums of this CTA have arrived)
  float4 sumsq = make_float4(0.f, 0.f, 0.f, 0.f), csum = make_float4(0.f, 0.f, 0.f, 0.f);
  if (active) {
#pragma unroll
    for (int r = 0; r < kApplyTile / 8; ++r) {
      const int f = blockIdx.y * kApplyTile + g + 8 * r;
      if (f < F) {
        const int64_t i = (int64_t)f * K + k;
        const float4 w = make_float4(u[r].x * (numer[r].x / rs.x), u[r].y * (numer[r].y / rs.y), u[r].z * (numer[r].z / rs.z), u[r].w * (numer[r].w / rs.w));
        *reinterpret_cast<float4*>(U + i) = w;
        store_planes4(Up + i, plane, w, 4, true);
        sumsq.x += w.x * w.x; sumsq.y += w.y * w.y; sumsq.z += w.z * w.z; sumsq.w += w.w * w.w;
        csum.x += w.x; csum.y += w.y; csum.z += w.z; csum.w += w.w;
      }
    }
  }
  part[0][g][c] = sumsq;
  part[1][g][c] = csum;
  __syncthreads();
  if (g < 2 && active) {
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int j = 0; j < 8; ++j) { const float4 v = part[g][j][c]; s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w; }
    *reinterpret_cast<float4*>((g == 0 ? sumsq_part : colsum_part) + (int64_t)blockIdx.y * K + k) = s;
  }
  if (stamping) stamp[7] = tgemm::globaltimer_ns();
}
template <int MODE>
__global__ void __launch_bounds__(256)
tma_apply_w_kernel(float* __restrict__ U, bf16* __restrict__ Up, int64_t plane, const float* __restrict__ partial, int splits,
                   const float* __restrict__ rowsum, int rowsum_slots, int F, int K, float* __restrict__ sumsq_part, float* __restrict__ colsum_part,
                   const unsigned* arrival_counter, unsigned arrivals_expected, unsigned long long* stamp, PeerSet peers) {
  apply_w<MODE>(U, Up, plane, partial, splits, rowsum, rowsum_slots, F, K, sumsq_part, colsum_part, arrival_counter, arrivals_expected, stamp, peers);
}
// The single-GPU W update of every clip of a batch (this GPU's k-split slabs and row-sum slots), clip = blockIdx.z.
__global__ void __launch_bounds__(256)
tma_apply_w_clips_kernel(float* __restrict__ U, bf16* __restrict__ Up, int64_t plane, const float* __restrict__ partial, int splits,
                         const float* __restrict__ rowsum, int rowsum_slots, int F, int K, float* __restrict__ sumsq_part,
                         float* __restrict__ colsum_part, int64_t ws_clip_bytes) {
  const int64_t c = blockIdx.z, o = c * ws_clip_bytes;
  apply_w<kApplyLocal>(U + c * F * K, byte_offset(Up, o), plane, byte_offset(partial, o), splits, byte_offset(rowsum, o), rowsum_slots, F, K,
                       byte_offset(sumsq_part, o), byte_offset(colsum_part, o), nullptr, 0u, nullptr, PeerSet{});
}

// W update with the cross-rank exchange INSIDE it, tile by tile (frame-sharded runs, gccnmf_klnmf_step_pull form 2): the CTA that
// owns a 32 x 128 tile of U sums this rank's k-split slabs for that tile, writes the packed tile into this rank's symmetric buffer and
// adds 1 to the tile's flag on every rank (device-scope fence + relaxed red: the published data is local, peers fetch it through this
// GPU's L2); it then waits until its own flag shows one arrival per rank -- the same-tile CTAs of the other ranks, all resident: the
// grid is one wave -- reads their packed tiles and every rank's row-sum slots with plain peer loads, adds in rank order and updates U.
// No pack kernel, no slice-reduction kernel, no kernel boundary inside the exchange: five launches per iteration like the single-GPU
// loop.  Every rank adds the same values in the same order: bit-identical U.
__global__ void __launch_bounds__(256)
tma_apply_w_exchange_kernel(float* __restrict__ U, bf16* __restrict__ Up, int64_t plane, const float* __restrict__ partial, int splits, int rowsum_slots,
                            int F, int K, float* __restrict__ sumsq_part, float* __restrict__ colsum_part, PeerSet peers, int me, float* my_numer,
                            tgemm::PeerSignal flags, unsigned arrivals_expected, unsigned long long* stamp) {
  __shared__ float4 part[2][8][32];
  tgemm::pdl_launch_dependents();
  tgemm::pdl_wait_prior_grids();
  const int c = threadIdx.x, g = threadIdx.y;
  const bool first = c == 0 && g == 0;
  const bool stamping = stamp != nullptr && blockIdx.x == 0 && blockIdx.y == 0 && first;
  if (stamping) stamp[0] = tgemm::globaltimer_ns();
  const int tile_id = blockIdx.y * gridDim.x + blockIdx.x;
  const int k = blockIdx.x * kApplyAtoms + 4 * c;
  const int64_t slab = (int64_t)F * K;
  const bool active = k < K;
  float4 numer[kApplyTile / 8], u[kApplyTile / 8];
  float4 p[kApplyTile / 8][kMaxSplits];
  // ---- phase A: this rank's tile = sum of its k-split slabs (split order), published in the symmetric buffer
  if (active) {
#pragma unroll
    for (int r = 0; r < kApplyTile / 8; ++r) {
      const int f = blockIdx.y * kApplyTile + g + 8 * r;
      numer[r] = u[r] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (f < F) {
        const int64_t i = (int64_t)f * K + k;
        u[r] = *reinterpret_cast<const float4*>(U + i);
#pragma unroll
        for (int z = 0; z < kMaxSplits; ++z)
          p[r][z] = z < splits ? __ldg(reinterpret_cast<const float4*>(partial + (int64_t)z * slab + i)) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
#pragma unroll
    for (int r = 0; r < kApplyTile / 8; ++r) {
      const int f = blockIdx.y * kApplyTile + g + 8 * r;
      if (f < F) {
        numer[r] = p[r][0];
#pragma unroll
        for (int z = 1; z < kMaxSplits; ++z)
          if (z < splits) { numer[r].x += p[r][z].x; numer[r].y += p[r][z].y; numer[r].z += p[r][z].z; numer[r].w += p[r][z].w; }
        *reinterpret_cast<float4*>(my_numer + (int64_t)f * K + k) = numer[r];
      }
    }
  }
  __syncthreads();
  if (first) {
    __threadfence();
    for (int r = 0; r < flags.world; ++r)
      asm volatile("red.relaxed.sys.global.add.u32 [%0], %1;" ::"l"(flags.counters[r] + tile_id), "r"(1u) : "memory");
    if (stamping) stamp[1] = tgemm::globaltimer_ns();
    // ---- phase B: the same tile of every rank has been published
    unsigned seen;
    unsigned long long spins = 0;
    do {
      asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(seen) : "l"(flags.counters[me] + tile_id) : "memory");
      if (++spins > (1ull << 25)) __trap();     // a lost peer must not hang the box
    } while ((int)(seen - arrivals_expected) < 0);
  }
  __syncthreads();
  if (stamping) stamp[2] = tgemm::globaltimer_ns();
  // ---- phase C: the other ranks' tiles and every rank's row sums of G, all loads in flight before the first add
  float4 rs_part = make_float4(0.f, 0.f, 0.f, 0.f);
  if (active) {
    for (int rank = 0; rank < peers.world; ++rank)
      for (int s = g; s < rowsum_slots; s += 8) {
        const float4 v = ld_sys_f32x4(peers.rowsum[rank] + (int64_t)s * K + k);
        rs_part.x += v.x; rs_part.y += v.y; rs_part.z += v.z; rs_part.w += v.w;
      }
#pragma unroll
    for (int r = 0; r < kApplyTile / 8; ++r) {
      const int f = blockIdx.y * kApplyTile + g + 8 * r;
      if (f < F) {
        const int64_t i = (int64_t)f * K + k;
#pragma unroll
        for (int z = 0; z < kMaxSplits; ++z)
          p[r][z] = (z < peers.world && z != me) ? ld_sys_f32x4(peers.numer[z] + i) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
  }
  part[0][g][c] = rs_part;
  __syncthreads();
  float4 rs = make_float4(1.f, 1.f, 1.f, 1.f);
  if (active) {
    rs = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int j = 0; j < 8; ++j) { const float4 v = part[0][j][c]; rs.x += v.x; rs.y += v.y; rs.z += v.z; rs.w += v.w; }
#pragma unroll
    for (int r = 0; r < kApplyTile / 8; ++r) {          // ranks added in rank order (mine from registers)
      const float4 mine = numer[r];
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int z = 0; z < kMaxSplits; ++z)
        if (z < peers.world) {
          const float4 v = z == me ? mine : p[r][z];
          if (z == 0) acc = v;
          else { acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w; }
        }
      numer[r] = acc;
    }
  }
  __syncthreads();                                       // part[] is reused below
  if (stamping) stamp[3] = tgemm::globaltimer_ns();
  float4 sumsq = make_float4(0.f, 0.f, 0.f, 0.f), csum = make_float4(0.f, 0.f, 0.f, 0.f);
  if (active) {
#pragma unroll
    for (int r = 0; r < kApplyTile / 8; ++r) {
      const int f = blockIdx.y * kApplyTile + g + 8 * r;
      if (f < F) {
        const int64_t i = (int64_t)f * K + k;
        const float4 w = make_float4(u[r].x * (numer[r].x / rs.x), u[r].y * (numer[r].y / rs.y), u[r].z * (numer[r].z / rs.z), u[r].w * (numer[r].w / rs.w));
        *reinterpret_cast<float4*>(U + i) = w;
        store_planes4(Up + i, plane, w, 4, true);
        sumsq.x += w.x * w.x; sumsq.y += w.y * w.y; sumsq.z += w.z * w.z; sumsq.w += w.w * w.w;
        csum.x += w.x; csum.y += w.y; csum.z += w.z; csum.w += w.w;
      }
    }
  }
  part[0][g][c] = sumsq;
  part[1][g][c] = csum;
  __syncthreads();
  if (g < 2 && active) {
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int j = 0; j < 8; ++j) { const float4 v = part[g][j][c]; s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w; }
    *reinterpret_cast<float4*>((g == 0 ? sumsq_part : colsum_part) + (int64_t)blockIdx.y * K + k) = s;
  }
  if (stamping) stamp[7] = tgemm::globaltimer_ns();
}

// finish: the reference's normalisation (:79-:81), applied once.  c[k] = sqrt(sum of the row-block partial sums of squares).
__device__ __forceinline__ float column_norm(const float* __restrict__ sumsq_part, int row_blocks, int K, int k) {
  float q = 0.f;
  for (int b = 0; b < row_blocks; ++b) q += sumsq_part[(int64_t)b * K + k];
  return sqrtf(q);
}
__device__ __forceinline__ void finish_w(float* __restrict__ W, int F, int K, const float* __restrict__ sumsq_part, int row_blocks) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= K) return;
  const float nrm = column_norm(sumsq_part, row_blocks, K, k);
  for (int f = blockIdx.y; f < F; f += gridDim.y) W[(int64_t)f * K + k] = W[(int64_t)f * K + k] / nrm;      // W /= norms (:80)
}
__global__ void tma_finish_w_kernel(float* __restrict__ W, int F, int K, const float* __restrict__ sumsq_part, int row_blocks) {
  finish_w(W, F, K, sumsq_part, row_blocks);
}
__global__ void tma_finish_w_clips_kernel(float* __restrict__ W, int F, int K, const float* __restrict__ sumsq_part, int row_blocks,
                                          int64_t ws_clip_bytes) {
  const int64_t c = blockIdx.z;
  finish_w(W + c * F * K, F, K, byte_offset(sumsq_part, c * ws_clip_bytes), row_blocks);
}

// H (K, T2; caller) = HT32 (T2, K)^T * c (H *= norms, :81) -- or a plain transpose when there was no W update.
__device__ __forceinline__ void finish_h(const float* __restrict__ HT, int T2, int K, const float* __restrict__ sumsq_part, int row_blocks,
                                         float* __restrict__ H) {
  __shared__ float tile[32][33];
  __shared__ float nrm_s[32];
  const int k0 = blockIdx.x * 32, t0 = blockIdx.y * 32;
  if (threadIdx.y == 0) nrm_s[threadIdx.x] = (sumsq_part && k0 + threadIdx.x < K) ? column_norm(sumsq_part, row_blocks, K, k0 + threadIdx.x) : 1.f;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int t = t0 + i, k = k0 + threadIdx.x;
    tile[i][threadIdx.x] = (t < T2 && k < K) ? HT[(int64_t)t * K + k] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int k = k0 + i, t = t0 + threadIdx.x;
    if (k < K && t < T2) {
      const float v = tile[threadIdx.x][i];
      H[(int64_t)k * T2 + t] = sumsq_part ? v * nrm_s[i] : v;
    }
  }
}
__global__ void tma_finish_h_kernel(const float* __restrict__ HT, int T2, int K, const float* __restrict__ sumsq_part, int row_blocks,
                                    float* __restrict__ H) {
  finish_h(HT, T2, K, sumsq_part, row_blocks, H);
}
__global__ void tma_finish_h_clips_kernel(const float* __restrict__ HT, int T2, int K, const float* __restrict__ sumsq_part, int row_blocks,
                                          float* __restrict__ H, int64_t ws_clip_bytes) {
  const int64_t c = blockIdx.z, o = c * ws_clip_bytes;
  finish_h(byte_offset(HT, o), T2, K, byte_offset(sumsq_part, o), row_blocks, H + c * K * T2);
}

// Ragged forms (gccnmf_klnmf_ragged): the clip is the last grid index, its buffers and length come from the table; a grid sized for
// the longest clip returns at once in the frame blocks past a shorter clip's end.
__global__ void tma_prepare_v_ragged_kernel(const RaggedClip* clips, int F, int64_t Fp) {
  const RaggedClip& c = clips[blockIdx.z];
  if ((int)blockIdx.x * 32 >= c.T2) return;
  transpose_split(c.V, F, c.T2, c.ld_v, c.VT, Fp, nullptr, 0, 0);
}
__global__ void tma_prepare_h_ragged_kernel(const RaggedClip* clips, int K) {
  const RaggedClip& c = clips[blockIdx.z];
  if ((int)blockIdx.x * 32 >= c.T2) return;
  transpose_split(c.H, K, c.T2, c.T2, c.HT, K, c.HTp, K, c.plane_ht);
}
__global__ void tma_split_ragged_kernel(const RaggedClip* clips, int64_t n) {
  const RaggedClip& c = clips[blockIdx.y];
  split_planes(c.W, n, c.Wp, n);
}
__global__ void tma_colsum_ragged_kernel(const RaggedClip* clips, int F, int K) {
  const RaggedClip& c = clips[blockIdx.y];
  column_sums(c.W, F, K, c.colsum);
}
__global__ void __launch_bounds__(256) tma_apply_w_ragged_kernel(const RaggedClip* clips, int F, int K) {
  const RaggedClip& c = clips[blockIdx.z];
  apply_w<kApplyLocal>(c.W, c.Wp, (int64_t)F * K, c.partial, c.splits, c.rowsum_part, c.rowsum_slots, F, K, c.sumsq_part, c.colsum, nullptr, 0u,
                       nullptr, PeerSet{});
}
__global__ void tma_finish_h_ragged_kernel(const RaggedClip* clips, int K, int row_blocks, int normalise) {
  const RaggedClip& c = clips[blockIdx.z];
  if ((int)blockIdx.y * 32 >= c.T2) return;
  finish_h(c.HT, c.T2, K, normalise ? c.sumsq_part : nullptr, row_blocks, c.H);
}
__global__ void tma_finish_w_ragged_kernel(const RaggedClip* clips, int F, int K, int row_blocks) {
  finish_w(clips[blockIdx.z].W, F, K, clips[blockIdx.z].sumsq_part, row_blocks);
}

// numer = [sum_z partial[z] (F*K) | sum_s rowsum_part[s] (K)] for the cross-rank sum.
// With `mc_counter` (the NVLink multicast address of a per-buffer arrival counter that every rank holds at the same offset of its
// symmetric buffer): the last CTA to finish adds 1 to that counter ON EVERY RANK with one multimem.red -- "this rank's partial is
// complete" -- so no host-launched barrier sits between the numerator and the W update (tma_apply_w_kernel<true> waits on its own
// copy of the counter).
__global__ void tma_pack_numer_kernel(const float* partial, int splits, int64_t n, const float* rowsum, int rowsum_slots, int K, float* numer,
                                      unsigned* done_counter, unsigned* mc_counter, int light_signal, unsigned long long* stamp,
                                      tgemm::PeerSignal peers_signal) {
  tgemm::pdl_launch_dependents();
  tgemm::pdl_wait_prior_grids();
  if (stamp && blockIdx.x == 0 && threadIdx.x == 0) stamp[0] = tgemm::globaltimer_ns();
  // partial == NULL: the numerator itself is already in place (k-splits summed inside clusters by the contraction): row sums only.
  // 16 bytes per thread and matrix, every slab's load of an item in flight before the first add, a few hundred CTAs (grid-stride):
  // the scalar one-item-per-thread form (2 053 CTAs) took 3.6 us and its completion count 4 more.
  const int64_t n4 = n >> 2, k4 = K >> 2;
  const int64_t first = partial ? 0 : n4, total = n4 + k4;
  for (int64_t i = first + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    if (i < n4) {
      float4 v[kMaxSplits];
#pragma unroll
      for (int z = 0; z < kMaxSplits; ++z)
        v[z] = z < splits ? __ldcg(reinterpret_cast<const float4*>(partial + (int64_t)z * n) + i) : make_float4(0.f, 0.f, 0.f, 0.f);
      acc = v[0];
#pragma unroll
      for (int z = 1; z < kMaxSplits; ++z)
        if (z < splits) { acc.x += v[z].x; acc.y += v[z].y; acc.z += v[z].z; acc.w += v[z].w; }
    } else {
      for (int j = 0; j < rowsum_slots; ++j) {
        const float4 v = __ldcg(reinterpret_cast<const float4*>(rowsum + (int64_t)j * K) + (i - n4));
        acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
      }
    }
    reinterpret_cast<float4*>(numer)[i] = acc;
  }
  if (mc_counter || peers_signal.world > 0) {
    // One device-scope fence per CTA (cumulative over the CTA's stores through the barrier) and ONE system-scope release by the
    // last CTA: a __threadfence_system() per thread (MEMBAR.SC.SYS x 500 k) cost ~20 us per iteration at 2 ranks.
    __syncthreads();
    if (threadIdx.x == 0) {
      __threadfence();
      const unsigned prev = atomicAdd(done_counter, 1u);
      if (prev == gridDim.x - 1) {
        __threadfence();                        // acquire side of the CTA count
        *done_counter = 0;                      // ready for the next iteration (this kernel is never concurrent with itself)
        if (peers_signal.world > 0) {
          tgemm::signal_peers(peers_signal);     // pull exchange: relaxed adds to every rank's counter (see tgemm::PeerSignal)
        } else if (light_signal) {
          // The data this signal publishes lies in THIS GPU's memory and peers fetch it over NVLink through this GPU's L2: a
          // device-scope fence has already put it there, so the arrival is sent relaxed (no MEMBAR.SYS, which costs microseconds).
          asm volatile("multimem.red.relaxed.sys.global.add.u32 [%0], %1;" ::"l"(mc_counter), "r"(1u) : "memory");
        } else {
          __threadfence_system();
          asm volatile("multimem.red.release.sys.global.add.u32 [%0], %1;" ::"l"(mc_counter), "r"(1u) : "memory");
        }
        if (stamp) stamp[7] = tgemm::globaltimer_ns();
      }
    }
  } else if (stamp && blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) {
    stamp[7] = tgemm::globaltimer_ns();
  }
}

// Two-shot all-reduce of the packed numerator inside the NVSwitch (frame-sharded runs, gccnmf_klnmf_step_multimem2): rank r owns the
// r-th slice of the (F*K + K) floats; once every rank's pack has arrived it reads the cross-rank SUM of its slice with
// multimem.ld_reduce and writes it to EVERY rank's `reduced` buffer with multimem.st, then counts itself in on the second arrival
// counter.  Per GPU and iteration the links carry one numerator out and one in, whatever the world size (the one-shot form, every rank
// pulling the whole sum, makes each GPU serve `world` numerators: 16.8 MB per iteration at 8 ranks).
__global__ void tma_reduce_bcast_kernel(const float* numer_mc, float* reduced_mc, int64_t n4, int rank, int world, const unsigned* arrivals_in,
                                        unsigned arrivals_expected, unsigned* done_counter, unsigned* arrivals_out_mc, unsigned long long* stamp) {
  tgemm::pdl_launch_dependents();
  tgemm::pdl_wait_prior_grids();
  const bool stamping = stamp != nullptr && blockIdx.x == 0 && threadIdx.x == 0;
  if (stamping) stamp[0] = tgemm::globaltimer_ns();
  if (threadIdx.x == 0) {
    unsigned seen;
    unsigned long long spins = 0;
    do {
      asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(seen) : "l"(arrivals_in) : "memory");
      if (++spins > (1ull << 25)) __trap();     // a lost peer must not hang the box
    } while ((int)(seen - arrivals_expected) < 0);
  }
  __syncthreads();
  if (stamping) stamp[1] = tgemm::globaltimer_ns();
  const int64_t chunk = (n4 + world - 1) / world, begin = rank * chunk, end = begin + chunk < n4 ? begin + chunk : n4;
  for (int64_t i = begin + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < end; i += (int64_t)gridDim.x * blockDim.x) {
    const float4 v = multimem_sum_f32x4(numer_mc + 4 * i);
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(reduced_mc + 4 * i), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
                 : "memory");
  }
  // this CTA's multicast stores travel over the links: one system-scope fence per CTA (thread 0, after the barrier -- cumulative over
  // the CTA's stores) before the CTA is counted; the last CTA signals every rank
  __syncthreads();
  if (threadIdx.x == 0) {
    if (stamping) stamp[2] = tgemm::globaltimer_ns();
    __threadfence_system();
    if (stamping) stamp[3] = tgemm::globaltimer_ns();
    const unsigned prev = atomicAdd(done_counter, 1u);
    if (prev == gridDim.x - 1) {
      __threadfence();
      *done_counter = 0;
      asm volatile("multimem.red.release.sys.global.add.u32 [%0], %1;" ::"l"(arrivals_out_mc), "r"(1u) : "memory");
      if (stamp) stamp[7] = tgemm::globaltimer_ns();
    }
  }
}

// Two-shot PULL exchange, first shot: rank r sums its slice of the numerator over the ranks with plain loads from their memories
// (rank order: every rank would obtain the same bits) into its OWN `reduced` buffer and signals; the W update of every rank then
// fetches each word from its owner (tma_apply_w_kernel<kApplyPullOwner>).  Per GPU and iteration the links carry one numerator in
// each direction for any world size, nothing is pushed (no system-scope fence), and the loads pipeline.
__global__ void tma_reduce_pull_kernel(PeerSet peers, float* reduced_local, int64_t n4, int rank, const unsigned* arrivals_in,
                                       unsigned arrivals_expected, unsigned* done_counter, tgemm::PeerSignal signal, unsigned long long* stamp) {
  tgemm::pdl_launch_dependents();
  tgemm::pdl_wait_prior_grids();
  const bool stamping = stamp != nullptr && blockIdx.x == 0 && threadIdx.x == 0;
  if (stamping) stamp[0] = tgemm::globaltimer_ns();
  if (threadIdx.x == 0) {
    unsigned seen;
    unsigned long long spins = 0;
    do {
      asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(seen) : "l"(arrivals_in) : "memory");
      if (++spins > (1ull << 25)) __trap();     // a lost peer must not hang the box
    } while ((int)(seen - arrivals_expected) < 0);
  }
  __syncthreads();
  if (stamping) stamp[1] = tgemm::globaltimer_ns();
  const int64_t begin = rank * peers.chunk4, end = begin + peers.chunk4 < n4 ? begin + peers.chunk4 : n4;
  for (int64_t i = begin + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < end; i += (int64_t)gridDim.x * blockDim.x) {
    float4 v[8];
#pragma unroll
    for (int r = 0; r < 8; ++r) v[r] = r < peers.world ? ld_sys_f32x4(peers.numer[r] + 4 * i) : make_float4(0.f, 0.f, 0.f, 0.f);
    float4 acc = v[0];
#pragma unroll
    for (int r = 1; r < 8; ++r)
      if (r < peers.world) { acc.x += v[r].x; acc.y += v[r].y; acc.z += v[r].z; acc.w += v[r].w; }
    *reinterpret_cast<float4*>(reduced_local + 4 * i) = acc;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    if (stamping) stamp[2] = tgemm::globaltimer_ns();
    __threadfence();
    const unsigned prev = atomicAdd(done_counter, 1u);
    if (prev == gridDim.x - 1) {
      *done_counter = 0;
      __threadfence();
      tgemm::signal_peers(signal);
      if (stamp) stamp[7] = tgemm::globaltimer_ns();
    }
  }
}

// ------------------------------------------------------------------------------------------------ tile plan
// Cost model of the planner, in SM cycles of one 128-row CTA, from the per-CTA phase stamps of tools/nmf_phases.py at the benchmark
// shape (H100 SXM, DESIGN.md 4.1).  Per 16-deep k-step the dual-N loop issues MMAs of N = bn and N = 2 bn, the plain loop three of
// N = bn; an MMA costs 1.1 - 1.2 cycles per column of N (both warpgroups; G1 - G4 main loops at widths 120 - 256).  The epilogue
// costs about 95 cycles per column for the ratio (G1 / G3), 93 for the H update (G2), 33 for the plain store of the W-update
// numerator (G4); the fill, the launch and the gaps about 8 k cycles per wave.
constexpr double kEpiRatioCycles = 95.0, kEpiUpdateHCycles = 93.0, kEpiStoreCycles = 33.0;
double mma_cycles(int n) { return 1.2 * n; }
double kstep_cycles(int bn, bool dual) { return (dual && 2 * bn <= 256) ? mma_cycles(2 * bn) + mma_cycles(bn) : 3.0 * mma_cycles(bn); }
double epilogue_cycles(int bn, double per_column) { return per_column * bn; }
constexpr double kWaveCycles = 8000.0;

// m tiles of a launch of `bn`-column tiles, by the launch's own rule (launch_plane_gemm): SIMT tail rows only when the m tiles of
// an n tile can share its columns, at most 128 each (F = 129 .. 136 with 256-column tiles runs two m tiles, not one).
int m_tiles_of(int M, bool simt_tail, int bn) {
  const int tail = M % tgemm::kBM;
  return (simt_tail && tail != 0 && tail <= kTailRowsMax && M > tgemm::kBM && (M / tgemm::kBM) * 128 >= bn) ? M / tgemm::kBM
                                                                                                           : (M + tgemm::kBM - 1) / tgemm::kBM;
}

struct TilePlan { int bn, splits; };

// Picks the tile width (and k-split count when `allow_split`) with the smallest estimated time.
TilePlan plan_tiles(int sm_count, int M, bool simt_tail, int N, int Kc, bool allow_split, const int* widths, int n_widths, double epi_per_column,
                    bool dual = false) {
  TilePlan best{128, 1};
  double best_cost = 1e300;
  const int total_kb = (Kc + kKB - 1) / kKB;
  for (int i = 0; i < n_widths; ++i) {
    const int bn = widths[i];
    const int tiles = m_tiles_of(M, simt_tail, bn) * ((N + bn - 1) / bn);
    int splits = 1;
    if (allow_split) splits = std::max(1, std::min(std::min(kMaxSplits, sm_count / std::max(1, tiles)), total_kb / 4));
    const int kb = (total_kb + splits - 1) / splits;
    const int waves = (tiles * splits + sm_count - 1) / sm_count;
    const double cost = waves * (kb * (kKB / 16) * kstep_cycles(bn, dual) + epilogue_cycles(bn, epi_per_column) + kWaveCycles);
    if (cost < best_cost) { best_cost = cost; best = TilePlan{bn, splits}; }
  }
  return best;
}

const int kWidthsWH[] = {104, 120, 128, 256};     // K-major B: the dual-N loop applies up to 128 columns (112: wh_tile option)
const int kWidthsAll[] = {128, 176, 208, 240, 256};

struct Plan {
  int bn_wh;            // G1 / G3
  int bn_h;             // G2
  TilePlan w;           // G4
  int rowsum_slots;     // n-tiles of G2
};

Plan make_plan(const gccnmf_handle* h, int F, int T2, int K) {
  Plan p;
  p.bn_wh = h->wh_tile ? h->wh_tile : plan_tiles(h->sm_count, F, true, T2, K, false, kWidthsWH, 4, kEpiRatioCycles, true).bn;
  p.bn_h = plan_tiles(h->sm_count, K, false, T2, F, false, kWidthsAll, 5, kEpiUpdateHCycles).bn;
  p.w = plan_tiles(h->sm_count, K, false, F, T2, true, kWidthsAll, 5, kEpiStoreCycles);
  p.rowsum_slots = (T2 + p.bn_h - 1) / p.bn_h;
  return p;
}

// Diagnostics (gccnmf_debug_timing): one 8-slot record per launch of the W update / numerator pack / slice reduction, in launch
// order with the plane GEMMs' per-CTA records.
unsigned long long* next_stamp(gccnmf_handle* h) {
  if (!h->debug_timing) return nullptr;
  unsigned long long* p = h->debug_timing + h->debug_timing_cursor;
  h->debug_timing_cursor += 8;
  return p;
}

// ------------------------------------------------------------------------------------------------ workspace
struct TmaWorkspace {
  float *HT, *VT, *partial, *colsum, *sumsq_part, *rowsum_part;
  unsigned* done;          // CTA completion counter of the numerator pack (cross-rank signalling)
  bf16 *HTp, *Wp, *RTp;
  int64_t Fp, plane_w, plane_ht, plane_rt;
  int row_blocks;
  size_t bytes;
  bool ok;
};

int max_rowsum_slots(int T2) { return (T2 + 127) / 128; }

TmaWorkspace tma_carve(void* ws, size_t bytes, int F, int T2, int K) {
  WorkspaceCarver c(ws ? ws : reinterpret_cast<void*>(256), ws ? bytes : ~size_t(0) >> 1);
  TmaWorkspace w;
  w.Fp = (F + 7) & ~7;
  w.plane_w = (int64_t)F * K;
  w.plane_ht = (int64_t)T2 * K;
  w.plane_rt = (int64_t)T2 * w.Fp;
  w.row_blocks = (F + kApplyTile - 1) / kApplyTile;
  w.HT = c.take<float>((size_t)T2 * K);
  w.HTp = c.take<bf16>((size_t)2 * w.plane_ht);       // right after the float32 master: one L2 access-policy window covers both
  w.VT = c.take<float>((size_t)T2 * w.Fp);
  w.partial = c.take<float>((size_t)kMaxSplits * F * K);
  w.colsum = c.take<float>((size_t)w.row_blocks * K);
  w.sumsq_part = c.take<float>((size_t)w.row_blocks * K);
  w.rowsum_part = c.take<float>((size_t)max_rowsum_slots(T2) * K);
  w.done = c.take<unsigned>(4);
  w.Wp = c.take<bf16>((size_t)2 * w.plane_w);
  w.RTp = c.take<bf16>((size_t)2 * w.plane_rt);
  w.bytes = align_up(c.used, 256);
  w.ok = ws != nullptr && c.ok();
  return w;
}

size_t tma_workspace_bytes(int F, int T2, int K) { return tma_carve(nullptr, 0, F, T2, K).bytes; }

// The W.H contractions (G1, G3) in their second form (option wh_split2): plain 128 x 208 tiles (three MMAs of N = 208 per k-step)
// with the contraction split in two halves that a (1, 1, 2) cluster sums through distributed shared memory before the (non-linear)
// ratio epilogue; each CTA of the pair finishes half of the tile's columns.  72 tiles x 2 = 144 CTAs at the headline shape.
constexpr int kWhSplitTile = 208;
bool wh_split2(gccnmf_handle* h, int F, int T2, int K) {
  if (!h->wh_split2 || K < 128) return false;
  int resident = 0;
  if (plane_gemm_z_clusters<false, false, EpiRatioPlanes>(h, kWhSplitTile, 2, &resident)) return false;
  const int tiles = m_tiles_of(F, true, kWhSplitTile) * ((T2 + kWhSplitTile - 1) / kWhSplitTile);
  return resident >= tiles && 2 * tiles <= h->sm_count;
}
int launch_wh(gccnmf_handle* h, const Plan& p, const Operand& Wk, const Operand& HTk, int F, int T2, int K, const EpiRatioPlanes& e, void* stream) {
  if (wh_split2(h, F, T2, K))
    return plane_gemm_z_reduce<false, false>(h, kWhSplitTile, Wk, HTk, F, T2, K, 2, e, nullptr, stream, nullptr, nullptr, true);
  return plane_gemm<false, false>(h, p.bn_wh, Wk, HTk, F, T2, K, 1, true, e, nullptr, stream);
}

// Whether the W-update numerator contraction sums its k-splits inside (1, 1, splits) clusters through distributed shared memory
// (one (F, K) result, no slabs): when every cluster of the launch can be resident at once (GPC sizes decide), else the k-split slabs
// are written and summed by their consumer as before.
bool w_cluster_reduce(gccnmf_handle* h, const Plan& p, int F, int K) {
  if (!h->w_cluster_reduce || p.w.splits < 2 || p.w.splits > 8) return false;
  int resident = 0;
  if (plane_gemm_z_clusters<true, true, EpiStoreT>(h, p.w.bn, p.w.splits, &resident)) return false;
  const int tiles = m_tiles_of(K, false, p.w.bn) * ((F + p.w.bn - 1) / p.w.bn);
  return resident >= tiles;
}

#define TMA_CARVE_OR_FAIL(w)                                                                                        \
  TmaWorkspace w = tma_carve(workspace, workspace_bytes, F, T2, K);                                                 \
  if (!w.ok) return gccnmf_fail(h, GCCNMF_ERR_WORKSPACE, "klnmf (TMA tensor-core path) workspace too small: need %zu bytes", tma_workspace_bytes(F, T2, K))

}  // namespace

// Whether the TMA path supports this problem (else the float32 SIMT path of klnmf.cu is used).
bool gccnmf_klnmf_tma_supported(int F, int T2, int K) { return K % 8 == 0 && F >= 128 && T2 >= 128 && K >= 32; }
size_t gccnmf_klnmf_tma_workspace_bytes(int F, int T2, int K) { return tma_workspace_bytes(F, T2, K); }

// Builds the operand set from the caller's V (row pitch ld_v), W, H: V^T, planes of W, H^T (float32 + planes).
int gccnmf_klnmf_tma_prepare(gccnmf_handle* h, const float* V, int64_t ld_v, int F, int T2, const float* W, const float* H, int K,
                             void* workspace, size_t workspace_bytes, bool need_vt, bool need_w, bool need_ht, void* stream) {
  TMA_CARVE_OR_FAIL(w);
  const dim3 block(32, 8);
  GCCNMF_CHECK_CUDA(h, cudaMemsetAsync(w.done, 0, 16, (cudaStream_t)stream));
  if (need_vt)
    GCCNMF_LAUNCH(h, tma_transpose_split_kernel, dim3((T2 + 31) / 32, (int)((w.Fp + 31) / 32)), block, 0, stream, V, F, T2, ld_v, w.VT, w.Fp,
                  (bf16*)nullptr, (int64_t)0, (int64_t)0);
  if (need_w) {
    const int64_t n = (int64_t)F * K;
    GCCNMF_LAUNCH(h, tma_split_kernel, (unsigned)((n + 255) / 256), 256, 0, stream, W, n, w.Wp, w.plane_w);
  }
  if (need_ht)
    GCCNMF_LAUNCH(h, tma_transpose_split_kernel, dim3((T2 + 31) / 32, (K + 31) / 32), block, 0, stream, H, K, T2, (int64_t)T2, w.HT, (int64_t)K,
                  w.HTp, (int64_t)K, w.plane_ht);
  return 0;
}

// :76 in the (U, G) gauge: G = G * (U^T (V / (U G))) / (colsum(U) + c (alpha + eps)).
int gccnmf_klnmf_tma_update_H(gccnmf_handle* h, const float* V, int F, int T2, const float* W, float* H, int K, float alpha, float eps,
                              void* workspace, size_t workspace_bytes, int colsum_state, bool pending_norms, void* stream) {
  // colsum_state: 0 = compute colsum(U) now, c = 1 (before the first W update); 1 = reuse the one computed before (fixed dictionary);
  // 2 = per-row-block partial column sums and sums of squares left by the W update
  TMA_CARVE_OR_FAIL(w);
  (void)V; (void)H; (void)pending_norms;
  const Plan p = make_plan(h, F, T2, K);
  const Operand Wk{w.Wp, (int64_t)K, w.plane_w, false};
  const Operand HTk{w.HTp, (int64_t)K, w.plane_ht, false};
  {  // G1: RT = split(VT / (U . G^T))
    EpiRatioPlanes e{w.VT, w.RTp, w.Fp, w.plane_rt, F, T2, true};
    if (int st = launch_wh(h, p, Wk, HTk, F, T2, K, e, stream)) return st;
  }
  if (colsum_state == 0) GCCNMF_LAUNCH(h, tma_colsum_kernel, (K + 127) / 128, 128, 0, stream, W, F, K, w.colsum);
  {  // G2: HT32, HTp = G * (U^T . R) / denom
    const Operand Wmn{w.Wp, (int64_t)K, w.plane_w, true};
    const Operand RTk{w.RTp, w.Fp, w.plane_rt, false};
    EpiUpdateH e{w.HT, w.HTp, w.colsum, colsum_state == 2 ? w.sumsq_part : nullptr, h->xchg_rowsum ? h->xchg_rowsum : w.rowsum_part, alpha, eps,
                 (int64_t)K, w.plane_ht, K, T2,
                 colsum_state == 2 ? w.row_blocks : 1, true};
    if (int st = plane_gemm<true, false>(h, p.bn_h, Wmn, RTk, K, T2, F, 1, false, e, nullptr, stream)) return st;
  }
  return 0;
}

// :77 numerator: partial[z] = (V / (W H)) . H^T over the frame range of split z (row sums of H come from update_H).
int gccnmf_klnmf_tma_partial_W_to(gccnmf_handle* h, const float* V, int F, int T2, const float* W, const float* H, int K,
                                  void* workspace, size_t workspace_bytes, bool have_rowsum, float* numer_out, void* stream) {
  TMA_CARVE_OR_FAIL(w);
  (void)V; (void)W; (void)H;
  if (!have_rowsum) return gccnmf_fail(h, GCCNMF_ERR_UNSUPPORTED, "klnmf (TMA path): partial_W needs the row sums left by update_H");
  const Plan p = make_plan(h, F, T2, K);
  {  // G3: RT = split(VT / (W . H^T))
    const Operand Wk{w.Wp, (int64_t)K, w.plane_w, false};
    const Operand HTk{w.HTp, (int64_t)K, w.plane_ht, false};
    EpiRatioPlanes e{w.VT, w.RTp, w.Fp, w.plane_rt, F, T2, true};
    if (int st = launch_wh(h, p, Wk, HTk, F, T2, K, e, stream)) return st;
  }
  {  // G4: partial[z][f][atom] = sum_t H^T[t][atom] R^T[t][f]
    const Operand HTmn{w.HTp, (int64_t)K, w.plane_ht, true};
    const Operand RTmn{w.RTp, w.Fp, w.plane_rt, true};
    if (w_cluster_reduce(h, p, F, K)) {     // k-splits summed inside clusters: one (F, K) result, straight into numer_out when given
      EpiStoreT e{numer_out ? numer_out : w.partial, (int64_t)K, (int64_t)F * K, K, F, true, false};
      tgemm::PeerSignal sig{};
      sig.world = h->xchg_world;
      for (int r = 0; r < sig.world; ++r) sig.counters[r] = h->xchg_counters[r];
      if (int st = plane_gemm_z_reduce<true, true>(h, p.w.bn, HTmn, RTmn, K, F, T2, p.w.splits, e, nullptr, stream, h->xchg_done, &sig)) return st;
    } else {
      EpiStoreT e{w.partial, (int64_t)K, (int64_t)F * K, K, F, true, h->gemm_streaming != 0};
      if (int st = plane_gemm<true, true>(h, p.w.bn, HTmn, RTmn, K, F, T2, p.w.splits, false, e, nullptr, stream)) return st;
    }
  }
  return 0;
}
int gccnmf_klnmf_tma_partial_W(gccnmf_handle* h, const float* V, int F, int T2, const float* W, const float* H, int K,
                               void* workspace, size_t workspace_bytes, bool have_rowsum, void* stream) {
  return gccnmf_klnmf_tma_partial_W_to(h, V, F, T2, W, H, K, workspace, workspace_bytes, have_rowsum, nullptr, stream);
}

// :77 in the (U, G) gauge (the normalisation of :79-:81 is applied by finish).  Numerator and row sums come from `numer`
// (F*K + K floats, all-reduced across ranks) when given, else from this rank's partials.
int gccnmf_klnmf_tma_apply_W_mc(gccnmf_handle* h, int F, int T2, float* W, int K, const float* numer, bool numer_is_multicast,
                                const unsigned* arrival_counter, unsigned arrivals_expected, void* workspace, size_t workspace_bytes, void* stream) {
  TMA_CARVE_OR_FAIL(w);
  const Plan p = make_plan(h, F, T2, K);
  const float* partial = numer ? numer : w.partial;
  const float* rowsum = numer ? numer + (int64_t)F * K : w.rowsum_part;
  const dim3 grid((K + kApplyAtoms - 1) / kApplyAtoms, w.row_blocks), block(32, 8);
  const PeerSet none{};
  if (numer_is_multicast)
    return launch_ex(h, "tma_apply_w_kernel", tma_apply_w_kernel<kApplyMultimem>, grid, block, 0, stream, h->nmf_pdl, dim3(1, 1, 1), W, w.Wp, w.plane_w,
                     partial, 1, rowsum, 1, F, K, w.sumsq_part, w.colsum, arrival_counter, arrivals_expected, next_stamp(h), none);
  return launch_ex(h, "tma_apply_w_kernel", tma_apply_w_kernel<kApplyLocal>, grid, block, 0, stream, h->nmf_pdl, dim3(1, 1, 1), W, w.Wp, w.plane_w, partial,
                   (numer || w_cluster_reduce(h, p, F, K)) ? 1 : p.w.splits, rowsum, numer ? 1 : p.rowsum_slots, F, K, w.sumsq_part, w.colsum,
                   arrival_counter, arrivals_expected, next_stamp(h), none);
}

// ---- pull exchange (gccnmf_klnmf_step_pull).  Layout of every rank's symmetric buffer, in floats:
//   [numerator F*K + K (packed row sums)] x 2 (iteration parity) | [row-sum slots max_slots*K] x 2 | reduced F*K | 64 floats: arrival
//   counters (u32) 0, 1 | one u32 flag per tile of U.  With the cluster-reduced numerator contraction the contraction writes the numerator and G2's epilogue the
//   row-sum slots directly; otherwise the pack kernel sums the k-split slabs and the slots into [F*K + K].
struct PullLayout { int64_t numer[2], rowsum[2], reduced, counters, flags, total; };
PullLayout pull_layout(int F, int T2, int K) {
  PullLayout l;
  const int64_t fk = (int64_t)F * K, rs = (int64_t)max_rowsum_slots(T2) * K;
  l.numer[0] = 0; l.numer[1] = fk + K;
  l.rowsum[0] = 2 * (fk + K); l.rowsum[1] = l.rowsum[0] + rs;
  l.reduced = l.rowsum[1] + rs;
  l.counters = l.reduced + fk;
  l.flags = l.counters + 64;                // one u32 per 32 x 128 tile of U (exchange inside the W update)
  const int64_t tiles = (int64_t)((F + kApplyTile - 1) / kApplyTile) * ((K + kApplyAtoms - 1) / kApplyAtoms);
  l.total = l.flags + ((tiles + 63) & ~(int64_t)63);
  return l;
}
PeerSet pull_peers(const float* const* bases, int world, const PullLayout& l, int parity, int F, int K, bool packed) {
  PeerSet ps{};
  ps.world = world;
  for (int r = 0; r < world; ++r) {
    ps.numer[r] = bases[r] + l.numer[parity];
    ps.rowsum[r] = packed ? bases[r] + l.numer[parity] + (int64_t)F * K : bases[r] + l.rowsum[parity];
    ps.reduced[r] = bases[r] + l.reduced;
  }
  const int64_t n4 = (int64_t)F * K / 4;
  ps.chunk4 = (n4 + world - 1) / world;
  return ps;
}
tgemm::PeerSignal pull_signal(float* const* bases, int world, const PullLayout& l, int which) {
  tgemm::PeerSignal sg{};
  sg.world = world;
  for (int r = 0; r < world; ++r) sg.counters[r] = reinterpret_cast<unsigned*>(bases[r] + l.counters) + which;
  return sg;
}

int64_t gccnmf_klnmf_tma_pull_floats(int F, int layout_T2, int K) { return pull_layout(F, layout_T2, K).total; }
bool gccnmf_klnmf_tma_pull_supported(gccnmf_handle* h, int F, int T2, int K) { (void)h; return gccnmf_klnmf_tma_supported(F, T2, K); }
// form 2 (exchange inside the W update) spins on flags set by the same-tile CTAs of the other ranks: every CTA of the grid must be
// resident at once
bool gccnmf_klnmf_tma_pull_fused_ok(gccnmf_handle* h, int F, int K) {
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, tma_apply_w_exchange_kernel, 256, 0) != cudaSuccess) { (void)cudaGetLastError(); return false; }
  const int64_t tiles = (int64_t)((F + kApplyTile - 1) / kApplyTile) * ((K + kApplyAtoms - 1) / kApplyAtoms);
  return (int64_t)per_sm * h->sm_count >= tiles;
}
bool gccnmf_klnmf_tma_pull_direct(gccnmf_handle* h, int F, int T2, int K) { return w_cluster_reduce(h, make_plan(h, F, T2, K), F, K) && !h->pull_force_pack; }

// One sharded iteration with the pull exchange; `bases`: host array of `world` device pointers, each rank's symmetric buffer as mapped
// in THIS process (bases[rank] is the local one).
int gccnmf_klnmf_tma_step_pull(gccnmf_handle* h, const float* V, int F, int T2, float* W, float* H, int K, float alpha, float eps, int iteration,
                               int64_t epoch, int rank, int world, float* const* bases, int layout_T2, int two_shot, int want_direct,
                               void* workspace, size_t workspace_bytes, void* stream) {
  TMA_CARVE_OR_FAIL(w);
  const Plan p = make_plan(h, F, T2, K);
  if (world > 8) return gccnmf_fail(h, GCCNMF_ERR_UNSUPPORTED, "klnmf_step_pull: at most 8 ranks");
  // (the layout is the same on every rank: built from the largest shard; a rank with fewer row-sum slots leaves the others zero)
  const PullLayout l = pull_layout(F, layout_T2, K);
  if (layout_T2 < T2) return gccnmf_fail(h, GCCNMF_ERR_INVALID_ARGUMENT, "klnmf_step_pull: layout_T2 %d < T2 %d", layout_T2, T2);
  // epoch: iterations of earlier runs on this buffer (the arrival counters keep counting; buffers alternate by global parity)
  const int parity = (int)((epoch + iteration) & 1);
  const unsigned expected = (unsigned)((uint64_t)world * (uint64_t)(epoch + iteration + 1));
  float* local = bases[rank];
  const unsigned* counters_local = reinterpret_cast<const unsigned*>(local + l.counters);
  const tgemm::PeerSignal sig0 = pull_signal(bases, world, l, 0);
  // direct = the numerator contraction sums its k-splits inside clusters (when every cluster of the launch is resident at once): it
  // writes the numerator, and G2's epilogue the row-sum slots, straight into the symmetric buffer, and its last CTA signals the ranks.
  // Otherwise the pack kernel sums the k-split slabs and the row-sum slots into the buffer and signals.
  if (two_shot == 2) {
    if (!gccnmf_klnmf_tma_pull_fused_ok(h, F, K))
      return gccnmf_fail(h, GCCNMF_ERR_UNSUPPORTED, "klnmf_step_pull: form 2 needs every tile CTA of the W update resident at once");
    // form 2: the exchange happens inside the W update, tile by tile (tma_apply_w_exchange_kernel): G2 writes its row-sum slots into
    // the symmetric buffer, the numerator contraction its k-split slabs (or cluster-reduced single slab) as in the single-GPU loop
    h->xchg_rowsum = local + l.rowsum[parity];
    int e = gccnmf_klnmf_tma_update_H(h, V, F, T2, W, H, K, alpha, eps, workspace, workspace_bytes, iteration > 0 ? 2 : 0, iteration > 0, stream);
    h->xchg_rowsum = nullptr;
    if (!e) e = gccnmf_klnmf_tma_partial_W_to(h, V, F, T2, W, H, K, workspace, workspace_bytes, true, nullptr, stream);
    if (e) return e;
    PeerSet ps{};
    tgemm::PeerSignal flags{};
    ps.world = flags.world = world;
    for (int r = 0; r < world; ++r) {
      ps.numer[r] = bases[r] + l.numer[parity];
      ps.rowsum[r] = bases[r] + l.rowsum[parity];
      flags.counters[r] = reinterpret_cast<unsigned*>(bases[r] + l.flags);
    }
    const dim3 grid((K + kApplyAtoms - 1) / kApplyAtoms, w.row_blocks), block(32, 8);
    return launch_ex(h, "tma_apply_w_exchange_kernel", tma_apply_w_exchange_kernel, grid, block, 0, stream, h->nmf_pdl, dim3(1, 1, 1), W, w.Wp, w.plane_w,
                     (const float*)w.partial, w_cluster_reduce(h, p, F, K) ? 1 : p.w.splits, max_rowsum_slots(layout_T2), F, K, w.sumsq_part, w.colsum,
                     ps, rank, local + l.numer[parity], flags, expected, next_stamp(h));
  }
  // Every rank must take the same branch (the readers' addresses depend on it): the caller passes the agreed choice.
  const bool direct = want_direct != 0;
  if (direct && !(w_cluster_reduce(h, p, F, K) && !h->pull_force_pack))
    return gccnmf_fail(h, GCCNMF_ERR_UNSUPPORTED, "klnmf_step_pull: direct form asked for, but the cluster-reduced contraction is unavailable here");
  const int rs_slots = direct ? max_rowsum_slots(layout_T2) : 1;
  int st = 0;
  if (direct) {
    h->xchg_rowsum = local + l.rowsum[parity];
    h->xchg_numer = local + l.numer[parity];
    h->xchg_world = world;
    for (int r = 0; r < world; ++r) h->xchg_counters[r] = sig0.counters[r];
    h->xchg_done = w.done + 2;
    st = gccnmf_klnmf_tma_update_H(h, V, F, T2, W, H, K, alpha, eps, workspace, workspace_bytes, iteration > 0 ? 2 : 0, iteration > 0, stream);
    if (!st) st = gccnmf_klnmf_tma_partial_W_to(h, V, F, T2, W, H, K, workspace, workspace_bytes, true, h->xchg_numer, stream);
    h->xchg_rowsum = nullptr; h->xchg_numer = nullptr; h->xchg_world = 0; h->xchg_done = nullptr;
    if (st) return st;
  } else {
    st = gccnmf_klnmf_tma_update_H(h, V, F, T2, W, H, K, alpha, eps, workspace, workspace_bytes, iteration > 0 ? 2 : 0, iteration > 0, stream);
    if (!st) st = gccnmf_klnmf_tma_partial_W_to(h, V, F, T2, W, H, K, workspace, workspace_bytes, true, nullptr, stream);
    if (st) return st;
    const int64_t n = (int64_t)F * K;
    const bool summed = w_cluster_reduce(h, p, F, K);       // (pull_force_pack: the contraction left one slab, not p.w.splits)
    if (int e = launch_ex(h, "tma_pack_numer_kernel", tma_pack_numer_kernel, dim3((unsigned)std::min<int64_t>(((n + K) / 4 + 255) / 256, 2 * h->sm_count)), dim3(256), 0, stream, h->nmf_pdl,
                          dim3(1, 1, 1), (const float*)w.partial, summed ? 1 : p.w.splits, n, (const float*)w.rowsum_part, p.rowsum_slots, K,
                          local + l.numer[parity], w.done, (unsigned*)nullptr, 0, next_stamp(h), sig0)) return e;
  }
  const PeerSet peers = pull_peers(bases, world, l, parity, F, K, !direct);
  const int64_t n4 = (int64_t)F * K / 4;
  (void)n4;
  if (two_shot) {
    const unsigned ctas = (unsigned)std::max<int64_t>(1, std::min<int64_t>(h->sm_count, (peers.chunk4 + 255) / 256));
    if (int e = launch_ex(h, "tma_reduce_pull_kernel", tma_reduce_pull_kernel, dim3(ctas), dim3(256), 0, stream, h->nmf_pdl, dim3(1, 1, 1), peers,
                          local + l.reduced, n4, rank, counters_local, expected, w.done + 1, pull_signal(bases, world, l, 1), next_stamp(h))) return e;
  }
  const dim3 grid((K + kApplyAtoms - 1) / kApplyAtoms, w.row_blocks), block(32, 8);
  if (two_shot)
    return launch_ex(h, "tma_apply_w_kernel", tma_apply_w_kernel<kApplyPullOwner>, grid, block, 0, stream, h->nmf_pdl, dim3(1, 1, 1), W, w.Wp, w.plane_w,
                     (const float*)nullptr, 1, (const float*)nullptr, rs_slots, F, K, w.sumsq_part, w.colsum, counters_local + 1, expected,
                     next_stamp(h), peers);
  return launch_ex(h, "tma_apply_w_kernel", tma_apply_w_kernel<kApplyPull>, grid, block, 0, stream, h->nmf_pdl, dim3(1, 1, 1), W, w.Wp, w.plane_w,
                   (const float*)nullptr, world, (const float*)nullptr, rs_slots, F, K, w.sumsq_part, w.colsum, counters_local, expected,
                   next_stamp(h), peers);
}

int gccnmf_klnmf_tma_reduce_bcast(gccnmf_handle* h, int F, int T2, int K, const float* numer_multicast, float* reduced_multicast, int rank, int world,
                                  const unsigned* arrivals_in, unsigned arrivals_expected, unsigned* arrivals_out_mc, void* workspace,
                                  size_t workspace_bytes, void* stream) {
  TMA_CARVE_OR_FAIL(w);
  const int64_t n4 = ((int64_t)F * K + K) / 4;                       // K % 8 == 0 on this path
  const int64_t chunk = (n4 + world - 1) / world;
  const unsigned ctas = (unsigned)std::max<int64_t>(1, std::min<int64_t>(h->sm_count, (chunk + 255) / 256));
  return launch_ex(h, "tma_reduce_bcast_kernel", tma_reduce_bcast_kernel, dim3(ctas), dim3(256), 0, stream, h->nmf_pdl, dim3(1, 1, 1), numer_multicast,
                   reduced_multicast, n4, rank, world, arrivals_in, arrivals_expected, w.done + 1, arrivals_out_mc, next_stamp(h));
}

int gccnmf_klnmf_tma_apply_W(gccnmf_handle* h, int F, int T2, float* W, int K, const float* numer, bool numer_is_multicast,
                             void* workspace, size_t workspace_bytes, void* stream) {
  return gccnmf_klnmf_tma_apply_W_mc(h, F, T2, W, K, numer, numer_is_multicast, nullptr, 0u, workspace, workspace_bytes, stream);
}

// Writes the caller's H from G^T (H = c G, :81) and normalises the caller's W in place (W = U / c, :80) when W was updated.
int gccnmf_klnmf_tma_finish(gccnmf_handle* h, int F, int T2, float* H, int K, bool pending_norms, void* workspace,
                            size_t workspace_bytes, void* stream) {
  TMA_CARVE_OR_FAIL(w);
  GCCNMF_LAUNCH(h, tma_finish_h_kernel, dim3((K + 31) / 32, (T2 + 31) / 32), dim3(32, 8), 0, stream, w.HT, T2, K,
                pending_norms ? w.sumsq_part : (const float*)nullptr, w.row_blocks, H);
  return 0;
}
int gccnmf_klnmf_tma_finish_W(gccnmf_handle* h, int F, int T2, float* W, int K, void* workspace, size_t workspace_bytes, void* stream) {
  TMA_CARVE_OR_FAIL(w);
  GCCNMF_LAUNCH(h, tma_finish_w_kernel, dim3((K + 127) / 128, std::min(F, 64)), 128, 0, stream, W, F, K, w.sumsq_part, w.row_blocks);
  return 0;
}

// Option l2_persist: while the loop runs, every launch through launch_ex carries an access-policy window (persisting) over the
// float32 master of G^T (1) or the master and its planes (2) -- the H update re-reads and rewrites the master every iteration and
// the ncu capture shows those 30 MB going to DRAM and back although the working set of an iteration is ~65 MB.  enable = false
// clears the window (the persisting lines decay as other data replaces them).
int gccnmf_klnmf_tma_l2_window(gccnmf_handle* h, int F, int T2, int K, bool enable, void* workspace, size_t workspace_bytes) {
  h->l2_window_base = nullptr;
  h->l2_window_bytes = 0;
  if (!enable || h->l2_persist <= 0) return 0;
  TMA_CARVE_OR_FAIL(w);
  int dev = 0, max_window = 0, max_persist = 0;
  GCCNMF_CHECK_CUDA(h, cudaGetDevice(&dev));
  GCCNMF_CHECK_CUDA(h, cudaDeviceGetAttribute(&max_window, cudaDevAttrMaxAccessPolicyWindowSize, dev));
  GCCNMF_CHECK_CUDA(h, cudaDeviceGetAttribute(&max_persist, cudaDevAttrMaxPersistingL2CacheSize, dev));
  size_t bytes = (size_t)T2 * K * 4;
  if (h->l2_persist >= 2) bytes = (size_t)((const char*)(w.HTp + 2 * w.plane_ht) - (const char*)w.HT);
  bytes = std::min(bytes, std::min((size_t)max_window, (size_t)max_persist));
  if (bytes == 0) return 0;
  if (!h->l2_limit_set) {
    GCCNMF_CHECK_CUDA(h, cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, std::min((size_t)max_persist, (size_t)48 << 20)));
    h->l2_limit_set = true;
  }
  h->l2_window_base = w.HT;
  h->l2_window_bytes = bytes;
  return 0;
}

// ---- batched runs (gccnmf_klnmf_batched): B clips of one shape.  Clip b's workspace is the single-clip carve at
// workspace + b * clip_bytes; every launch of an iteration covers all clips (clip from the grid), and each clip runs the tile plan
// of a solo run on its shape, so its W and H carry the bits of gccnmf_klnmf on it alone.  The W-update numerator is always
// written as k-split slabs and summed by the W update in split order, the sum the cluster-reduced form makes in the same order:
// the cluster form needs all of a launch's clusters resident, which B clips can break.

// The options the batch form leaves out (the L2 access-policy window, the split W.H contractions): the caller runs such a clip set
// one clip at a time by the solo path.
bool gccnmf_klnmf_tma_batch_supported(gccnmf_handle* h, int F, int T2, int K) { return h->l2_persist <= 0 && !wh_split2(h, F, T2, K); }

int gccnmf_klnmf_tma_batched(gccnmf_handle* h, const float* V, int64_t ld_v, int64_t clip_stride_v, int B, int F, int T2, float* W, float* H, int K,
                             int iterations, float alpha, float eps, bool update_W, void* workspace, size_t clip_bytes, void* stream) {
  const TmaWorkspace w = tma_carve(workspace, clip_bytes, F, T2, K);      // clip 0; clip b is the same carve b * clip_bytes on
  if (!w.ok) return gccnmf_fail(h, GCCNMF_ERR_WORKSPACE, "klnmf_batched: %zu bytes per clip, need %zu", clip_bytes, tma_workspace_bytes(F, T2, K));
  const int64_t cb = (int64_t)clip_bytes;
  const Plan p = make_plan(h, F, T2, K);
  const dim3 block(32, 8);
  GCCNMF_LAUNCH(h, tma_transpose_split_clips_kernel, dim3((T2 + 31) / 32, (int)((w.Fp + 31) / 32), B), block, 0, stream, V, F, T2, ld_v, clip_stride_v,
                w.VT, w.Fp, (bf16*)nullptr, (int64_t)0, (int64_t)0, cb);
  const int64_t fk = (int64_t)F * K;
  GCCNMF_LAUNCH(h, tma_split_clips_kernel, dim3((unsigned)((fk + 255) / 256), B), 256, 0, stream, (const float*)W, fk, w.Wp, w.plane_w, cb);
  GCCNMF_LAUNCH(h, tma_transpose_split_clips_kernel, dim3((T2 + 31) / 32, (K + 31) / 32, B), block, 0, stream, (const float*)H, K, T2, (int64_t)T2,
                (int64_t)K * T2, w.HT, (int64_t)K, w.HTp, (int64_t)K, w.plane_ht, cb);
  const Operand Wk{w.Wp, (int64_t)K, w.plane_w, false}, Wmn{w.Wp, (int64_t)K, w.plane_w, true};
  const Operand HTk{w.HTp, (int64_t)K, w.plane_ht, false}, HTmn{w.HTp, (int64_t)K, w.plane_ht, true};
  const Operand RTk{w.RTp, w.Fp, w.plane_rt, false}, RTmn{w.RTp, w.Fp, w.plane_rt, true};
  const tgemm::Clips<EpiRatioPlanes> ratio{EpiRatioPlanes{w.VT, w.RTp, w.Fp, w.plane_rt, F, T2, true}, cb, 1};
  const tgemm::Clips<EpiStoreT> numer{EpiStoreT{w.partial, (int64_t)K, fk, K, F, true, h->gemm_streaming != 0}, cb, p.w.splits};
  for (int it = 0; it < iterations; ++it) {
    // (gccnmf_klnmf's loop: colsum(U) computed at the first iteration, then left by the W update, or kept with a fixed dictionary)
    const int colsum_state = it == 0 ? 0 : (update_W ? 2 : 1);
    if (int st = plane_gemm_clips<false, false>(h, p.bn_wh, Wk, HTk, F, T2, K, 1, true, ratio, B, stream)) return st;        // G1
    if (colsum_state == 0) GCCNMF_LAUNCH(h, tma_colsum_clips_kernel, dim3((K + 127) / 128, B), 128, 0, stream, (const float*)W, F, K, w.colsum, cb);
    const tgemm::Clips<EpiUpdateH> upd{EpiUpdateH{w.HT, w.HTp, w.colsum, colsum_state == 2 ? w.sumsq_part : nullptr, w.rowsum_part, alpha, eps,
                                                  (int64_t)K, w.plane_ht, K, T2, colsum_state == 2 ? w.row_blocks : 1, true}, cb, 1};
    if (int st = plane_gemm_clips<true, false>(h, p.bn_h, Wmn, RTk, K, T2, F, 1, false, upd, B, stream)) return st;          // G2
    if (!update_W) continue;
    if (int st = plane_gemm_clips<false, false>(h, p.bn_wh, Wk, HTk, F, T2, K, 1, true, ratio, B, stream)) return st;        // G3
    if (int st = plane_gemm_clips<true, true>(h, p.w.bn, HTmn, RTmn, K, F, T2, p.w.splits, false, numer, B, stream)) return st;  // G4
    if (int st = launch_ex(h, "tma_apply_w_clips_kernel", tma_apply_w_clips_kernel, dim3((K + kApplyAtoms - 1) / kApplyAtoms, w.row_blocks, B), block,
                           0, stream, h->nmf_pdl, dim3(1, 1, 1), W, w.Wp, w.plane_w, (const float*)w.partial, p.w.splits, (const float*)w.rowsum_part,
                           p.rowsum_slots, F, K, w.sumsq_part, w.colsum, cb)) return st;
  }
  GCCNMF_LAUNCH(h, tma_finish_h_clips_kernel, dim3((K + 31) / 32, (T2 + 31) / 32, B), block, 0, stream, (const float*)w.HT, T2, K,
                update_W ? (const float*)w.sumsq_part : (const float*)nullptr, w.row_blocks, H, cb);
  if (update_W)
    GCCNMF_LAUNCH(h, tma_finish_w_clips_kernel, dim3((K + 127) / 128, std::min(F, 64), B), 128, 0, stream, W, F, K, (const float*)w.sumsq_part, w.row_blocks, cb);
  return 0;
}

// ---- ragged runs (gccnmf_klnmf_ragged): n clips of different lengths T2[i], each on its own workspace carve ws[i] and its solo plan.
// Each plane-GEMM contraction is launched once per distinct tile width among the clips' plans (tgemm::Ragged: a flat grid of the
// clips' own tiles), every small kernel once for all clips; so each clip computes what gccnmf_klnmf computes on it alone.  The W-update
// numerator is written as k-split slabs, as in batched runs.  The per-call table (the clips' tensor maps, RaggedClip records and
// the launches' RaggedTile lists) is built on the host and copied into `table` (kRaggedTablePerClip bytes per clip, 128-byte
// aligned) by one stream-ordered copy before the first launch.
constexpr size_t kRaggedTablePerClip = 1280;
constexpr int kRaggedMaps = 6;              // per clip: A and B of G1 / G3, of G2 and of G4
static_assert(kRaggedMaps * sizeof(CUtensorMap) + sizeof(RaggedClip) + 3 * sizeof(tgemm::RaggedTile) + 3 * 16 <= kRaggedTablePerClip,
              "ragged table entry");
size_t gccnmf_klnmf_tma_ragged_table_per_clip() { return kRaggedTablePerClip; }

int gccnmf_klnmf_tma_ragged(gccnmf_handle* h, int n, const float* const* V, const int64_t* ld_v, const int* T2, float* const* W, float* const* H,
                            void* const* ws, int F, int K, int iterations, float alpha, float eps, bool update_W, void* table, void* stream) {
  enum { kWH, kH, kW, kContractions };
  std::vector<RaggedClip> clips(n);
  std::vector<CUtensorMap> maps((size_t)n * kRaggedMaps);
  std::vector<tgemm::RaggedTile> tiles[kContractions];
  std::vector<int> width[kContractions];
  const int64_t Fp = (F + 7) & ~7, fk = (int64_t)F * K;
  const int row_blocks = (F + kApplyTile - 1) / kApplyTile;
  int max_T2 = 0;
  unsigned char* dev = static_cast<unsigned char*>(table);
  const CUtensorMap* maps_d = reinterpret_cast<const CUtensorMap*>(dev);
  const size_t clips_off = (size_t)n * kRaggedMaps * sizeof(CUtensorMap);
  const size_t tiles_off = align_up(clips_off + (size_t)n * sizeof(RaggedClip), 16);
  std::vector<Plan> plans(n);
  for (int i = 0; i < n; ++i) {
    const TmaWorkspace w = tma_carve(ws[i], tma_workspace_bytes(F, T2[i], K), F, T2[i], K);
    const Plan p = plans[i] = make_plan(h, F, T2[i], K);
    clips[i] = RaggedClip{V[i], ld_v[i], W[i], H[i], w.HT, w.VT, w.partial, w.colsum, w.sumsq_part, w.rowsum_part, w.HTp, w.Wp, w.RTp,
                          w.plane_ht, w.plane_rt, T2[i], p.w.splits, p.rowsum_slots};
    max_T2 = std::max(max_T2, T2[i]);
    const Operand Wk{w.Wp, (int64_t)K, w.plane_w, false}, Wmn{w.Wp, (int64_t)K, w.plane_w, true};
    const Operand HTk{w.HTp, (int64_t)K, w.plane_ht, false}, HTmn{w.HTp, (int64_t)K, w.plane_ht, true};
    const Operand RTk{w.RTp, w.Fp, w.plane_rt, false}, RTmn{w.RTp, w.Fp, w.plane_rt, true};
    CUtensorMap* m = &maps[(size_t)i * kRaggedMaps];
    if (int st = ragged_maps<false, false>(h, Wk, HTk, F, T2[i], K, p.bn_wh, m)) return st;
    if (int st = ragged_maps<true, false>(h, Wmn, RTk, K, T2[i], F, p.bn_h, m + 2)) return st;
    if (int st = ragged_maps<true, true>(h, HTmn, RTmn, K, F, T2[i], p.w.bn, m + 4)) return st;
    const int kb_k = (K + kKB - 1) / kKB, kb_f = (F + kKB - 1) / kKB, kb_t = (T2[i] + kKB - 1) / kKB;
    const tgemm::RaggedTile t[kContractions] = {
        {0, i, T2[i], K, (T2[i] + p.bn_wh - 1) / p.bn_wh, kb_k, maps_d + i * kRaggedMaps, maps_d + i * kRaggedMaps + 1, w.Wp, w.HTp, w.plane_w, w.plane_ht},
        {0, i, T2[i], F, (T2[i] + p.bn_h - 1) / p.bn_h, kb_f, maps_d + i * kRaggedMaps + 2, maps_d + i * kRaggedMaps + 3, nullptr, nullptr, 0, 0},
        {0, i, F, T2[i], (F + p.w.bn - 1) / p.w.bn, (kb_t + p.w.splits - 1) / p.w.splits, maps_d + i * kRaggedMaps + 4, maps_d + i * kRaggedMaps + 5,
         nullptr, nullptr, 0, 0}};
    const int widths[kContractions] = {p.bn_wh, p.bn_h, p.w.bn};
    for (int c = 0; c < kContractions; ++c) { tiles[c].push_back(t[c]); width[c].push_back(widths[c]); }
  }
  // Each contraction's clips ordered by tile width (stable): one launch per run of equal widths, CTAs numbered along the run.
  struct Launch { int bn, begin, count, ctas; };
  std::vector<Launch> launches[kContractions];
  std::vector<unsigned char> host(tiles_off + (size_t)kContractions * n * sizeof(tgemm::RaggedTile));
  for (int c = 0; c < kContractions; ++c) {
    std::vector<int> order(n);
    for (int i = 0; i < n; ++i) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return width[c][a] < width[c][b]; });
    const int M = c == kWH ? F : K;
    tgemm::RaggedTile* out = reinterpret_cast<tgemm::RaggedTile*>(host.data() + tiles_off) + (size_t)c * n;
    for (int j = 0; j < n; ++j) {
      const int i = order[j], bn = width[c][i];
      if (launches[c].empty() || launches[c].back().bn != bn) launches[c].push_back(Launch{bn, j, 0, 0});
      Launch& l = launches[c].back();
      tgemm::RaggedTile t = tiles[c][i];
      t.cta_begin = l.ctas;
      l.ctas += t.n_tiles * m_tiles_of(M, c == kWH, bn) * (c == kW ? plans[i].w.splits : 1);
      l.count++;
      std::memcpy(out + j, &t, sizeof(t));
    }
  }
  std::memcpy(host.data(), maps.data(), maps.size() * sizeof(CUtensorMap));
  std::memcpy(host.data() + clips_off, clips.data(), clips.size() * sizeof(RaggedClip));
  GCCNMF_CHECK_CUDA(h, cudaMemcpyAsync(table, host.data(), host.size(), cudaMemcpyHostToDevice, (cudaStream_t)stream));
  const RaggedClip* clips_d = reinterpret_cast<const RaggedClip*>(dev + clips_off);
  const tgemm::RaggedTile* tiles_d = reinterpret_cast<const tgemm::RaggedTile*>(dev + tiles_off);

  const dim3 block(32, 8);
  GCCNMF_LAUNCH(h, tma_prepare_v_ragged_kernel, dim3((max_T2 + 31) / 32, (unsigned)((Fp + 31) / 32), n), block, 0, stream, clips_d, F, Fp);
  GCCNMF_LAUNCH(h, tma_split_ragged_kernel, dim3((unsigned)((fk + 255) / 256), n), 256, 0, stream, clips_d, fk);
  GCCNMF_LAUNCH(h, tma_prepare_h_ragged_kernel, dim3((max_T2 + 31) / 32, (K + 31) / 32, n), block, 0, stream, clips_d, K);
  auto contraction = [&](int c, auto epi, auto launch) -> int {
    for (const Launch& l : launches[c]) {
      epi.tiles = tiles_d + (size_t)c * n + l.begin;
      epi.count = l.count;
      if (int st = launch(l.bn, l.ctas, epi)) return st;
    }
    return 0;
  };
  const tgemm::Ragged<EpiRatioPlanes> ratio{EpiRatioPlanes{nullptr, nullptr, Fp, 0, F, 0, true}, nullptr, 0, clips_d};
  const tgemm::Ragged<EpiStoreT> numer{EpiStoreT{nullptr, (int64_t)K, fk, K, F, true, h->gemm_streaming != 0}, nullptr, 0, clips_d};
  auto wh = [&](int bn, int ctas, const tgemm::Ragged<EpiRatioPlanes>& e) { return plane_gemm_ragged<false, false>(h, bn, F, ctas, true, K, K, e, stream); };
  auto upd_h = [&](int bn, int ctas, const tgemm::Ragged<EpiUpdateH>& e) { return plane_gemm_ragged<true, false>(h, bn, K, ctas, false, 0, 0, e, stream); };
  auto num_w = [&](int bn, int ctas, const tgemm::Ragged<EpiStoreT>& e) { return plane_gemm_ragged<true, true>(h, bn, K, ctas, false, 0, 0, e, stream); };
  for (int it = 0; it < iterations; ++it) {
    const int colsum_state = it == 0 ? 0 : (update_W ? 2 : 1);     // (as in gccnmf_klnmf_tma_batched)
    if (int st = contraction(kWH, ratio, wh)) return st;                                                               // G1
    if (colsum_state == 0) GCCNMF_LAUNCH(h, tma_colsum_ragged_kernel, dim3((K + 127) / 128, n), 128, 0, stream, clips_d, F, K);
    const tgemm::Ragged<EpiUpdateH> upd{EpiUpdateH{nullptr, nullptr, nullptr, colsum_state == 2 ? clips[0].sumsq_part : nullptr, nullptr, alpha, eps,
                                                   (int64_t)K, 0, K, 0, colsum_state == 2 ? row_blocks : 1, true}, nullptr, 0, clips_d};
    if (int st = contraction(kH, upd, upd_h)) return st;                                                               // G2
    if (!update_W) continue;
    if (int st = contraction(kWH, ratio, wh)) return st;                                                               // G3
    if (int st = contraction(kW, numer, num_w)) return st;                                                             // G4
    if (int st = launch_ex(h, "tma_apply_w_ragged_kernel", tma_apply_w_ragged_kernel, dim3((K + kApplyAtoms - 1) / kApplyAtoms, row_blocks, n), block, 0,
                           stream, h->nmf_pdl, dim3(1, 1, 1), clips_d, F, K)) return st;
  }
  GCCNMF_LAUNCH(h, tma_finish_h_ragged_kernel, dim3((K + 31) / 32, (max_T2 + 31) / 32, n), block, 0, stream, clips_d, K, row_blocks, update_W ? 1 : 0);
  if (update_W) GCCNMF_LAUNCH(h, tma_finish_w_ragged_kernel, dim3((K + 127) / 128, std::min(F, 64), n), 128, 0, stream, clips_d, F, K, row_blocks);
  return 0;
}

int gccnmf_klnmf_tma_pack_numer_mc(gccnmf_handle* h, int F, int T2, int K, float* numer, unsigned* mc_counter, void* workspace, size_t workspace_bytes,
                                   void* stream) {
  TMA_CARVE_OR_FAIL(w);
  const Plan p = make_plan(h, F, T2, K);
  const int64_t n = (int64_t)F * K;
  // (pairs with gccnmf_klnmf_tma_partial_W_to(..., numer): with cluster-reduced k-splits the numerator is already in `numer`)
  const bool in_place = w_cluster_reduce(h, p, F, K);
  const int64_t items = ((in_place ? 0 : n) + K) / 4;
  return launch_ex(h, "tma_pack_numer_kernel", tma_pack_numer_kernel, dim3((unsigned)std::min<int64_t>((items + 255) / 256, 2 * h->sm_count)), dim3(256), 0, stream,
                   h->nmf_pdl, dim3(1, 1, 1), in_place ? (const float*)nullptr : (const float*)w.partial, p.w.splits, n, (const float*)w.rowsum_part,
                   p.rowsum_slots, K, numer, w.done, mc_counter, h->mc_light_signal, next_stamp(h), tgemm::PeerSignal{});
}
int gccnmf_klnmf_tma_pack_numer(gccnmf_handle* h, int F, int T2, int K, float* numer, void* workspace, size_t workspace_bytes, void* stream) {
  return gccnmf_klnmf_tma_pack_numer_mc(h, F, T2, K, numer, nullptr, workspace, workspace_bytes, stream);
}

extern "C" {

// The tile plan of the TMA KL-NMF path for a device with `sm_count` SMs (pure host logic, no device needed):
// out[0] tile width of the W.H contractions, out[1] of the H update, out[2] / out[3] tile width / k-splits of the W-update
// numerator, out[4] row-sum slots (n tiles of the H update), out[5..7] CTAs of G1/G3, G2, G4.  Returns 0, or < 0 when the
// shape is not covered by the TMA path.
int gccnmf_klnmf_tile_plan(int sm_count, int F, int T2, int K, int* out) {
  if (!out || sm_count <= 0 || F <= 0 || T2 <= 0 || K <= 0) return GCCNMF_ERR_INVALID_ARGUMENT;
  if (!gccnmf_klnmf_tma_supported(F, T2, K)) return GCCNMF_ERR_UNSUPPORTED;
  gccnmf_handle h;
  h.sm_count = sm_count;
  const Plan p = make_plan(&h, F, T2, K);
  out[0] = p.bn_wh; out[1] = p.bn_h; out[2] = p.w.bn; out[3] = p.w.splits; out[4] = p.rowsum_slots;
  out[5] = m_tiles_of(F, true, p.bn_wh) * ((T2 + p.bn_wh - 1) / p.bn_wh);
  out[6] = m_tiles_of(K, false, p.bn_h) * ((T2 + p.bn_h - 1) / p.bn_h);
  out[7] = m_tiles_of(K, false, p.w.bn) * ((F + p.w.bn - 1) / p.w.bn) * p.w.splits;
  return GCCNMF_OK;
}

// Diagnostics: while `stamps` is non-NULL every plane GEMM launched through this handle appends 8 uint64 per CTA
// (see tma_gemm.cuh) at a running offset; returns the offset (in uint64) reached so far and resets it when asked.
int64_t gccnmf_debug_timing(gccnmf_handle* h, unsigned long long* stamps, int reset) {
  if (!h) return -1;
  const int64_t reached = (int64_t)h->debug_timing_cursor;
  h->debug_timing = stamps;
  if (reset) h->debug_timing_cursor = 0;
  return reached;
}

size_t gccnmf_gemm_planes_workspace_bytes(int M, int N, int Kc) {
  auto pad8 = [](size_t x) { return (x + 7) & ~(size_t)7; };
  const size_t a = std::max((size_t)M * pad8(Kc), (size_t)Kc * pad8(M)), b = std::max((size_t)N * pad8(Kc), (size_t)Kc * pad8(N));
  return align_up(2 * a * 2, 256) + align_up(2 * b * 2, 256) + 512;
}

// Test / diagnostics entry of the TMA plane GEMM: DT (N, M) row-major = (A . B^T)^T.
//   a_mn_major = 0: A is (M, Kc) row-major;  1: A is (Kc, M) row-major (m contiguous).  Same for B with N.
// The float32 operands are split into bf16 hi/lo planes in the workspace first.  tile_n: see plane_gemm (tma_gemm_host.cuh);
// splits > 1 writes `splits` partial slabs DT[z] (N * M floats each).  timing: 6 clock64 stamps per CTA, or NULL.
int gccnmf_gemm_planes(gccnmf_handle* h, const float* A, int a_mn_major, const float* B, int b_mn_major, float* DT, int M, int N, int Kc,
                       int tile_n, int splits, void* workspace, size_t workspace_bytes, unsigned long long* timing, void* stream) {
  GCCNMF_ENTER(h);
  GCCNMF_REQUIRE(h, A && B && DT && M > 0 && N > 0 && Kc > 0 && splits >= 1 && splits <= kMaxSplits, "gemm_planes: bad arguments");
  if (!workspace || workspace_bytes < gccnmf_gemm_planes_workspace_bytes(M, N, Kc))
    return gccnmf_fail(h, GCCNMF_ERR_WORKSPACE, "gemm_planes workspace too small: need %zu bytes", gccnmf_gemm_planes_workspace_bytes(M, N, Kc));
  WorkspaceCarver c(workspace, workspace_bytes);
  // planes keep the operand's own orientation: rows x pitch with pitch = inner extent rounded up to 8
  const int a_rows = a_mn_major ? Kc : M, a_inner = a_mn_major ? M : Kc;
  const int b_rows = b_mn_major ? Kc : N, b_inner = b_mn_major ? N : Kc;
  const int64_t a_pitch = (a_inner + 7) & ~7, b_pitch = (b_inner + 7) & ~7;
  bf16* Ap = c.take<bf16>((size_t)2 * a_rows * a_pitch);
  bf16* Bp = c.take<bf16>((size_t)2 * b_rows * b_pitch);
  if (!c.ok()) return gccnmf_fail(h, GCCNMF_ERR_WORKSPACE, "gemm_planes workspace too small");
  GCCNMF_CHECK_CUDA(h, cudaMemsetAsync(Ap, 0, (size_t)2 * a_rows * a_pitch * 2, (cudaStream_t)stream));
  GCCNMF_CHECK_CUDA(h, cudaMemsetAsync(Bp, 0, (size_t)2 * b_rows * b_pitch * 2, (cudaStream_t)stream));
  const int64_t na = (int64_t)a_rows * a_inner, nb = (int64_t)b_rows * b_inner;
  GCCNMF_LAUNCH(h, tma_split_rows_kernel, (unsigned)((na + 255) / 256), 256, 0, stream, A, a_rows, a_inner, Ap, a_pitch, (int64_t)a_rows * a_pitch);
  GCCNMF_LAUNCH(h, tma_split_rows_kernel, (unsigned)((nb + 255) / 256), 256, 0, stream, B, b_rows, b_inner, Bp, b_pitch, (int64_t)b_rows * b_pitch);
  const Operand Ao{Ap, a_pitch, (int64_t)a_rows * a_pitch, a_mn_major != 0};
  const Operand Bo{Bp, b_pitch, (int64_t)b_rows * b_pitch, b_mn_major != 0};
  EpiStoreT e{DT, (int64_t)M, (int64_t)N * M, M, N, M % 4 == 0 && (reinterpret_cast<uintptr_t>(DT) & 15) == 0, false};
  if (!a_mn_major && !b_mn_major) return plane_gemm<false, false>(h, tile_n, Ao, Bo, M, N, Kc, splits, true, e, timing, stream);
  if (a_mn_major && !b_mn_major) return plane_gemm<true, false>(h, tile_n, Ao, Bo, M, N, Kc, splits, false, e, timing, stream);
  if (a_mn_major && b_mn_major) return plane_gemm<true, true>(h, tile_n, Ao, Bo, M, N, Kc, splits, false, e, timing, stream);
  return gccnmf_fail(h, GCCNMF_ERR_UNSUPPORTED, "gemm_planes: A K-major with B MN-major is not instantiated");
}

}  // extern "C"
