// Shared host-side plumbing for the gccnmf_b200 C ABI: handle, error capture, launch counting.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>

#include "../../include/gccnmf_b200.h"

struct gccnmf_handle {
  int device = 0;
  int sm_count = 132;
  int64_t launches = 0;
  bool force_simt_nmf = false;   // GCCNMF_NMF_PATH=simt: float32 SIMT contractions instead of the wgmma plane GEMM
  bool nmf_pdl = true;           // programmatic dependent launch between the kernels of a KL-NMF iteration
  int wh_tile = 0;               // diagnostics: tile width of the W.H contractions (0 = planned)
  bool argmax_refine_shared = true;   // exact float64 refinement of near-tie argmax decisions: E staged in shared memory (0 = one warp per pair from L2)
  int gemm_streaming = 0;        // st.global.cs for the k-split partials of the W-update numerator (diagnostics)
  bool argmax_persistent = true; // all-TDOA argmax GEMM as one persistent CTA per SM, epilogue straight from the accumulator registers (0: one CTA per tile)
  int gemm_preload = 1;          // plane GEMM epilogues that fetch their global operands during the main loop: bit 0 ratio (W.H), bit 1 H update
  int gemm_pair = -1;            // plane GEMM on CTA pairs (two m tiles share the B tile in a 1 x 2 cluster): -1 where the call site prefers it, 0 never, 1 wherever possible
  int wh_split2 = 0;             // W.H contractions as plain 128 x 208 tiles split in two k-halves summed inside (1, 1, 2) clusters (0: dual-N 104-column tiles)
  bool w_cluster_reduce = true;  // W-update numerator: k-splits summed inside (1, 1, splits) clusters through distributed shared memory (0: k-split slabs)
  // set by gccnmf_klnmf_tma_step_pull around the contractions of a sharded iteration (pull exchange): where the row sums of G and the
  // W-update numerator go (this rank's symmetric buffer) and whom the numerator contraction signals when its last CTA is done
  float* xchg_rowsum = nullptr;
  float* xchg_numer = nullptr;
  unsigned* xchg_done = nullptr;
  unsigned* xchg_counters[8] = {nullptr};
  int xchg_world = 0;
  int pull_force_pack = 0;       // pull exchange: always go through the pack kernel (diagnostics)
  int mc_light_signal = 1;       // sharded runs: arrival signal of the numerator pack as device-scope fence + relaxed multimem.red (0: MEMBAR.SYS + release)
  int l2_persist = 0;            // KL-NMF loop: launch-attribute L2 access-policy window (persisting) over G^T: 1 = float32 master, 2 = master + planes
  const void* l2_window_base = nullptr;   // set by the KL-NMF loop while it runs
  size_t l2_window_bytes = 0;
  bool l2_limit_set = false;
  int gemm_cluster = -1;         // diagnostics: force the plane GEMM cluster shape 10 CN + CM (11 = no cluster); -1 = automatic
  unsigned long long* debug_timing = nullptr;   // diagnostics (gccnmf_debug_timing): CTA stamps of every plane GEMM
  size_t debug_timing_cursor = 0;
  struct gccnmf_tmap_cache* tmaps = nullptr;   // TMA tensor maps, keyed by (buffer, shape, box)
  std::string last_error;
  // twiddle tables e^{-2 pi i j / n}, j < n/2, float64 and float32, cached per FFT size
  static constexpr int kMaxPlans = 8;
  int plan_n[kMaxPlans] = {0};
  double* plan_tw64[kMaxPlans] = {nullptr};
  float* plan_tw32[kMaxPlans] = {nullptr};
};

inline int gccnmf_fail(gccnmf_handle* h, int status, const char* fmt, ...) __attribute__((format(printf, 3, 4)));
#include <cstdarg>
inline int gccnmf_fail(gccnmf_handle* h, int status, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  if (h) h->last_error = buf;
  return status;
}

#define GCCNMF_CHECK_CUDA(h, expr)                                                              \
  do {                                                                                          \
    cudaError_t err__ = (expr);                                                                 \
    if (err__ != cudaSuccess)                                                                   \
      return gccnmf_fail((h), GCCNMF_ERR_CUDA, "%s failed: %s (%s:%d)", #expr,                  \
                         cudaGetErrorString(err__), __FILE__, __LINE__);                        \
  } while (0)

// Every kernel launch goes through this so that launch errors are captured and counted.
#define GCCNMF_LAUNCH(h, kernel, grid, block, smem, stream, ...)                                \
  do {                                                                                          \
    kernel<<<(grid), (block), (smem), (cudaStream_t)(stream)>>>(__VA_ARGS__);                   \
    cudaError_t err__ = cudaGetLastError();                                                     \
    if (err__ != cudaSuccess)                                                                   \
      return gccnmf_fail((h), GCCNMF_ERR_CUDA, "launch of %s failed: %s (%s:%d)", #kernel,      \
                         cudaGetErrorString(err__), __FILE__, __LINE__);                        \
    (h)->launches++;                                                                            \
  } while (0)

#define GCCNMF_REQUIRE(h, cond, ...)                                                            \
  do {                                                                                          \
    if (!(cond)) return gccnmf_fail((h), GCCNMF_ERR_INVALID_ARGUMENT, __VA_ARGS__);             \
  } while (0)

// Every ABI entry that takes a handle starts here: NULL check + make the handle's device current (a process may hold
// handles on several devices; kernel attributes and occupancy caches below are kept per device index).
constexpr int kGccnmfMaxDevices = 64;
inline int gccnmf_enter(gccnmf_handle* h) {
  if (!h) return GCCNMF_ERR_INVALID_ARGUMENT;
  const cudaError_t err = cudaSetDevice(h->device);
  if (err != cudaSuccess) return gccnmf_fail(h, GCCNMF_ERR_CUDA, "cudaSetDevice(%d) failed: %s", h->device, cudaGetErrorString(err));
  return GCCNMF_OK;
}
#define GCCNMF_ENTER(h)                                                                         \
  do {                                                                                          \
    if (int st__ = gccnmf_enter(h)) return st__;                                                \
  } while (0)
// Per-device once-flag for cudaFuncSetAttribute and friends (function-local `static DeviceFlags configured;`).
struct DeviceFlags {
  bool done[kGccnmfMaxDevices] = {false};
  bool& operator()(const gccnmf_handle* h) { return done[h->device % kGccnmfMaxDevices]; }
};

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// Carves aligned sub-buffers out of a caller-owned workspace.
struct WorkspaceCarver {
  char* base;
  size_t size, used = 0;
  WorkspaceCarver(void* p, size_t n) : base(static_cast<char*>(p)), size(n) {}
  template <typename T>
  T* take(size_t count) {
    used = align_up(used, 256);
    T* p = reinterpret_cast<T*>(base + used);
    used += count * sizeof(T);
    return p;
  }
  bool ok() const { return base != nullptr && used <= size; }
};

// A bank of Qe steering tables for the columns of a low-latency call (gccnmf_llbank_*): table e is E + e F D, (F, D) complex128 as
// gccnmf_ll_init stores E, and ET + e D Fp its transpose (D, Fp), bins F .. Fp - 1 zero.  Column t = s hops + i (frame i of stream
// s) is on table assign[s].  order lists the streams by entry, stable, and seg[e] .. seg[e + 1] are entry e's positions in it, so
// the kernels that reuse a table row across a tile of columns take their tiles from one entry at a time (steer_tile).
struct SteerBank {
  const double2 *E, *ET;
  const int32_t *assign, *order, *seg;
  int Qe, hops;
  int64_t Fp;
  __device__ __forceinline__ int entry(int t) const { return __ldg(assign + t / hops); }
  __device__ __forceinline__ int column(int u) const { return __ldg(order + u / hops) * hops + u % hops; }   // sorted position -> column
};

// Tile `cta` of the column tiles of width `tile` cut from each entry's sorted columns in turn: its entry (-1 past the last tile)
// and sorted positions [u0, u1).  At most ceil(T / tile) + Qe - 1 tiles exist.
__device__ __forceinline__ int steer_tile(const SteerBank& b, int tile, int cta, int& u0, int& u1) {
  int first = 0;
  for (int e = 0; e < b.Qe; ++e) {
    const int c0 = __ldg(b.seg + e) * b.hops, c1 = __ldg(b.seg + e + 1) * b.hops, n = (c1 - c0 + tile - 1) / tile;
    if (cta < first + n) {
      u0 = c0 + (cta - first) * tile;
      u1 = u0 + tile < c1 ? u0 + tile : c1;
      return e;
    }
    first += n;
  }
  u0 = u1 = 0;
  return -1;
}
inline int steer_tiles_max(int T, int tile, int Qe) { return (T + tile - 1) / tile + Qe; }

// A bank of Qd dictionaries for the columns of a low-latency call (gccnmf_lldict_*): entry e has K[e] <= Kmax atoms, W (F, K[e])
// f32 row-major at W + e wstride, its |W| column sums at colsum + e Kp, its transpose (K[e], Fp) at WT + e Kp Fp, rowsum(W) at
// rowsum + e F and its bf16 hi / lo planes as columns [e Kp, e Kp + Kp) of two (F, Qd Kp) planes (zero past K[e]).  Column t is on
// entry assign[t / hops]; order / seg sort the streams by entry as SteerBank's do, and segments() views them for steer_tile.
struct DictBank {
  const float *W, *colsum, *WT, *rowsum;
  const void* planes;
  const int32_t *K, *assign, *order, *seg;
  int Qd, hops, Kp, Kmax;
  int64_t wstride, Fp;
  __device__ __forceinline__ int entry(int t) const { return __ldg(assign + t / hops); }
  __device__ __forceinline__ int column(int u) const { return __ldg(order + u / hops) * hops + u % hops; }
  __device__ __forceinline__ SteerBank segments() const { return SteerBank{nullptr, nullptr, assign, order, seg, Qd, hops, Fp}; }
};

// scipy.signal.argrelmax(x) (order 1, mode 'clip': strict local maxima, never the end points), then the S largest peaks
// (gccNMFFunctions.py:100: peakIndexes[argsort(x[peakIndexes])[-numSources:]]) in ascending index order (:113), by every thread of
// one CTA.  x: D values in shared memory, written before the call; peak / chosen: D bytes of shared scratch.  Thread 0 writes the
// min(S, peaks) chosen indexes to out and gets the number of peaks back (the other threads' return value is unspecified).
// Equal peak values are ranked in stable order (argsort(kind='stable'): of two equal peaks the higher index ranks higher, so it
// is kept first).  The reference's default np.argsort is not stable, so when peak values tie exactly the host drop-in may keep a
// different one of them; with distinct peak values the two choose the same targets.
__device__ inline int select_peaks(const double* x, int D, int S, unsigned char* peak, unsigned char* chosen, int* num_peaks, int32_t* out) {
  if (threadIdx.x == 0) *num_peaks = 0;
  __syncthreads();
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    const bool p = d > 0 && d < D - 1 && x[d] > x[d - 1] && x[d] > x[d + 1];
    peak[d] = p ? 1 : 0;
    chosen[d] = 0;
    if (p) atomicAdd(num_peaks, 1);
  }
  __syncthreads();
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    if (!peak[d]) continue;
    int larger = 0;      // peaks that argsort places after this one: larger value, or the same value at a higher index
    for (int e = 0; e < D; ++e)
      if (peak[e] && (x[e] > x[d] || (x[e] == x[d] && e > d))) ++larger;
    chosen[d] = larger < S ? 1 : 0;
  }
  __syncthreads();
  if (threadIdx.x != 0) return 0;
  int n = 0;
  for (int d = 0; d < D && n < S; ++d)
    if (chosen[d]) out[n++] = d;
  return *num_peaks;
}

void gccnmf_tmap_cache_free(gccnmf_handle* h);
int gccnmf_get_twiddles(gccnmf_handle* h, int n, const double** tw64, const float** tw32);
