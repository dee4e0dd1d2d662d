// KL-NMF multiplicative updates (reference: gccNMF/gccNMFFunctions.py:69-83), float32 SIMT path.
//
// One iteration in reference order:
//   R = V / (W.H)                          gemm  (F x T2) over K     -> fused epilogue, R only
//   H *= (W^T.R) / (colsum(W) + a + eps)   gemm  (K x T2) over F     -> fused multiplicative epilogue
//   R = V / (W.H)                          again with the new H
//   numer = R.H^T, rowsum(H)               gemm  (F x K) over T2, split along T2 (output is small)
//   W *= numer / rowsum(H); unit-L2 atoms; H *= norms
// The float32 arithmetic follows numpy's (division, then multiply; column sums of W in row order).
#include "common.cuh"
#include "gemm_simt.cuh"

#include <algorithm>
#include <vector>

namespace {

constexpr int BM = 128, BN = 128, BK = 16, TM = 8, TN = 8;
constexpr int kGemmThreads = (BM / TM) * (BN / TN);
constexpr int kSplitT = 8;  // split of the T2 contraction for the (F x K) numerator

struct LoadRowMajorK {  // element (row, k) at p[row * ld + k]  (k contiguous)
  static constexpr bool kContigK = true;
  const float* p; int rows, kc; int64_t ld;
  __device__ float operator()(int r, int k) const { return (r < rows && k < kc) ? __ldg(p + (int64_t)r * ld + k) : 0.f; }
};
struct LoadColMajorK {  // element (row, k) at p[k * ld + row]  (row contiguous)
  static constexpr bool kContigK = false;
  const float* p; int rows, kc; int64_t ld;
  __device__ float operator()(int r, int k) const { return (r < rows && k < kc) ? __ldg(p + (int64_t)k * ld + r) : 0.f; }
};
struct LoadRowMajorKRange {  // k offset window [k_begin, k_end) for split-K
  static constexpr bool kContigK = true;
  const float* p; int rows; int k_begin, k_end; int64_t ld;
  __device__ float operator()(int r, int k) const {
    const int kk = k_begin + k;
    return (r < rows && kk < k_end) ? __ldg(p + (int64_t)r * ld + kk) : 0.f;
  }
};

struct EpiRatio {  // R = V / acc                                  gccNMFFunctions.py:76,77  V / dot(W, H)
  const float* V; float* R; int64_t ld;
  __device__ void operator()(int m, int n, float acc) const { R[(int64_t)m * ld + n] = V[(int64_t)m * ld + n] / acc; }
};
struct EpiUpdateH {  // H *= acc / (colsum(W) + alpha + eps)        gccNMFFunctions.py:76
  float* H; const float* colsumW; float alpha, eps; int64_t ld;
  __device__ void operator()(int m, int n, float acc) const {
    const float denom = (colsumW[m] + alpha) + eps;
    float* h = H + (int64_t)m * ld + n;
    *h = *h * (acc / denom);
  }
};
struct EpiStore {
  float* D; int64_t ld;
  __device__ void operator()(int m, int n, float acc) const { D[(int64_t)m * ld + n] = acc; }
};

// split-K variant of the plain kernel: blockIdx.z selects the k range and the output slab.
template <class Epi>
__global__ void __launch_bounds__(kGemmThreads, 2)
numer_splitk_kernel(int M, int N, int T2, int chunk, const float* R, const float* H, float* partial) {
  float acc[TM][TN];
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  const int k_begin = blockIdx.z * chunk;
  const int k_end = min(T2, k_begin + chunk);
  LoadRowMajorKRange a{R, M, k_begin, k_end, T2};
  LoadRowMajorKRange b{H, N, k_begin, k_end, T2};
  gemm_simt_mainloop<float, BM, BN, BK, TM, TN>(acc, m0, n0, max(0, k_end - k_begin), a, b);
  float* out = partial + (int64_t)blockIdx.z * M * N;
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const int m = gemm_row<BM, TM, BN / TN>(m0, i);
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      const int n = gemm_col<BN, TN, BN / TN>(n0, j);
      if (n < N) out[(int64_t)m * N + n] = acc[i][j];
    }
  }
}

// numer[i] = sum_s partial[s][i] in split order (deterministic).
__global__ void reduce_splits_kernel(const float* partial, int64_t n, int splits, float* out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float s = partial[i];
  for (int k = 1; k < splits; ++k) s += partial[(int64_t)k * n + i];
  out[i] = s;
}

// colsum[k] = sum_f W[f][k], rows added in order like numpy.sum(W, axis=0)  (gccNMFFunctions.py:76).
__global__ void colsum_kernel(const float* W, int F, int K, float* colsum) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= K) return;
  float s = 0.f;
  for (int f = 0; f < F; ++f) s += W[(int64_t)f * K + k];
  colsum[k] = s;
}

// rowsum[k] = sum_t H[k][t]   (gccNMFFunctions.py:77 sum(H, axis=1)); one block per row.
__global__ void rowsum_kernel(const float* H, int T2, float* rowsum) {
  __shared__ float warp_sums[32];
  const float* row = H + (int64_t)blockIdx.x * T2;
  float s = 0.f;
  for (int t = threadIdx.x; t < T2; t += blockDim.x) s += row[t];
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) warp_sums[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    s = threadIdx.x < (blockDim.x >> 5) ? warp_sums[threadIdx.x] : 0.f;
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (threadIdx.x == 0) rowsum[blockIdx.x] = s;
  }
}

// W *= numer / rowsum(H) (:77); norms = sqrt(sum(W^2, 0)) (:79); W /= norms (:80).
// Block = 32 columns x 32 row-groups; column reductions go through shared memory in row-group order.
constexpr int kApplyCols = 32, kApplyGroups = 32;
__global__ void __launch_bounds__(kApplyCols * kApplyGroups)
apply_w_kernel(float* W, const float* numer, const float* rowsumH, int F, int K, float* norms) {
  __shared__ float part[kApplyGroups][kApplyCols + 1];
  __shared__ float norm_s[kApplyCols];
  const int c = threadIdx.x % kApplyCols, g = threadIdx.x / kApplyCols;
  const int k = blockIdx.x * kApplyCols + c;
  // rows f = g, g + 32, ... (one column per thread, 32 row groups per CTA)
  float sumsq = 0.f;
  if (k < K) {
    const float rs = rowsumH[k];
    for (int f = g; f < F; f += kApplyGroups) {
      const int64_t i = (int64_t)f * K + k;
      const float w = W[i] * (numer[i] / rs);
      W[i] = w;
      sumsq += w * w;
    }
  }
  part[g][c] = sumsq;
  __syncthreads();
  if (g == 0) {
    float s = 0.f;
    for (int j = 0; j < kApplyGroups; ++j) s += part[j][c];
    const float nrm = sqrtf(s);
    norm_s[c] = nrm;
    if (k < K) norms[k] = nrm;
  }
  __syncthreads();
  if (k < K) {
    const float nrm = norm_s[c];
    for (int f = g; f < F; f += kApplyGroups) {
      const int64_t i = (int64_t)f * K + k;
      W[i] = W[i] / nrm;
    }
  }
}

// H *= norms[:, None]   (:81)
__global__ void scale_rows_kernel(float* H, const float* norms, int K, int T2) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)K * T2) return;
  H[i] = H[i] * norms[i / T2];
}

struct Workspace {
  float *R, *partial, *numer, *colsumW, *norms;
  bool ok;
};
Workspace carve(void* ws, size_t bytes, int F, int T2, int K) {
  WorkspaceCarver c(ws, bytes);
  Workspace w;
  w.R = c.take<float>((size_t)F * T2);
  w.partial = c.take<float>((size_t)kSplitT * F * K);
  w.numer = c.take<float>((size_t)F * K + K);
  w.colsumW = c.take<float>(K);
  w.norms = c.take<float>(K);
  w.ok = c.ok();
  return w;
}

dim3 gemm_grid(int M, int N) { return dim3((N + BN - 1) / BN, (M + BM - 1) / BM, 1); }

int check_dims(gccnmf_handle* h, int F, int T2, int K) {
  GCCNMF_REQUIRE(h, F > 0 && T2 > 0 && K > 0, "klnmf: F, T2, K must be positive (got %d, %d, %d)", F, T2, K);
  return 0;
}

int ratio(gccnmf_handle* h, const float* V, int F, int T2, const float* W, const float* H, int K, float* R, void* stream) {
  LoadRowMajorK a{W, F, K, K};
  LoadColMajorK b{H, T2, K, T2};
  EpiRatio e{V, R, T2};
  auto kernel = gemm_simt_kernel<float, BM, BN, BK, TM, TN, LoadRowMajorK, LoadColMajorK, EpiRatio>;
  GCCNMF_LAUNCH(h, kernel, gemm_grid(F, T2), kGemmThreads, 0, stream, F, T2, K, a, b, e);
  return 0;
}

int update_H_impl(gccnmf_handle* h, const float* V, int F, int T2, const float* W, float* H, int K, float alpha,
                  float eps, const Workspace& w, bool have_colsum, void* stream) {
  int st = ratio(h, V, F, T2, W, H, K, w.R, stream);
  if (st) return st;
  if (!have_colsum) GCCNMF_LAUNCH(h, colsum_kernel, (K + 127) / 128, 128, 0, stream, W, F, K, w.colsumW);
  LoadColMajorK a{W, K, F, K};    // A(m = atom, k = f) = W[f][atom]
  LoadColMajorK b{w.R, T2, F, T2};  // B(n = t,   k = f) = R[f][t]
  EpiUpdateH e{H, w.colsumW, alpha, eps, T2};
  auto kernel = gemm_simt_kernel<float, BM, BN, BK, TM, TN, LoadColMajorK, LoadColMajorK, EpiUpdateH>;
  GCCNMF_LAUNCH(h, kernel, gemm_grid(K, T2), kGemmThreads, 0, stream, K, T2, F, a, b, e);
  return 0;
}

int partial_W_impl(gccnmf_handle* h, const float* V, int F, int T2, const float* W, const float* H, int K,
                   float* numer, const Workspace& w, void* stream) {
  int st = ratio(h, V, F, T2, W, H, K, w.R, stream);
  if (st) return st;
  const int chunk = ((T2 + kSplitT - 1) / kSplitT + BK - 1) / BK * BK;
  const int splits = (T2 + chunk - 1) / chunk;
  dim3 grid = gemm_grid(F, K);
  grid.z = splits;
  auto kernel = numer_splitk_kernel<EpiStore>;
  GCCNMF_LAUNCH(h, kernel, grid, kGemmThreads, 0, stream, F, K, T2, chunk, w.R, H, w.partial);
  const int64_t n = (int64_t)F * K;
  GCCNMF_LAUNCH(h, reduce_splits_kernel, (unsigned)((n + 255) / 256), 256, 0, stream, w.partial, n, splits, numer);
  GCCNMF_LAUNCH(h, rowsum_kernel, K, 256, 0, stream, H, T2, numer + n);
  return 0;
}

int apply_W_impl(gccnmf_handle* h, int F, int T2, float* W, float* H, int K, const float* numer, const Workspace& w, void* stream) {
  GCCNMF_LAUNCH(h, apply_w_kernel, (K + kApplyCols - 1) / kApplyCols, kApplyCols * kApplyGroups, 0, stream,
                W, numer, numer + (int64_t)F * K, F, K, w.norms);
  const int64_t n = (int64_t)K * T2;
  GCCNMF_LAUNCH(h, scale_rows_kernel, (unsigned)((n + 255) / 256), 256, 0, stream, H, w.norms, K, T2);
  return 0;
}

}  // namespace

// tensor-core path: TMA-fed plane GEMM (klnmf_tma.cu)
bool gccnmf_klnmf_tma_supported(int F, int T2, int K);
size_t gccnmf_klnmf_tma_workspace_bytes(int F, int T2, int K);
int gccnmf_klnmf_tma_prepare(gccnmf_handle* h, const float* V, int64_t ld_v, int F, int T2, const float* W, const float* H, int K, void* workspace,
                             size_t workspace_bytes, bool need_vt, bool need_w, bool need_ht, void* stream);
bool gccnmf_klnmf_tma_batch_supported(gccnmf_handle* h, int F, int T2, int K);
int gccnmf_klnmf_tma_batched(gccnmf_handle* h, const float* V, int64_t ld_v, int64_t clip_stride_v, int B, int F, int T2, float* W, float* H, int K,
                             int iterations, float alpha, float eps, bool update_W, void* workspace, size_t clip_bytes, void* stream);
size_t gccnmf_klnmf_tma_ragged_table_per_clip();
int gccnmf_klnmf_tma_ragged(gccnmf_handle* h, int n, const float* const* V, const int64_t* ld_v, const int* T2, float* const* W, float* const* H,
                            void* const* ws, int F, int K, int iterations, float alpha, float eps, bool update_W, void* table, void* stream);
int gccnmf_klnmf_tma_update_H(gccnmf_handle* h, const float* V, int F, int T2, const float* W, float* H, int K, float alpha, float eps,
                              void* workspace, size_t workspace_bytes, int colsum_state, bool pending_norms, void* stream);
int gccnmf_klnmf_tma_partial_W(gccnmf_handle* h, const float* V, int F, int T2, const float* W, const float* H, int K, void* workspace,
                               size_t workspace_bytes, bool have_rowsum, void* stream);
int gccnmf_klnmf_tma_partial_W_to(gccnmf_handle* h, const float* V, int F, int T2, const float* W, const float* H, int K, void* workspace,
                                  size_t workspace_bytes, bool have_rowsum, float* numer_out, void* stream);
int gccnmf_klnmf_tma_apply_W(gccnmf_handle* h, int F, int T2, float* W, int K, const float* numer, bool numer_is_multicast,
                             void* workspace, size_t workspace_bytes, void* stream);
int gccnmf_klnmf_tma_finish(gccnmf_handle* h, int F, int T2, float* H, int K, bool pending_norms, void* workspace,
                            size_t workspace_bytes, void* stream);
int gccnmf_klnmf_tma_pack_numer(gccnmf_handle* h, int F, int T2, int K, float* numer, void* workspace, size_t workspace_bytes, void* stream);
// The TMA path keeps W unnormalised inside the loop (see klnmf_tma.cu): the caller's W is normalised here, once
int gccnmf_klnmf_tma_finish_W(gccnmf_handle* h, int F, int T2, float* W, int K, void* workspace, size_t workspace_bytes, void* stream);
// cross-rank signalling folded into the numerator pack / the W update (no host-launched barrier in between)
int gccnmf_klnmf_tma_pack_numer_mc(gccnmf_handle* h, int F, int T2, int K, float* numer, unsigned* mc_counter, void* workspace, size_t workspace_bytes,
                                   void* stream);
int gccnmf_klnmf_tma_apply_W_mc(gccnmf_handle* h, int F, int T2, float* W, int K, const float* numer, bool numer_is_multicast,
                                const unsigned* arrival_counter, unsigned arrivals_expected, void* workspace, size_t workspace_bytes, void* stream);

// Shapes the plane GEMM does not cover (K % 8 != 0, tiny problems) and the force_simt_nmf option run the float32 SIMT kernels above.
int gccnmf_klnmf_tma_reduce_bcast(gccnmf_handle* h, int F, int T2, int K, const float* numer_multicast, float* reduced_multicast, int rank, int world,
                                  const unsigned* arrivals_in, unsigned arrivals_expected, unsigned* arrivals_out_mc, void* workspace,
                                  size_t workspace_bytes, void* stream);

int gccnmf_klnmf_tma_l2_window(gccnmf_handle* h, int F, int T2, int K, bool enable, void* workspace, size_t workspace_bytes);

int64_t gccnmf_klnmf_tma_pull_floats(int F, int layout_T2, int K);
bool gccnmf_klnmf_tma_pull_supported(gccnmf_handle* h, int F, int T2, int K);
int gccnmf_klnmf_tma_step_pull(gccnmf_handle* h, const float* V, int F, int T2, float* W, float* H, int K, float alpha, float eps, int iteration,
                               int64_t epoch, int rank, int world, float* const* bases, int layout_T2, int two_shot, int want_direct,
                               void* workspace, size_t workspace_bytes, void* stream);
bool gccnmf_klnmf_tma_pull_direct(gccnmf_handle* h, int F, int T2, int K);
bool gccnmf_klnmf_tma_pull_fused_ok(gccnmf_handle* h, int F, int K);

static bool use_tc(const gccnmf_handle* h, int F, int T2, int K) { return !h->force_simt_nmf && gccnmf_klnmf_tma_supported(F, T2, K); }

static size_t simt_workspace_bytes(int F, int T2, int K) {
  size_t n = 0;
  auto add = [&](size_t count) { n = align_up(n, 256) + count * sizeof(float); };
  add((size_t)F * T2);
  add((size_t)kSplitT * F * K);
  add((size_t)F * K + K);
  add(K);
  add(K);
  return align_up(n, 256);
}

// The whole loop on the tensor-core path; V is read at row pitch ld_v.
static int klnmf_tc(gccnmf_handle* h, const float* V, int64_t ld_v, int F, int T2, float* W, float* H, int K, int iterations, float sparsity_alpha,
                    float epsilon, int update_W, void* workspace, size_t workspace_bytes, void* stream) {
  if (int st = gccnmf_klnmf_tma_prepare(h, V, ld_v, F, T2, W, H, K, workspace, workspace_bytes, true, true, true, stream)) return st;
  if (int st = gccnmf_klnmf_tma_l2_window(h, F, T2, K, true, workspace, workspace_bytes)) return st;
  struct WindowGuard { gccnmf_handle* h; ~WindowGuard() { h->l2_window_base = nullptr; h->l2_window_bytes = 0; } } guard{h};
  for (int it = 0; it < iterations; ++it) {
    // colsum(W) comes out of the previous W update; with a fixed dictionary it is computed once
    // (in the (U, G) gauge nothing is rescaled inside the loop: see klnmf_tma.cu)
    if (int st = gccnmf_klnmf_tma_update_H(h, V, F, T2, W, H, K, sparsity_alpha, epsilon, workspace, workspace_bytes,
                                          it == 0 ? 0 : (update_W ? 2 : 1), update_W && it > 0, stream)) return st;
    if (!update_W) continue;
    if (int st = gccnmf_klnmf_tma_partial_W(h, V, F, T2, W, H, K, workspace, workspace_bytes, true, stream)) return st;
    if (int st = gccnmf_klnmf_tma_apply_W(h, F, T2, W, K, nullptr, false, workspace, workspace_bytes, stream)) return st;
  }
  if (int st = gccnmf_klnmf_tma_finish(h, F, T2, H, K, update_W != 0, workspace, workspace_bytes, stream)) return st;
  if (update_W) return gccnmf_klnmf_tma_finish_W(h, F, T2, W, K, workspace, workspace_bytes, stream);
  return GCCNMF_OK;
}

// The whole loop on the float32 SIMT path (V at pitch T2).
static int klnmf_simt(gccnmf_handle* h, const float* V, int F, int T2, float* W, float* H, int K, int iterations, float sparsity_alpha, float epsilon,
                      int update_W, void* workspace, size_t workspace_bytes, void* stream) {
  Workspace w = carve(workspace, workspace_bytes, F, T2, K);
  for (int it = 0; it < iterations; ++it) {
    // with a fixed dictionary colsum(W) only has to be computed once
    int st = update_H_impl(h, V, F, T2, W, H, K, sparsity_alpha, epsilon, w, !update_W && it > 0, stream);
    if (st) return st;
    if (!update_W) continue;
    st = partial_W_impl(h, V, F, T2, W, H, K, w.numer, w, stream);
    if (st) return st;
    st = apply_W_impl(h, F, T2, W, H, K, w.numer, w, stream);
    if (st) return st;
  }
  return GCCNMF_OK;
}

// Per-clip region of a batched run's workspace: the single-clip workspace, or -- when larger -- the float32 path's workspace plus a
// packed copy of the clip's V (that path reads V at pitch T2; at tensor-core shapes the copy fits inside the single-clip size).
static size_t batch_clip_bytes(int F, int T2, int K) {
  return std::max(gccnmf_klnmf_workspace_bytes(F, T2, K), simt_workspace_bytes(F, T2, K) + align_up((size_t)F * T2 * sizeof(float), 256));
}
constexpr int kMaxBatchClips = 65535 / 8;     // grid z of a batched contraction = clips x k-splits (at most 8)

// A ragged run's workspace: the per-call table (its size depends on B only; 256 bytes of it keep the table 128-byte aligned), then
// clip b's region of a batched run on its shape, back to back.
static size_t ragged_table_bytes(int B) { return (size_t)B * gccnmf_klnmf_tma_ragged_table_per_clip() + 256; }

// One clip alone, on its region of a batched or ragged run's workspace: the tensor-core loop, or the float32 SIMT loop on a packed copy
// of V when its rows are not T2 apart.
static int klnmf_one_clip(gccnmf_handle* h, const float* V, int64_t ld_v, int F, int T2, float* W, float* H, int K, int iterations, float sparsity_alpha,
                          float epsilon, int update_W, char* ws, size_t clip_bytes, void* stream) {
  if (use_tc(h, F, T2, K)) return klnmf_tc(h, V, ld_v, F, T2, W, H, K, iterations, sparsity_alpha, epsilon, update_W, ws, clip_bytes, stream);
  const size_t simt_bytes = simt_workspace_bytes(F, T2, K);
  if (ld_v != T2) {
    float* packed = reinterpret_cast<float*>(ws + simt_bytes);
    GCCNMF_CHECK_CUDA(h, cudaMemcpy2DAsync(packed, (size_t)T2 * sizeof(float), V, (size_t)ld_v * sizeof(float), (size_t)T2 * sizeof(float), F,
                                           cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
    V = packed;
  }
  return klnmf_simt(h, V, F, T2, W, H, K, iterations, sparsity_alpha, epsilon, update_W, ws, simt_bytes, stream);
}

extern "C" {

int gccnmf_klnmf_uses_tensor_cores(const gccnmf_handle* h, int F, int T2, int K) { return h && use_tc(h, F, T2, K) ? 1 : 0; }

size_t gccnmf_klnmf_workspace_bytes(int F, int T2, int K) {
  if (F <= 0 || T2 <= 0 || K <= 0) return 0;
  size_t n = simt_workspace_bytes(F, T2, K);
  if (gccnmf_klnmf_tma_supported(F, T2, K)) n = std::max(n, gccnmf_klnmf_tma_workspace_bytes(F, T2, K));
  return n;
}

int gccnmf_klnmf_begin(gccnmf_handle* h, const float* V, int F, int T2, const float* W, const float* H, int K,
                       void* workspace, size_t workspace_bytes, void* stream) {
  GCCNMF_ENTER(h);
  if (int st = check_dims(h, F, T2, K)) return st;
  if (!workspace || workspace_bytes < gccnmf_klnmf_workspace_bytes(F, T2, K))
    return gccnmf_fail(h, GCCNMF_ERR_WORKSPACE, "klnmf workspace too small: need %zu bytes", gccnmf_klnmf_workspace_bytes(F, T2, K));
  if (use_tc(h, F, T2, K)) {
    if (int st = gccnmf_klnmf_tma_prepare(h, V, (int64_t)T2, F, T2, W, H, K, workspace, workspace_bytes, true, true, true, stream)) return st;
    return gccnmf_klnmf_tma_l2_window(h, F, T2, K, true, workspace, workspace_bytes);      // cleared by gccnmf_klnmf_end
  }
  return GCCNMF_OK;
}

int gccnmf_klnmf_step_numer(gccnmf_handle* h, const float* V, int F, int T2, const float* W, float* H, int K,
                            float sparsity_alpha, float epsilon, int iteration, float* numer, void* workspace,
                            size_t workspace_bytes, void* stream) {
  GCCNMF_ENTER(h);
  if (int st = check_dims(h, F, T2, K)) return st;
  GCCNMF_REQUIRE(h, numer != nullptr && iteration >= 0, "klnmf_step_numer: bad arguments");
  if (!workspace || workspace_bytes < gccnmf_klnmf_workspace_bytes(F, T2, K))
    return gccnmf_fail(h, GCCNMF_ERR_WORKSPACE, "klnmf workspace too small: need %zu bytes", gccnmf_klnmf_workspace_bytes(F, T2, K));
  if (use_tc(h, F, T2, K)) {
    if (int st = gccnmf_klnmf_tma_update_H(h, V, F, T2, W, H, K, sparsity_alpha, epsilon, workspace, workspace_bytes, iteration > 0 ? 2 : 0,
                                          iteration > 0, stream)) return st;
    if (int st = gccnmf_klnmf_tma_partial_W_to(h, V, F, T2, W, H, K, workspace, workspace_bytes, true, numer, stream)) return st;
    return gccnmf_klnmf_tma_pack_numer(h, F, T2, K, numer, workspace, workspace_bytes, stream);
  }
  Workspace w = carve(workspace, workspace_bytes, F, T2, K);
  if (int st = update_H_impl(h, V, F, T2, W, H, K, sparsity_alpha, epsilon, w, false, stream)) return st;
  return partial_W_impl(h, V, F, T2, W, H, K, numer, w, stream);
}

int gccnmf_klnmf_step_apply(gccnmf_handle* h, int F, int T2, float* W, float* H, int K, const float* numer,
                            void* workspace, size_t workspace_bytes, void* stream) {
  GCCNMF_ENTER(h);
  if (int st = check_dims(h, F, T2, K)) return st;
  GCCNMF_REQUIRE(h, numer != nullptr, "klnmf_step_apply: NULL numerator");
  if (!workspace || workspace_bytes < gccnmf_klnmf_workspace_bytes(F, T2, K))
    return gccnmf_fail(h, GCCNMF_ERR_WORKSPACE, "klnmf workspace too small: need %zu bytes", gccnmf_klnmf_workspace_bytes(F, T2, K));
  if (use_tc(h, F, T2, K)) return gccnmf_klnmf_tma_apply_W(h, F, T2, W, K, numer, false, workspace, workspace_bytes, stream);
  Workspace w = carve(workspace, workspace_bytes, F, T2, K);
  return apply_W_impl(h, F, T2, W, H, K, numer, w, stream);
}

int gccnmf_klnmf_step_apply_multimem(gccnmf_handle* h, int F, int T2, float* W, float* H, int K, const float* numer_multicast,
                                     void* workspace, size_t workspace_bytes, void* stream) {
  GCCNMF_ENTER(h);
  if (int st = check_dims(h, F, T2, K)) return st;
  (void)H;
  GCCNMF_REQUIRE(h, numer_multicast != nullptr, "klnmf_step_apply_multimem: NULL multicast address");
  if (!use_tc(h, F, T2, K)) return gccnmf_fail(h, GCCNMF_ERR_UNSUPPORTED, "klnmf_step_apply_multimem: only the tensor-core path reads the numerator through multimem");
  if (!workspace || workspace_bytes < gccnmf_klnmf_workspace_bytes(F, T2, K))
    return gccnmf_fail(h, GCCNMF_ERR_WORKSPACE, "klnmf workspace too small: need %zu bytes", gccnmf_klnmf_workspace_bytes(F, T2, K));
  return gccnmf_klnmf_tma_apply_W(h, F, T2, W, K, numer_multicast, true, workspace, workspace_bytes, stream);
}

// One KL-NMF iteration of a frame-sharded run with the cross-rank sum of the W-update numerator formed INSIDE the NVSwitch and no
// host-side step in between:  G1..G4 -> pack (this rank's (F*K + K) partial into its symmetric buffer; the last CTA adds 1 to the
// arrival counter of EVERY rank through the multicast address) -> W update (waits until its own copy of the counter shows
// `arrivals_expected` arrivals, then reads every word with multimem.ld_reduce).  numer_local / counter_local: this rank's addresses of
// the symmetric buffer; numer_multicast / counter_multicast: the multicast addresses of the same offsets.
int gccnmf_klnmf_step_multimem(gccnmf_handle* h, const float* V, int F, int T2, float* W, float* H, int K, float sparsity_alpha, float epsilon,
                               int iteration, float* numer_local, const float* numer_multicast, const uint32_t* counter_local,
                               uint32_t* counter_multicast, uint32_t arrivals_expected, void* workspace, size_t workspace_bytes, void* stream) {
  GCCNMF_ENTER(h);
  if (int st = check_dims(h, F, T2, K)) return st;
  GCCNMF_REQUIRE(h, numer_local && numer_multicast && counter_local && counter_multicast && iteration >= 0, "klnmf_step_multimem: bad arguments");
  if (!use_tc(h, F, T2, K)) return gccnmf_fail(h, GCCNMF_ERR_UNSUPPORTED, "klnmf_step_multimem: shape not covered by the tensor-core path");
  if (!workspace || workspace_bytes < gccnmf_klnmf_workspace_bytes(F, T2, K))
    return gccnmf_fail(h, GCCNMF_ERR_WORKSPACE, "klnmf workspace too small: need %zu bytes", gccnmf_klnmf_workspace_bytes(F, T2, K));
  if (int st = gccnmf_klnmf_tma_update_H(h, V, F, T2, W, H, K, sparsity_alpha, epsilon, workspace, workspace_bytes, iteration > 0 ? 2 : 0, iteration > 0,
                                         stream)) return st;
  if (int st = gccnmf_klnmf_tma_partial_W_to(h, V, F, T2, W, H, K, workspace, workspace_bytes, true, numer_local, stream)) return st;
  if (int st = gccnmf_klnmf_tma_pack_numer_mc(h, F, T2, K, numer_local, counter_multicast, workspace, workspace_bytes, stream)) return st;
  return gccnmf_klnmf_tma_apply_W_mc(h, F, T2, W, K, numer_multicast, true, counter_local, arrivals_expected, workspace, workspace_bytes, stream);
}

// The same iteration with a TWO-SHOT exchange (reduce-scatter + all-gather inside the switch): after the pack every rank sums only its
// 1 / world slice of the numerator with multimem.ld_reduce and multicasts the result into the `reduced` buffer of every rank
// (multimem.st); the W update then reads plain local memory once the second arrival counter is complete.  Link traffic per GPU and
// iteration is one numerator in each direction for any world size.  counters_*: two uint32 (pack arrivals, slice arrivals).
int gccnmf_klnmf_step_multimem2(gccnmf_handle* h, const float* V, int F, int T2, float* W, float* H, int K, float sparsity_alpha, float epsilon,
                                int iteration, int rank, int world, float* numer_local, const float* numer_multicast, const float* reduced_local,
                                float* reduced_multicast, const uint32_t* counters_local, uint32_t* counters_multicast, uint32_t arrivals_expected,
                                void* workspace, size_t workspace_bytes, void* stream) {
  GCCNMF_ENTER(h);
  if (int st = check_dims(h, F, T2, K)) return st;
  GCCNMF_REQUIRE(h, numer_local && numer_multicast && reduced_local && reduced_multicast && counters_local && counters_multicast && iteration >= 0 &&
                        world >= 1 && rank >= 0 && rank < world, "klnmf_step_multimem2: bad arguments");
  if (!use_tc(h, F, T2, K)) return gccnmf_fail(h, GCCNMF_ERR_UNSUPPORTED, "klnmf_step_multimem2: shape not covered by the tensor-core path");
  if (!workspace || workspace_bytes < gccnmf_klnmf_workspace_bytes(F, T2, K))
    return gccnmf_fail(h, GCCNMF_ERR_WORKSPACE, "klnmf workspace too small: need %zu bytes", gccnmf_klnmf_workspace_bytes(F, T2, K));
  if (int st = gccnmf_klnmf_tma_update_H(h, V, F, T2, W, H, K, sparsity_alpha, epsilon, workspace, workspace_bytes, iteration > 0 ? 2 : 0, iteration > 0,
                                         stream)) return st;
  if (int st = gccnmf_klnmf_tma_partial_W_to(h, V, F, T2, W, H, K, workspace, workspace_bytes, true, numer_local, stream)) return st;
  if (int st = gccnmf_klnmf_tma_pack_numer_mc(h, F, T2, K, numer_local, counters_multicast, workspace, workspace_bytes, stream)) return st;
  if (int st = gccnmf_klnmf_tma_reduce_bcast(h, F, T2, K, numer_multicast, reduced_multicast, rank, world, counters_local, arrivals_expected,
                                             counters_multicast + 1, workspace, workspace_bytes, stream)) return st;
  return gccnmf_klnmf_tma_apply_W_mc(h, F, T2, W, K, reduced_local, false, counters_local + 1, arrivals_expected, workspace, workspace_bytes, stream);
}

// PULL exchange (two_shot: 0 one-shot, 1 two-shot, 2 inside the W update): nothing is pushed over the links and nothing is reduced in
// the switch.  Form 2: the W-update CTA that owns a tile sums this rank's k-split slabs for it, publishes the tile, flags it on every
// rank, waits for the same tile of the other ranks and reads them -- no pack kernel, no kernel boundary inside the exchange.  Forms
// 0 / 1:  The numerator contraction writes this rank's
// (F, K) partial straight into its symmetric buffer and its last CTA adds 1 to every rank's arrival counter; then either every rank's
// W update reads all ranks' partials with plain peer loads and adds them in rank order (two_shot = 0: (world - 1) numerators inbound
// per GPU), or each rank first sums its 1 / world slice the same way into its own buffer and the W updates fetch each word from its
// owner (two_shot = 1: one numerator each way for any world size).  Row sums of G are read from every rank's slots directly.  No pack
// pass, no system-scope fence, no multimem instruction; works on any peer-mapped symmetric buffer.
// bases: HOST array of `world` device pointers -- every rank's buffer as mapped in this process (gccnmf_klnmf_pull_buffer_floats
// floats each, zero before the first iteration); layout_T2: the largest 2T over the ranks (same value on every rank); epoch: how
// many iterations earlier runs have executed on this buffer (its arrival counters keep counting, its halves alternate by parity).
int64_t gccnmf_klnmf_pull_buffer_floats(int F, int layout_T2, int K) {
  if (F <= 0 || layout_T2 <= 0 || K <= 0) return 0;
  return gccnmf_klnmf_tma_pull_floats(F, layout_T2, K);
}

int gccnmf_klnmf_pull_supported(gccnmf_handle* h, int F, int T2, int K) {
  GCCNMF_ENTER(h);
  if (!(F > 0 && T2 > 0 && K > 0 && use_tc(h, F, T2, K) && gccnmf_klnmf_tma_pull_supported(h, F, T2, K))) return 0;
  return 1 | (gccnmf_klnmf_tma_pull_direct(h, F, T2, K) ? 2 : 0) | (gccnmf_klnmf_tma_pull_fused_ok(h, F, K) ? 4 : 0);
}

int gccnmf_klnmf_step_pull(gccnmf_handle* h, const float* V, int F, int T2, float* W, float* H, int K, float sparsity_alpha, float epsilon,
                           int iteration, int64_t epoch, int rank, int world, void* const* bases, int layout_T2, int two_shot, int direct,
                           void* workspace, size_t workspace_bytes, void* stream) {
  GCCNMF_ENTER(h);
  if (int st = check_dims(h, F, T2, K)) return st;
  GCCNMF_REQUIRE(h, bases && iteration >= 0 && epoch >= 0 && world >= 1 && world <= 8 && rank >= 0 && rank < world, "klnmf_step_pull: bad arguments");
  for (int r = 0; r < world; ++r) GCCNMF_REQUIRE(h, bases[r] != nullptr, "klnmf_step_pull: NULL buffer of rank %d", r);
  if (!use_tc(h, F, T2, K)) return gccnmf_fail(h, GCCNMF_ERR_UNSUPPORTED, "klnmf_step_pull: shape not covered by the tensor-core path");
  if (!workspace || workspace_bytes < gccnmf_klnmf_workspace_bytes(F, T2, K))
    return gccnmf_fail(h, GCCNMF_ERR_WORKSPACE, "klnmf workspace too small: need %zu bytes", gccnmf_klnmf_workspace_bytes(F, T2, K));
  return gccnmf_klnmf_tma_step_pull(h, V, F, T2, W, H, K, sparsity_alpha, epsilon, iteration, epoch, rank, world, reinterpret_cast<float* const*>(bases),
                                    layout_T2, two_shot, direct, workspace, workspace_bytes, stream);
}

int gccnmf_klnmf_end(gccnmf_handle* h, int F, int T2, float* W, float* H, int K, int iterations_done, void* workspace,
                     size_t workspace_bytes, void* stream) {
  GCCNMF_ENTER(h);
  if (int st = check_dims(h, F, T2, K)) return st;
  h->l2_window_base = nullptr;
  h->l2_window_bytes = 0;
  if (use_tc(h, F, T2, K)) {
    if (int st = gccnmf_klnmf_tma_finish(h, F, T2, H, K, iterations_done > 0, workspace, workspace_bytes, stream)) return st;
    if (iterations_done > 0) return gccnmf_klnmf_tma_finish_W(h, F, T2, W, K, workspace, workspace_bytes, stream);
  }
  return GCCNMF_OK;
}

int gccnmf_klnmf(gccnmf_handle* h, const float* V, int F, int T2, float* W, float* H, int K, int iterations,
                 float sparsity_alpha, float epsilon, int update_W, void* workspace, size_t workspace_bytes, void* stream) {
  GCCNMF_ENTER(h);
  if (int st = check_dims(h, F, T2, K)) return st;
  GCCNMF_REQUIRE(h, iterations >= 0, "klnmf: iterations must be >= 0 (got %d)", iterations);
  if (!workspace || workspace_bytes < gccnmf_klnmf_workspace_bytes(F, T2, K))
    return gccnmf_fail(h, GCCNMF_ERR_WORKSPACE, "klnmf workspace too small: need %zu bytes", gccnmf_klnmf_workspace_bytes(F, T2, K));
  if (iterations == 0) return GCCNMF_OK;
  if (use_tc(h, F, T2, K))
    return klnmf_tc(h, V, (int64_t)T2, F, T2, W, H, K, iterations, sparsity_alpha, epsilon, update_W, workspace, workspace_bytes, stream);
  return klnmf_simt(h, V, F, T2, W, H, K, iterations, sparsity_alpha, epsilon, update_W, workspace, workspace_bytes, stream);
}

size_t gccnmf_klnmf_batched_workspace_bytes(int B, int F, int T2, int K) {
  if (B < 1 || B > kMaxBatchClips || F <= 0 || T2 <= 0 || K <= 0) return 0;
  return (size_t)B * batch_clip_bytes(F, T2, K);
}

int gccnmf_klnmf_batched(gccnmf_handle* h, const float* V, int64_t ld_v, int64_t clip_stride_v, int B, int F, int T2, float* W, float* H, int K,
                         int iterations, float sparsity_alpha, float epsilon, int update_W, void* workspace, size_t workspace_bytes, void* stream) {
  GCCNMF_ENTER(h);
  GCCNMF_REQUIRE(h, B >= 1 && B <= kMaxBatchClips, "klnmf_batched: B must be 1 .. %d (got %d)", kMaxBatchClips, B);
  if (int st = check_dims(h, F, T2, K)) return st;
  GCCNMF_REQUIRE(h, V && W && H, "klnmf_batched: NULL V, W or H");
  GCCNMF_REQUIRE(h, ld_v >= T2 && clip_stride_v >= 0, "klnmf_batched: V pitch %lld < T2 %d or negative clip stride %lld", (long long)ld_v, T2,
                 (long long)clip_stride_v);
  GCCNMF_REQUIRE(h, iterations >= 0, "klnmf_batched: iterations must be >= 0 (got %d)", iterations);
  const size_t clip_bytes = batch_clip_bytes(F, T2, K);
  if (!workspace || workspace_bytes < (size_t)B * clip_bytes)
    return gccnmf_fail(h, GCCNMF_ERR_WORKSPACE, "klnmf_batched workspace too small: need %zu bytes", (size_t)B * clip_bytes);
  if (iterations == 0) return GCCNMF_OK;
  char* ws = static_cast<char*>(workspace);
  const int64_t fk = (int64_t)F * K, kt = (int64_t)K * T2;
  if (use_tc(h, F, T2, K) && gccnmf_klnmf_tma_batch_supported(h, F, T2, K))
    return gccnmf_klnmf_tma_batched(h, V, ld_v, clip_stride_v, B, F, T2, W, H, K, iterations, sparsity_alpha, epsilon, update_W != 0, workspace,
                                    clip_bytes, stream);
  // an option the batch form leaves out, or the float32 SIMT path (tiny or odd shapes, force_simt_nmf): one clip at a time
  for (int b = 0; b < B; ++b)
    if (int st = klnmf_one_clip(h, V + b * clip_stride_v, ld_v, F, T2, W + b * fk, H + b * kt, K, iterations, sparsity_alpha, epsilon, update_W,
                                ws + b * clip_bytes, clip_bytes, stream)) return st;
  return GCCNMF_OK;
}

size_t gccnmf_klnmf_ragged_workspace_bytes(int B, int F, const int* T2, int K) {
  if (B < 1 || B > kMaxBatchClips || F <= 0 || K <= 0 || !T2) return 0;
  size_t n = ragged_table_bytes(B);
  for (int b = 0; b < B; ++b) {
    if (T2[b] <= 0) return 0;
    n += batch_clip_bytes(F, T2[b], K);
  }
  return n;
}

int gccnmf_klnmf_ragged(gccnmf_handle* h, const float* const* V, const int64_t* ld_v, const int* T2, int B, int F, float* W, float* const* H, int K,
                        int iterations, float sparsity_alpha, float epsilon, int update_W, void* workspace, size_t workspace_bytes, void* stream) {
  GCCNMF_ENTER(h);
  GCCNMF_REQUIRE(h, B >= 1 && B <= kMaxBatchClips, "klnmf_ragged: B must be 1 .. %d (got %d)", kMaxBatchClips, B);
  GCCNMF_REQUIRE(h, V && ld_v && T2 && W && H, "klnmf_ragged: NULL V, ld_v, T2, W or H");
  for (int b = 0; b < B; ++b) {
    if (int st = check_dims(h, F, T2[b], K)) return st;
    GCCNMF_REQUIRE(h, V[b] && H[b], "klnmf_ragged: NULL V or H of clip %d", b);
    GCCNMF_REQUIRE(h, ld_v[b] >= T2[b], "klnmf_ragged: V pitch %lld < T2 %d of clip %d", (long long)ld_v[b], T2[b], b);
  }
  GCCNMF_REQUIRE(h, iterations >= 0, "klnmf_ragged: iterations must be >= 0 (got %d)", iterations);
  const size_t need = gccnmf_klnmf_ragged_workspace_bytes(B, F, T2, K);
  if (!workspace || workspace_bytes < need) return gccnmf_fail(h, GCCNMF_ERR_WORKSPACE, "klnmf_ragged workspace too small: need %zu bytes", need);
  if (iterations == 0) return GCCNMF_OK;
  char* table = reinterpret_cast<char*>(align_up(reinterpret_cast<uintptr_t>(workspace), 128));
  char* ws = static_cast<char*>(workspace) + ragged_table_bytes(B);
  const int64_t fk = (int64_t)F * K;
  // the clips the tensor-core batch form takes run as one ragged loop; the others one at a time, as gccnmf_klnmf_batched runs them
  std::vector<const float*> tv;
  std::vector<int64_t> tld;
  std::vector<int> tt;
  std::vector<float*> tw, th;
  std::vector<void*> tws;
  for (int b = 0; b < B; ++b) {
    if (use_tc(h, F, T2[b], K) && gccnmf_klnmf_tma_batch_supported(h, F, T2[b], K)) {
      tv.push_back(V[b]); tld.push_back(ld_v[b]); tt.push_back(T2[b]); tw.push_back(W + b * fk); th.push_back(H[b]); tws.push_back(ws);
    } else if (int st = klnmf_one_clip(h, V[b], ld_v[b], F, T2[b], W + b * fk, H[b], K, iterations, sparsity_alpha, epsilon, update_W, ws,
                                       batch_clip_bytes(F, T2[b], K), stream)) {
      return st;
    }
    ws += batch_clip_bytes(F, T2[b], K);
  }
  if (tt.empty()) return GCCNMF_OK;
  return gccnmf_klnmf_tma_ragged(h, (int)tt.size(), tv.data(), tld.data(), tt.data(), tw.data(), th.data(), tws.data(), F, K, iterations, sparsity_alpha,
                                 epsilon, update_W != 0, table, stream);
}

}  // extern "C"
