// Host side of the TMA-fed plane GEMM (tma_gemm.cuh): tensor maps over bf16 plane pairs (cached in the handle), the launch helper
// (programmatic dependent launch + cluster dimensions), one launcher per template instantiation with its per-device attribute /
// occupancy cache, the cluster-shape policy, and the epilogue helpers (hi/lo split of 4 consecutive values, guarded vector access).
// Included by klnmf_tma.cu (the four contractions of a KL-NMF iteration) and gcc_tc.cu (all-TDOA argmax GEMM, masked reconstruction).
#pragma once
#include <algorithm>
#include <mutex>
#include <utility>
#include <vector>

#include "common.cuh"
#include "tma_gemm.cuh"

namespace tgemm_host {

using tgemm::PlaneGemmArgs;
using tgemm::split_bf16;
typedef __nv_bfloat16 bf16;

constexpr int kKB = 32;              // k-block: 64-byte K-major rows (SWIZZLE_64B), 32 k-rows per MN-major atom
constexpr int kTailRowsMax = 8;
constexpr int kMaxSplits = 8;

// ------------------------------------------------------------------------------------------------ tensor maps
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline EncodeTiledFn encode_tiled_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

struct TmapKey {
  const void* base;
  uint64_t inner, rows, pitch_bytes, plane_bytes;
  uint32_t box_inner, box_rows, box_planes;
  uint64_t clips, clip_bytes;     // clips > 0: a fourth, clip dimension (batched launches, tgemm::Clips)
  bool operator==(const TmapKey& o) const {
    return base == o.base && inner == o.inner && rows == o.rows && pitch_bytes == o.pitch_bytes && plane_bytes == o.plane_bytes &&
           box_inner == o.box_inner && box_rows == o.box_rows && box_planes == o.box_planes && clips == o.clips && clip_bytes == o.clip_bytes;
  }
};

}  // namespace tgemm_host

struct gccnmf_tmap_cache {
  std::vector<std::pair<tgemm_host::TmapKey, CUtensorMap>> entries;
};

namespace tgemm_host {

// Tensor map over a plane pair [2][rows][pitch] of bf16: dims (inner, rows, 2), box (box_inner, box_rows, box_planes).
// box_inner * 2 bytes = 64 -> SWIZZLE_64B (K-major k-blocks of 32), 128 -> SWIZZLE_128B (MN-major atoms of 64).
// clips > 0: `clips` such pairs clip_bytes apart, dims (inner, rows, 2, clips), box of one clip.
// encode_tmap encodes the map of `key` (byte strides); get_tmap looks it up in the handle's cache first.
inline int encode_tmap(gccnmf_handle* h, const TmapKey& key, CUtensorMap* out) {
  EncodeTiledFn encode = encode_tiled_fn();
  if (!encode) return gccnmf_fail(h, GCCNMF_ERR_CUDA, "cuTensorMapEncodeTiled is not available from the driver");
  if ((reinterpret_cast<uintptr_t>(key.base) & 15) || (key.pitch_bytes & 15) || (key.plane_bytes & 15) || (key.clip_bytes & 15))
    return gccnmf_fail(h, GCCNMF_ERR_INVALID_ARGUMENT, "tensor map: base / pitch / plane / clip stride must be 16-byte aligned");
  const cuuint64_t dims[4] = {key.inner, key.rows, 2, key.clips};
  const cuuint64_t strides[3] = {key.pitch_bytes, key.plane_bytes, key.clip_bytes};
  const cuuint32_t box[4] = {key.box_inner, key.box_rows, key.box_planes, 1};
  const cuuint32_t elem_strides[4] = {1, 1, 1, 1};
  const CUtensorMapSwizzle swz = (key.box_inner * 2 == 128) ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
  const CUresult r = encode(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, key.clips ? 4 : 3, const_cast<void*>(key.base), dims, strides, box, elem_strides,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return gccnmf_fail(h, GCCNMF_ERR_CUDA, "cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
  return 0;
}

inline int get_tmap(gccnmf_handle* h, const bf16* base, uint64_t inner, uint64_t rows, uint64_t pitch_elems, uint64_t plane_elems,
             uint32_t box_inner, uint32_t box_rows, uint32_t box_planes, CUtensorMap* out, uint64_t clips = 0, uint64_t clip_bytes = 0) {
  if (!h->tmaps) h->tmaps = new gccnmf_tmap_cache();
  const TmapKey key{base, inner, rows, pitch_elems * 2, plane_elems * 2, box_inner, box_rows, box_planes, clips, clips ? clip_bytes : 0};
  for (auto& e : h->tmaps->entries)
    if (e.first == key) { *out = e.second; return 0; }
  CUtensorMap m;
  if (int st = encode_tmap(h, key, &m)) return st;
  if (h->tmaps->entries.size() > 256) h->tmaps->entries.clear();
  h->tmaps->entries.emplace_back(key, m);
  *out = m;
  return 0;
}

// float32 matrix of `cols` rows of `inner` elements (pitch in elements), one box = box_inner x box_rows, no swizzle: the
// epilogue operand tile of a plane GEMM (tgemm::wants_smem_operand).
inline int tmap_f32_2d(gccnmf_handle* h, const float* base, uint64_t inner, uint64_t rows, uint64_t pitch_elems, uint32_t box_inner,
                       uint32_t box_rows, CUtensorMap* out) {
  if (!h->tmaps) h->tmaps = new gccnmf_tmap_cache();
  const TmapKey key{base, inner, rows, pitch_elems * 4, 0, box_inner, box_rows, 0, 0, 0};     // (box_planes = 0: not a plane pair)
  for (auto& e : h->tmaps->entries)
    if (e.first == key) { *out = e.second; return 0; }
  EncodeTiledFn encode = encode_tiled_fn();
  if (!encode) return gccnmf_fail(h, GCCNMF_ERR_CUDA, "cuTensorMapEncodeTiled is not available from the driver");
  if ((reinterpret_cast<uintptr_t>(base) & 15) || (key.pitch_bytes & 15))
    return gccnmf_fail(h, GCCNMF_ERR_INVALID_ARGUMENT, "tensor map: base / pitch must be 16-byte aligned");
  const cuuint64_t dims[2] = {inner, rows};
  const cuuint64_t strides[1] = {key.pitch_bytes};
  const cuuint32_t box[2] = {box_inner, box_rows};
  const cuuint32_t elem_strides[2] = {1, 1};
  CUtensorMap m;
  const CUresult r = encode(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), dims, strides, box, elem_strides,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return gccnmf_fail(h, GCCNMF_ERR_CUDA, "cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
  if (h->tmaps->entries.size() > 256) h->tmaps->entries.clear();
  h->tmaps->entries.emplace_back(key, m);
  *out = m;
  return 0;
}

// K-major operand: rows x kc, k contiguous; one box = one plane of a row slice (box_rows = tile rows / cluster extent).
inline int tmap_kmajor(gccnmf_handle* h, const bf16* planes, int rows, int kc, int64_t pitch, int64_t plane, int box_rows, CUtensorMap* out,
                       int clips = 0, int64_t clip_bytes = 0) {
  return get_tmap(h, planes, (uint64_t)kc, (uint64_t)rows, (uint64_t)pitch, (uint64_t)plane, kKB, (uint32_t)box_rows, 1, out, clips, clip_bytes);
}
// MN-major operand: stored as kc rows x mn contiguous; one box = one 64-wide atom, both planes.
inline int tmap_mnmajor(gccnmf_handle* h, const bf16* planes, int mn, int kc, int64_t pitch, int64_t plane, CUtensorMap* out,
                        int clips = 0, int64_t clip_bytes = 0) {
  return get_tmap(h, planes, (uint64_t)mn, (uint64_t)kc, (uint64_t)pitch, (uint64_t)plane, 64, kKB, 2, out, clips, clip_bytes);
}

// ------------------------------------------------------------------------------------------------ launch helper
template <class... KArgs, class... Args>
int launch_ex(gccnmf_handle* h, const char* name, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, void* stream, bool pdl,
              dim3 cluster, Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = (cudaStream_t)stream;
  cudaLaunchAttribute attr[3];
  int n = 0;
  if (h->l2_window_bytes > 0) {          // KL-NMF loop: keep G^T resident in L2 (set by gccnmf_klnmf_tma_l2_window)
    attr[n].id = cudaLaunchAttributeAccessPolicyWindow;
    attr[n].val.accessPolicyWindow.base_ptr = const_cast<void*>(h->l2_window_base);
    attr[n].val.accessPolicyWindow.num_bytes = h->l2_window_bytes;
    attr[n].val.accessPolicyWindow.hitRatio = 1.0f;
    attr[n].val.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
    attr[n].val.accessPolicyWindow.missProp = cudaAccessPropertyNormal;
    ++n;
  }
  if (pdl) {
    attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[n].val.programmaticStreamSerializationAllowed = 1;
    ++n;
  }
  if (cluster.x * cluster.y * cluster.z > 1) {
    attr[n].id = cudaLaunchAttributeClusterDimension;
    attr[n].val.clusterDim.x = cluster.x;
    attr[n].val.clusterDim.y = cluster.y;
    attr[n].val.clusterDim.z = cluster.z;
    ++n;
  }
  cfg.attrs = attr;
  cfg.numAttrs = n;
  const cudaError_t err = cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
  if (err != cudaSuccess) return gccnmf_fail(h, GCCNMF_ERR_CUDA, "launch of %s failed: %s", name, cudaGetErrorString(err));
  h->launches++;
  return 0;
}

// ------------------------------------------------------------------------------------------------ epilogue helpers
__device__ __forceinline__ uint32_t bf162_bits(__nv_bfloat162 v) { return *reinterpret_cast<uint32_t*>(&v); }
// four consecutive values -> 4 hi + 4 lo bf16, packed in element order
__device__ __forceinline__ void split4(const float4& x, uint2& hi, uint2& lo) {
  const __nv_bfloat162 h01 = __floats2bfloat162_rn(x.x, x.y), h23 = __floats2bfloat162_rn(x.z, x.w);
  const float2 f01 = __bfloat1622float2(h01), f23 = __bfloat1622float2(h23);
  hi = make_uint2(bf162_bits(h01), bf162_bits(h23));
  lo = make_uint2(bf162_bits(__floats2bfloat162_rn(x.x - f01.x, x.y - f01.y)), bf162_bits(__floats2bfloat162_rn(x.z - f23.x, x.w - f23.y)));
}
__device__ __forceinline__ void store_planes4(bf16* hi_ptr, int64_t plane, const float4& x, int valid, bool vec) {
  uint2 hi, lo;
  split4(x, hi, lo);
  if (vec && valid == 4) {
    *reinterpret_cast<uint2*>(hi_ptr) = hi;
    *reinterpret_cast<uint2*>(hi_ptr + plane) = lo;
  } else {
    const uint32_t hw[2] = {hi.x, hi.y}, lw[2] = {lo.x, lo.y};
#pragma unroll
    for (int i = 0; i < 4; ++i)
      if (i < valid) {
        reinterpret_cast<uint16_t*>(hi_ptr)[i] = (uint16_t)(hw[i >> 1] >> (16 * (i & 1)));
        reinterpret_cast<uint16_t*>(hi_ptr + plane)[i] = (uint16_t)(lw[i >> 1] >> (16 * (i & 1)));
      }
  }
}
__device__ __forceinline__ float4 load4(const float* p, int valid, bool vec, float fill) {
  if (vec && valid == 4) return *reinterpret_cast<const float4*>(p);
  float4 r = make_float4(fill, fill, fill, fill);
  if (valid > 0) r.x = p[0];
  if (valid > 1) r.y = p[1];
  if (valid > 2) r.z = p[2];
  if (valid > 3) r.w = p[3];
  return r;
}
// streaming variant (st.global.cs): data that is written once and read once by the next kernel (the k-split partials of the
// W-update numerator, 12.6 MB per iteration) should not push the H^T master and planes out of the L2
__device__ __forceinline__ void store4_streaming(float* p, const float4& v, int valid, bool vec) {
  if (vec && valid == 4) { __stcs(reinterpret_cast<float4*>(p), v); return; }
  if (valid > 0) __stcs(p, v.x);
  if (valid > 1) __stcs(p + 1, v.y);
  if (valid > 2) __stcs(p + 2, v.z);
  if (valid > 3) __stcs(p + 3, v.w);
}
__device__ __forceinline__ void store4(float* p, const float4& v, int valid, bool vec) {
  if (vec && valid == 4) { *reinterpret_cast<float4*>(p) = v; return; }
  if (valid > 0) p[0] = v.x;
  if (valid > 1) p[1] = v.y;
  if (valid > 2) p[2] = v.z;
  if (valid > 3) p[3] = v.w;
}

// ------------------------------------------------------------------------------------------------ GEMM launch
struct Operand {
  const bf16* planes;      // hi plane; lo at + plane
  int64_t pitch, plane;    // elements
  bool mn_major;           // false: (rows, kc) k contiguous; true: (kc, rows) rows contiguous
};

struct GemmShape {
  int M, N, Kc, splits, m_tiles, n_tiles, tail_rows;
  bool m_fastest;       // grid (m tiles, n tiles, splits): see PlaneGemmArgs
  int z_cluster;        // > 1: the k-splits of a tile form a (1, 1, splits) cluster and are summed through distributed shared memory
  unsigned* done_counter;          // completion signal of the launch to the ranks of a sharded run (see tgemm::PeerSignal)
  tgemm::PeerSignal signal;
  int clips;                       // > 0: batched launch over `clips` clips clip_bytes apart (tgemm::Clips)
  int64_t clip_bytes;
};

// One instantiation: kernel attributes + how many of its clusters can be resident at once (queried once).
template <int BN, bool A_MN, bool B_MN, int CN, int CM, class Epi>
struct PlaneGemmInstance {
  static constexpr bool kDual = tgemm::wants_dual_n<Epi>::value && !B_MN && 2 * BN <= 256;
  using C = tgemm::Config<BN, kKB, A_MN, B_MN, kDual ? 2 : 1, tgemm::wants_smem_operand<Epi>::value && !tgemm::has_tile_epilogue<Epi>::value>;
  static int max_clusters(gccnmf_handle* h, int* out) {
    static int cached_per_device[kGccnmfMaxDevices];     // 0 = not queried yet, else value + 1 (per device: attribute + occupancy)
    int& slot = cached_per_device[h->device % kGccnmfMaxDevices];
    int cached = slot - 1;
    if (cached < 0) {
      auto kernel = tgemm::plane_gemm_kernel<BN, kKB, A_MN, B_MN, CN, CM, Epi>;
      GCCNMF_CHECK_CUDA(h, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, C::kTotal));
      if (CN * CM == 1) {
        cached = h->sm_count;
      } else {
        cudaLaunchConfig_t cfg{};
        cfg.gridDim = dim3(CN * 64, CM * 64, 1);      // (the m-fastest orientation has the same occupancy)
        cfg.blockDim = dim3(tgemm::kThreads);
        cfg.dynamicSmemBytes = C::kTotal;
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeClusterDimension;
        attr[0].val.clusterDim.x = CN; attr[0].val.clusterDim.y = CM; attr[0].val.clusterDim.z = 1;
        cfg.attrs = attr;
        cfg.numAttrs = 1;
        int n = 0;
        GCCNMF_CHECK_CUDA(h, cudaOccupancyMaxActiveClusters(&n, kernel, &cfg));
        cached = n;
      }
      slot = cached + 1;
    }
    *out = cached;
    return 0;
  }
  // How many (1, 1, S) clusters of this kernel (k-splits summed through distributed shared memory) can be resident at once.
  static int max_z_clusters(gccnmf_handle* h, int S, int* out) {
    static int cached_per_device[kGccnmfMaxDevices][9];
    if (S < 2 || S > 8 || CN * CM != 1) { *out = 0; return 0; }
    int& slot = cached_per_device[h->device % kGccnmfMaxDevices][S];
    if (slot == 0) {
      int unused;
      if (int st = max_clusters(h, &unused)) return st;     // (sets the shared-memory attribute)
      auto kernel = tgemm::plane_gemm_kernel<BN, kKB, A_MN, B_MN, CN, CM, Epi>;
      cudaLaunchConfig_t cfg{};
      cfg.gridDim = dim3(16, 16, S);
      cfg.blockDim = dim3(tgemm::kThreads);
      cfg.dynamicSmemBytes = C::kTotal;
      cudaLaunchAttribute attr[1];
      attr[0].id = cudaLaunchAttributeClusterDimension;
      attr[0].val.clusterDim.x = 1; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = S;
      cfg.attrs = attr;
      cfg.numAttrs = 1;
      int n = 0;
      const cudaError_t err = cudaOccupancyMaxActiveClusters(&n, kernel, &cfg);
      if (err != cudaSuccess) { (void)cudaGetLastError(); n = 0; }     // cluster shape not launchable: the caller keeps the slabs
      slot = n + 1;
    }
    *out = slot - 1;
    return 0;
  }
  static int launch(gccnmf_handle* h, const Operand& A, const Operand& B, const GemmShape& g, const Epi& epi, unsigned long long* timing, void* stream) {
    auto kernel = tgemm::plane_gemm_kernel<BN, kKB, A_MN, B_MN, CN, CM, Epi>;
    int unused;
    if (int st = max_clusters(h, &unused)) return st;     // (sets the shared-memory attribute on first use)
    CUtensorMap map_a, map_b;
    if (int st = A_MN ? tmap_mnmajor(h, A.planes, g.M, g.Kc, A.pitch, A.plane, &map_a, g.clips, g.clip_bytes)
                      : tmap_kmajor(h, A.planes, g.M, g.Kc, A.pitch, A.plane, tgemm::kBM / CN, &map_a, g.clips, g.clip_bytes)) return st;
    if (int st = B_MN ? tmap_mnmajor(h, B.planes, g.N, g.Kc, B.pitch, B.plane, &map_b, g.clips, g.clip_bytes)
                      : tmap_kmajor(h, B.planes, g.N, g.Kc, B.pitch, B.plane, BN / CM, &map_b, g.clips, g.clip_bytes)) return st;
    Epi e = epi;
    if constexpr (C::kOperandBytes > 0)
      if (int st = tmap_f32_2d(h, e.operand(), (uint64_t)e.operand_ld(), (uint64_t)e.operand_cols(), (uint64_t)e.operand_ld(), tgemm::kBM, BN,
                               &e.operand_map)) return st;
    PlaneGemmArgs args{};
    args.M = g.M; args.N = g.N; args.Kc = g.Kc;
    args.m_tiles = g.m_tiles;
    args.tail_rows = g.tail_rows;
    args.tail_cols = (((BN + g.m_tiles - 1) / g.m_tiles) + 1) & ~1;
    const int total_kb = (g.Kc + kKB - 1) / kKB;
    args.kblocks_per_split = (total_kb + g.splits - 1) / g.splits;
    args.A = A.planes; args.a_plane = A.plane; args.lda = A.pitch;
    args.B = B.planes; args.b_plane = B.plane; args.ldb = B.pitch;
    args.timing = timing;
    args.preload = (g.z_cluster > 1) ? 0 : (h->gemm_preload & 1);     // (only epilogues that opt in with kPreloadOperands have the code)
    const bool mf = g.m_fastest;      // grid (m tiles, n tiles, splits)
    args.m_fastest = mf ? 1 : 0;
    args.z_cluster = (CN * CM == 1 && g.z_cluster > 1) ? g.z_cluster : 0;
    args.done_counter = g.done_counter;
    args.signal = g.signal;
    const int zs = g.splits * std::max(1, g.clips);     // (batched: blockIdx.z = clip * splits + split)
    const dim3 grid = mf ? dim3(g.m_tiles, g.n_tiles, zs) : dim3(g.n_tiles, g.m_tiles, zs);
    if (!timing && h->debug_timing) {   // diagnostics: every plane GEMM of the KL-NMF loop appends its CTA stamps (8 per CTA)
      args.timing = h->debug_timing + h->debug_timing_cursor;
      h->debug_timing_cursor += (size_t)grid.x * grid.y * grid.z * 8;
    }
    return launch_ex(h, "plane_gemm_kernel", kernel, grid, dim3(tgemm::kThreads), (size_t)C::kTotal, stream, h->nmf_pdl,
                     args.z_cluster > 1 ? dim3(1, 1, args.z_cluster) : (mf ? dim3(CM, 1, 1) : dim3(CN, CM, 1)), map_a, map_b, args, e);
  }
};

// Cluster shape (CN n tiles x CM m tiles share operand slices by TMA multicast): the largest of 2x2, then the pair that
// shares the larger operand tile, that divides the grid and whose clusters are all resident in one wave (when the
// single-CTA grid is); h->gemm_cluster (diagnostics) forces 10 CN + CM.
template <int BN, bool A_MN, bool B_MN, class Epi>
int launch_plane_gemm(gccnmf_handle* h, const Operand& A, const Operand& B, int M, int N, int Kc, int splits, bool simt_tail,
                      const Epi& epi, unsigned long long* timing, void* stream, bool m_fastest = false, bool prefer_pair = false) {
  GemmShape g{};
  g.M = M; g.N = N; g.Kc = Kc; g.splits = splits; g.m_fastest = m_fastest;
  const int tail = M % tgemm::kBM;
  // (the m tiles of an n tile share its columns for the tail rows: at most 128 columns per CTA)
  const bool use_tail = simt_tail && !A_MN && !B_MN && tail != 0 && tail <= kTailRowsMax && M > tgemm::kBM && (M / tgemm::kBM) * 128 >= BN;
  g.m_tiles = use_tail ? M / tgemm::kBM : (M + tgemm::kBM - 1) / tgemm::kBM;
  g.tail_rows = use_tail ? tail : 0;
  g.n_tiles = (N + BN - 1) / BN;
  const int ctas = g.n_tiles * g.m_tiles * splits;
  // CTA pairs (option gemm_pair: -1 where the call site asks for them, 1 wherever the shape allows, 0 never): two m tiles share
  // the B tile through a 1 x 2 cluster, each CTA loading half of it and multicasting it to both.  The KL-NMF contractions do not
  // ask for them: on an H100 SXM their main loops run faster alone (tools/nmf_phases.py, DESIGN.md 4.1).
  const bool pair = h->gemm_pair > 0 || (h->gemm_pair < 0 && prefer_pair);
  const int order_share_b[4][2] = {{1, 2}, {1, 1}, {1, 1}, {1, 1}}, order_none[4][2] = {{1, 1}, {1, 1}, {1, 1}, {1, 1}};
  const int order_forced[4][2] = {{2, 2}, {1, 2}, {2, 1}, {1, 1}};
  const int (*order)[2] = h->gemm_cluster >= 0 ? order_forced : (pair ? order_share_b : order_none);
  for (int i = 0; i < 4; ++i) {
    const int cn = order[i][0], cm = order[i][1];
    if (h->gemm_cluster >= 0 && h->gemm_cluster != 10 * cn + cm && !(cn == 1 && cm == 1)) continue;
    if (g.n_tiles % cn != 0 || g.m_tiles % cm != 0) continue;
    if (m_fastest && cn != 1) continue;
    int resident = 0;
#define GCCNMF_TRY_CLUSTER(CN_, CM_)                                                                                         \
    if constexpr (B_MN || (BN / CM_) % 8 == 0) /* the B row slices of a CM-row cluster keep whole swizzle atoms */              \
    if (cn == CN_ && cm == CM_) {                                                                                            \
      if (int st = PlaneGemmInstance<BN, A_MN, B_MN, CN_, CM_, Epi>::max_clusters(h, &resident)) return st;                  \
      /* a single-wave grid must keep all its clusters resident at once; a multi-wave grid only needs one to fit */            \
      if (cn * cm == 1 || (resident > 0 && (ctas > h->sm_count || resident * cn * cm >= ctas)))                                \
          return PlaneGemmInstance<BN, A_MN, B_MN, CN_, CM_, Epi>::launch(h, A, B, g, epi, timing, stream);                  \
    }
    GCCNMF_TRY_CLUSTER(2, 2)
    GCCNMF_TRY_CLUSTER(1, 2)
    GCCNMF_TRY_CLUSTER(2, 1)
    GCCNMF_TRY_CLUSTER(1, 1)
#undef GCCNMF_TRY_CLUSTER
  }
  return gccnmf_fail(h, GCCNMF_ERR_UNSUPPORTED, "plane gemm: no launchable cluster shape");
}

template <bool A_MN, bool B_MN, class Epi>
int plane_gemm(gccnmf_handle* h, int bn, const Operand& A, const Operand& B, int M, int N, int Kc, int splits, bool simt_tail, const Epi& epi,
               unsigned long long* timing, void* stream, bool m_fastest = false, bool prefer_pair = false) {
  switch (bn) {
    case 104:      // only as a dual-N tile (MMAs of 104 + 208 columns per k-step; 104 alone is not a multiple of 16)
      if constexpr (tgemm::wants_dual_n<Epi>::value && !B_MN)
        return launch_plane_gemm<104, A_MN, B_MN>(h, A, B, M, N, Kc, splits, simt_tail, epi, timing, stream, m_fastest, prefer_pair);
      break;
    case 120:      // only as a dual-N tile (MMAs of 120 + 240 columns per k-step): the planner offers it to the W.H contractions only
      if constexpr (tgemm::wants_dual_n<Epi>::value && !B_MN)
        return launch_plane_gemm<120, A_MN, B_MN>(h, A, B, M, N, Kc, splits, simt_tail, epi, timing, stream, m_fastest, prefer_pair);
      break;
    case 112: return launch_plane_gemm<112, A_MN, B_MN>(h, A, B, M, N, Kc, splits, simt_tail, epi, timing, stream, m_fastest, prefer_pair);
    case 128: return launch_plane_gemm<128, A_MN, B_MN>(h, A, B, M, N, Kc, splits, simt_tail, epi, timing, stream, m_fastest, prefer_pair);
    case 176: return launch_plane_gemm<176, A_MN, B_MN>(h, A, B, M, N, Kc, splits, simt_tail, epi, timing, stream, m_fastest, prefer_pair);
    case 208: return launch_plane_gemm<208, A_MN, B_MN>(h, A, B, M, N, Kc, splits, simt_tail, epi, timing, stream, m_fastest, prefer_pair);
    case 240: return launch_plane_gemm<240, A_MN, B_MN>(h, A, B, M, N, Kc, splits, simt_tail, epi, timing, stream, m_fastest, prefer_pair);
    case 256: return launch_plane_gemm<256, A_MN, B_MN>(h, A, B, M, N, Kc, splits, simt_tail, epi, timing, stream, m_fastest, prefer_pair);
  }
  return gccnmf_fail(h, GCCNMF_ERR_UNSUPPORTED, "plane gemm: tile width %d (supported: 104, 112, 120, 128, 176, 208, 240, 256)", bn);
}

// Batched launch (tgemm::Clips) over `clips` clips of one shape, 1 x 1 clusters, k-splits as slabs: the tile plan, tail rows and
// k-split ranges of every clip are those of launch_plane_gemm on that clip alone.
template <int BN, bool A_MN, bool B_MN, class Epi>
int launch_plane_gemm_clips(gccnmf_handle* h, const Operand& A, const Operand& B, int M, int N, int Kc, int splits, bool simt_tail,
                            const tgemm::Clips<Epi>& epi, int clips, void* stream) {
  GemmShape g{};
  g.M = M; g.N = N; g.Kc = Kc; g.splits = splits;
  const int tail = M % tgemm::kBM;
  const bool use_tail = simt_tail && !A_MN && !B_MN && tail != 0 && tail <= kTailRowsMax && M > tgemm::kBM && (M / tgemm::kBM) * 128 >= BN;
  g.m_tiles = use_tail ? M / tgemm::kBM : (M + tgemm::kBM - 1) / tgemm::kBM;
  g.tail_rows = use_tail ? tail : 0;
  g.n_tiles = (N + BN - 1) / BN;
  g.clips = clips;
  g.clip_bytes = epi.clip_bytes;
  return PlaneGemmInstance<BN, A_MN, B_MN, 1, 1, tgemm::Clips<Epi>>::launch(h, A, B, g, epi, nullptr, stream);
}
template <bool A_MN, bool B_MN, class Epi>
int plane_gemm_clips(gccnmf_handle* h, int bn, const Operand& A, const Operand& B, int M, int N, int Kc, int splits, bool simt_tail,
                     const tgemm::Clips<Epi>& epi, int clips, void* stream) {
  switch (bn) {
    case 104:
      if constexpr (tgemm::wants_dual_n<Epi>::value && !B_MN) return launch_plane_gemm_clips<104, A_MN, B_MN>(h, A, B, M, N, Kc, splits, simt_tail, epi, clips, stream);
      break;
    case 120:
      if constexpr (tgemm::wants_dual_n<Epi>::value && !B_MN) return launch_plane_gemm_clips<120, A_MN, B_MN>(h, A, B, M, N, Kc, splits, simt_tail, epi, clips, stream);
      break;
    case 112: return launch_plane_gemm_clips<112, A_MN, B_MN>(h, A, B, M, N, Kc, splits, simt_tail, epi, clips, stream);
    case 128: return launch_plane_gemm_clips<128, A_MN, B_MN>(h, A, B, M, N, Kc, splits, simt_tail, epi, clips, stream);
    case 176: return launch_plane_gemm_clips<176, A_MN, B_MN>(h, A, B, M, N, Kc, splits, simt_tail, epi, clips, stream);
    case 208: return launch_plane_gemm_clips<208, A_MN, B_MN>(h, A, B, M, N, Kc, splits, simt_tail, epi, clips, stream);
    case 240: return launch_plane_gemm_clips<240, A_MN, B_MN>(h, A, B, M, N, Kc, splits, simt_tail, epi, clips, stream);
    case 256: return launch_plane_gemm_clips<256, A_MN, B_MN>(h, A, B, M, N, Kc, splits, simt_tail, epi, clips, stream);
  }
  return gccnmf_fail(h, GCCNMF_ERR_UNSUPPORTED, "plane gemm (batched): tile width %d", bn);
}

// Ragged launches (tgemm::Ragged).  ragged_maps encodes the two operand maps of one clip as launch() encodes them for a 1 x 1
// cluster of `bn`-column tiles, with the clip's own extents; the caller copies them into the launch's table.
template <bool A_MN, bool B_MN>
int ragged_maps(gccnmf_handle* h, const Operand& A, const Operand& B, int M, int N, int Kc, int bn, CUtensorMap* out) {
  auto key = [](const Operand& o, bool mn, int rows, int kc, uint32_t box_rows) {
    return mn ? TmapKey{o.planes, (uint64_t)rows, (uint64_t)kc, (uint64_t)o.pitch * 2, (uint64_t)o.plane * 2, 64, kKB, 2, 0, 0}
              : TmapKey{o.planes, (uint64_t)kc, (uint64_t)rows, (uint64_t)o.pitch * 2, (uint64_t)o.plane * 2, kKB, box_rows, 1, 0, 0};
  };
  if (int st = encode_tmap(h, key(A, A_MN, M, Kc, tgemm::kBM), &out[0])) return st;
  return encode_tmap(h, key(B, B_MN, N, Kc, (uint32_t)bn), &out[1]);
}
// One launch of `bn`-column tiles over the clips of epi.tiles (ctas = the sum of their tiles x splits); M, the SIMT tail rule and
// the tail operands' row pitches are the launch's.
template <int BN, bool A_MN, bool B_MN, class Epi>
int launch_plane_gemm_ragged(gccnmf_handle* h, int M, int ctas, bool simt_tail, int64_t lda, int64_t ldb, const tgemm::Ragged<Epi>& epi, void* stream) {
  using I = PlaneGemmInstance<BN, A_MN, B_MN, 1, 1, tgemm::Ragged<Epi>>;
  int unused;
  if (int st = I::max_clusters(h, &unused)) return st;     // (sets the shared-memory attribute on first use)
  const int tail = M % tgemm::kBM;
  const bool use_tail = simt_tail && !A_MN && !B_MN && tail != 0 && tail <= kTailRowsMax && M > tgemm::kBM && (M / tgemm::kBM) * 128 >= BN;
  PlaneGemmArgs args{};
  args.M = M;
  args.m_tiles = use_tail ? M / tgemm::kBM : (M + tgemm::kBM - 1) / tgemm::kBM;
  args.tail_rows = use_tail ? tail : 0;
  args.tail_cols = (((BN + args.m_tiles - 1) / args.m_tiles) + 1) & ~1;
  args.lda = lda;
  args.ldb = ldb;
  args.preload = h->gemm_preload & 1;
  const CUtensorMap none{};         // (the maps come from the table)
  return launch_ex(h, "plane_gemm_kernel", tgemm::plane_gemm_kernel<BN, kKB, A_MN, B_MN, 1, 1, tgemm::Ragged<Epi>>, dim3(ctas), dim3(tgemm::kThreads),
                   (size_t)I::C::kTotal, stream, h->nmf_pdl, dim3(1, 1, 1), none, none, args, epi);
}
template <bool A_MN, bool B_MN, class Epi>
int plane_gemm_ragged(gccnmf_handle* h, int bn, int M, int ctas, bool simt_tail, int64_t lda, int64_t ldb, const tgemm::Ragged<Epi>& epi, void* stream) {
  switch (bn) {
    case 104:
      if constexpr (tgemm::wants_dual_n<Epi>::value && !B_MN) return launch_plane_gemm_ragged<104, A_MN, B_MN>(h, M, ctas, simt_tail, lda, ldb, epi, stream);
      break;
    case 120:
      if constexpr (tgemm::wants_dual_n<Epi>::value && !B_MN) return launch_plane_gemm_ragged<120, A_MN, B_MN>(h, M, ctas, simt_tail, lda, ldb, epi, stream);
      break;
    case 112: return launch_plane_gemm_ragged<112, A_MN, B_MN>(h, M, ctas, simt_tail, lda, ldb, epi, stream);
    case 128: return launch_plane_gemm_ragged<128, A_MN, B_MN>(h, M, ctas, simt_tail, lda, ldb, epi, stream);
    case 176: return launch_plane_gemm_ragged<176, A_MN, B_MN>(h, M, ctas, simt_tail, lda, ldb, epi, stream);
    case 208: return launch_plane_gemm_ragged<208, A_MN, B_MN>(h, M, ctas, simt_tail, lda, ldb, epi, stream);
    case 240: return launch_plane_gemm_ragged<240, A_MN, B_MN>(h, M, ctas, simt_tail, lda, ldb, epi, stream);
    case 256: return launch_plane_gemm_ragged<256, A_MN, B_MN>(h, M, ctas, simt_tail, lda, ldb, epi, stream);
  }
  return gccnmf_fail(h, GCCNMF_ERR_UNSUPPORTED, "plane gemm (ragged): tile width %d", bn);
}

// k-splits reduced inside (1, 1, splits) clusters (no slabs): query how many such clusters are resident at once / launch.
template <bool A_MN, bool B_MN, class Epi>
int plane_gemm_z_clusters(gccnmf_handle* h, int bn, int splits, int* out) {
  switch (bn) {
    case 128: return PlaneGemmInstance<128, A_MN, B_MN, 1, 1, Epi>::max_z_clusters(h, splits, out);
    case 176: return PlaneGemmInstance<176, A_MN, B_MN, 1, 1, Epi>::max_z_clusters(h, splits, out);
    case 208: return PlaneGemmInstance<208, A_MN, B_MN, 1, 1, Epi>::max_z_clusters(h, splits, out);
    case 256: return PlaneGemmInstance<256, A_MN, B_MN, 1, 1, Epi>::max_z_clusters(h, splits, out);
  }
  *out = 0;
  return 0;
}
template <bool A_MN, bool B_MN, class Epi>
int plane_gemm_z_reduce(gccnmf_handle* h, int bn, const Operand& A, const Operand& B, int M, int N, int Kc, int splits, const Epi& epi,
                        unsigned long long* timing, void* stream, unsigned* done_counter = nullptr, const tgemm::PeerSignal* signal = nullptr,
                        bool simt_tail = false) {
  GemmShape g{};
  g.M = M; g.N = N; g.Kc = Kc; g.splits = splits; g.m_fastest = false; g.z_cluster = splits;
  if (signal && signal->world > 0) { g.done_counter = done_counter; g.signal = *signal; }
  const int tail = M % tgemm::kBM;
  const bool use_tail = simt_tail && !A_MN && !B_MN && tail != 0 && tail <= kTailRowsMax && M > tgemm::kBM && (M / tgemm::kBM) * 128 >= bn;
  g.m_tiles = use_tail ? M / tgemm::kBM : (M + tgemm::kBM - 1) / tgemm::kBM;
  g.tail_rows = use_tail ? tail : 0;
  g.n_tiles = (N + bn - 1) / bn;
  switch (bn) {
    case 128: return PlaneGemmInstance<128, A_MN, B_MN, 1, 1, Epi>::launch(h, A, B, g, epi, timing, stream);
    case 176: return PlaneGemmInstance<176, A_MN, B_MN, 1, 1, Epi>::launch(h, A, B, g, epi, timing, stream);
    case 208: return PlaneGemmInstance<208, A_MN, B_MN, 1, 1, Epi>::launch(h, A, B, g, epi, timing, stream);
    case 256: return PlaneGemmInstance<256, A_MN, B_MN, 1, 1, Epi>::launch(h, A, B, g, epi, timing, stream);
  }
  return gccnmf_fail(h, GCCNMF_ERR_UNSUPPORTED, "plane gemm (cluster-reduced k-splits): tile width %d", bn);
}

}  // namespace tgemm_host
