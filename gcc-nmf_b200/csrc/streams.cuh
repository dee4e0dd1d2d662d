// The per-stream control plane shared by the real-time (rt.cu) and low-latency (lowlatency.cu) engines: the check of a range of
// streams, the sort of the streams by bank entry, the by-value scatter of per-stream integer settings and the capture of one call
// as a CUDA graph.  The engines differ in their per-block kernels; these are the same job in both.
#pragma once
#include <cstring>

#include "common.cuh"

namespace {

// Streams [first, first + count) must be a non-empty range inside [0, S).  `name` names the calling entry in the message.
inline int stream_range_check(gccnmf_handle* h, const char* name, int S, int first, int count) {
  GCCNMF_REQUIRE(h, first >= 0 && count >= 1 && first < S && count <= S - first, "%s: streams [%d, %d + %d) outside [0, %d)", name, first, first,
                 count, S);
  return 0;
}

// ---- sort by entry
constexpr int kStreamMaxEntries = 64;                  // the most entries of any bank of either engine
static_assert(GCCNMF_RTBANK_MAX_ENTRIES <= kStreamMaxEntries && GCCNMF_LLBANK_MAX_STEERINGS <= kStreamMaxEntries &&
                  GCCNMF_LLDICT_MAX_DICTIONARIES <= kStreamMaxEntries,
              "bank entries");

// Stable counting sort of the S streams by entry, by one warp over chunks of 32 streams: stream s's entry in [0, Q) is the int32 at
// assign + s assign_stride bytes; order lists the streams of entry 0 in stream order, then those of entry 1, ...  Inactive streams
// are listed too (the kernels skip them).  Unless seg is NULL, seg[e] is entry e's first position in order and seg[Q] = S.
__global__ void __launch_bounds__(32) sort_by_entry_kernel(const int32_t* __restrict__ assign, size_t assign_stride, int S, int Q,
                                                           int32_t* __restrict__ order, int32_t* __restrict__ seg) {
  __shared__ int base[kStreamMaxEntries];
  const int lane = threadIdx.x;
  for (int i = lane; i < Q; i += 32) base[i] = 0;
  __syncwarp();
  for (int pass = 0; pass < 2; ++pass) {               // 0: count per entry, 1: place
    for (int s0 = 0; s0 < S; s0 += 32) {
      const int s = s0 + lane;
      const int e = s < S ? *reinterpret_cast<const int32_t*>(reinterpret_cast<const char*>(assign) + (size_t)s * assign_stride) : -1;
      const unsigned peers = __match_any_sync(0xffffffffu, e);
      const bool leader = lane == __ffs(peers) - 1;
      if (pass == 1 && e >= 0) order[base[e] + __popc(peers & ((1u << lane) - 1u))] = s;
      __syncwarp();
      if (leader && e >= 0) base[e] += __popc(peers);
      __syncwarp();
    }
    if (pass == 0 && lane == 0)                        // counts -> first positions
      for (int i = 0, sum = 0; i < Q; ++i) {
        const int n = base[i];
        base[i] = sum;
        if (seg) seg[i] = sum;
        sum += n;
      }
    __syncwarp();
  }
  if (seg && lane == 0) seg[Q] = S;
}

// ---- per-stream integers by value: row i of a batch (`width` int32 values) goes to the words at base + (first + i) stride + offset
// bytes.  The host array is consumed when the launch is enqueued, so a batch may be captured into a graph or freed at once.
constexpr int kStreamRowsPerLaunch = 64;
constexpr int kStreamRowsMaxWidth = 8;                 // the most sources of either engine
static_assert(GCCNMF_RTSEP_MAX_SOURCES <= kStreamRowsMaxWidth && GCCNMF_LLSEP_MAX_SOURCES <= kStreamRowsMaxWidth, "sources per row");
struct StreamRows {
  int32_t v[kStreamRowsPerLaunch * kStreamRowsMaxWidth];
};
enum StreamRowsMode { kRowsKeep, kRowsWrite, kRowsFill };   // keep: -1 leaves its word alone; fill: every stream gets row 0

__global__ void stream_rows_kernel(char* __restrict__ base, size_t stride, size_t offset, int first, int count, int width, int mode, StreamRows r) {
  for (int i = threadIdx.x; i < count; i += blockDim.x) {
    int32_t* row = reinterpret_cast<int32_t*>(base + (size_t)(first + i) * stride + offset);
    for (int q = 0; q < width; ++q) {
      const int32_t v = r.v[mode == kRowsFill ? q : i * width + q];
      if (mode != kRowsKeep || v >= 0) row[q] = v;
    }
  }
}

// values[i width + q] (width <= kStreamRowsMaxWidth) to word q of stream first + i's row, one launch per kStreamRowsPerLaunch streams;
// keep: -1 leaves the word as it was, else every value is written, -1 included.
int enqueue_stream_rows(gccnmf_handle* h, void* base, size_t stride, size_t offset, int first, int count, int width, const int32_t* values, bool keep,
                        void* stream) {
  for (int i0 = 0; i0 < count; i0 += kStreamRowsPerLaunch) {
    const int n = count - i0 < kStreamRowsPerLaunch ? count - i0 : kStreamRowsPerLaunch;
    StreamRows r{};
    memcpy(r.v, values + (size_t)i0 * width, (size_t)n * width * sizeof(int32_t));
    GCCNMF_LAUNCH(h, stream_rows_kernel, 1, kStreamRowsPerLaunch, 0, stream, static_cast<char*>(base), stride, offset, first + i0, n, width,
                  keep ? kRowsKeep : kRowsWrite, r);
  }
  return GCCNMF_OK;
}

// `value` to the one-word row of every stream of [first, first + count), in one launch whatever count is.
int enqueue_stream_fill(gccnmf_handle* h, void* base, size_t stride, int first, int count, int32_t value, void* stream) {
  StreamRows r{};
  r.v[0] = value;
  GCCNMF_LAUNCH(h, stream_rows_kernel, 1, 256, 0, stream, static_cast<char*>(base), stride, size_t(0), first, count, 1, kRowsFill, r);
  return GCCNMF_OK;
}

// ---- graph capture: [H2D of in_bytes from in_host to in_dev ->] enqueue() [-> D2H of out_bytes from out_dev to out_host] as one
// CUDA graph, captured on `stream` (not the default stream).  A NULL host pointer leaves its copy out.  enqueue() returns a status;
// on any failure the capture is ended and dropped, and *graph_exec is left alone.
template <typename Enqueue>
int capture_graph(gccnmf_handle* h, const char* name, void* stream, void* in_dev, const void* in_host, size_t in_bytes, const void* out_dev,
                  void* out_host, size_t out_bytes, Enqueue enqueue, void** graph_exec) {
  cudaStream_t s = (cudaStream_t)stream;
  GCCNMF_CHECK_CUDA(h, cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
  int st = GCCNMF_OK;
  if (in_host && cudaMemcpyAsync(in_dev, in_host, in_bytes, cudaMemcpyHostToDevice, s) != cudaSuccess) st = GCCNMF_ERR_CUDA;
  if (st == GCCNMF_OK) st = enqueue();
  if (st == GCCNMF_OK && out_host && cudaMemcpyAsync(out_host, out_dev, out_bytes, cudaMemcpyDeviceToHost, s) != cudaSuccess) st = GCCNMF_ERR_CUDA;
  cudaGraph_t graph = nullptr;
  const cudaError_t end = cudaStreamEndCapture(s, &graph);
  if (st != GCCNMF_OK || end != cudaSuccess) {
    if (graph) cudaGraphDestroy(graph);
    if (st == GCCNMF_OK) return gccnmf_fail(h, GCCNMF_ERR_CUDA, "%s: stream capture failed: %s", name, cudaGetErrorString(end));
    return st;
  }
  cudaGraphExec_t exec = nullptr;
  const cudaError_t inst = cudaGraphInstantiate(&exec, graph, 0);
  cudaGraphDestroy(graph);
  if (inst != cudaSuccess) return gccnmf_fail(h, GCCNMF_ERR_CUDA, "%s: cudaGraphInstantiate failed: %s", name, cudaGetErrorString(inst));
  *graph_exec = exec;
  return GCCNMF_OK;
}

}  // namespace
