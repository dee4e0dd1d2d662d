// Stream records, shared by the real-time (rt.cu) and low-latency (lowlatency.cu) engines: the list of a stream's state regions, the
// kernel body that copies them between the state and a staging record, the content digest (GCCNMF_RTREC_DIGEST_*) and the host
// checks of a record's header.  An engine form gets records by listing its regions and digest items; the copy, digest and checks
// are these.
#pragma once
#include <cstddef>

#include "common.cuh"

namespace {

// ---- regions: stream s's bytes of region g are [offset + s stride, + bytes) of the state; they go to [rec_offset, + bytes) of the
// stream's record payload, and [rec_offset + bytes, rec_offset + span) of the payload is zero.
struct RecordRegion { size_t offset, stride, rec_offset, bytes, span; };
constexpr int kRecordMaxRegions = 4 + GCCNMF_RTSEP_MAX_SOURCES + 2;   // the real-time sources form's regions, the most of any form
struct RecordMap {
  RecordRegion r[kRecordMaxRegions];
  int n;
  size_t payload;                        // payload bytes of one stream (16-aligned)
};

// Builds a RecordMap from stream 0's regions in a state carved at `base`.  Stream s's copy of a region lies s `stride` bytes on, or,
// with stride 0, s times the region's own size on (an array of per-stream blocks).
struct RecordMapBuilder {
  const void* base;
  size_t stride;
  RecordMap m{};
  // Appends [p, p + bytes) at the payload's end, padded to 16 bytes (nothing for 0 bytes).
  void add(const void* p, size_t bytes) {
    if (bytes == 0) return;
    const size_t next = align_up(m.payload + bytes, 16);
    m.r[m.n++] = RecordRegion{(size_t)((const char*)p - (const char*)base), stride ? stride : bytes, m.payload, bytes, next - m.payload};
    m.payload = next;
  }
};

// Region g of stream s between the state and the payload of its staging record: 16-byte words where both ends and the length allow
// it (every carve region is 256-aligned; some structs and odd ring lengths are not), else 4-byte words (every region is a whole
// number of them).  A save also zeroes the region's padding, so every payload byte of a record is defined.
__device__ __forceinline__ void record_copy_region(char* state, int s, const RecordRegion& g, char* payload, bool to_staging) {
  char* slot = state + g.offset + (size_t)s * g.stride;
  char* rec = payload + g.rec_offset;
  const char* src = to_staging ? slot : rec;
  char* dst = to_staging ? rec : slot;
  if ((((uintptr_t)src | (uintptr_t)dst | g.bytes) & 15) == 0) {
    for (size_t i = threadIdx.x; i < g.bytes / 16; i += blockDim.x) reinterpret_cast<uint4*>(dst)[i] = reinterpret_cast<const uint4*>(src)[i];
  } else {
    for (size_t i = threadIdx.x; i < g.bytes / 4; i += blockDim.x) reinterpret_cast<uint32_t*>(dst)[i] = reinterpret_cast<const uint32_t*>(src)[i];
  }
  if (to_staging)
    for (size_t i = g.bytes / 4 + threadIdx.x; i < g.span / 4; i += blockDim.x) reinterpret_cast<uint32_t*>(rec)[i] = 0;
}

// ---- content digests (GCCNMF_RTREC_DIGEST_*, include/gccnmf_b200.h).  Items come in up to three groups.  Item i of a group is the
// 32-bit words a[0 .. na) at a + i a_stride bytes, then b[0 .. nb) at b + i b_stride; with a K table, na and nb are words per atom
// and the item has K[i] atoms, else they are the item's words and it has `atoms` (0: not a dictionary).  Each item has `chunks`
// chunk slots in the workspace (enough for its largest size; the unused ones get 0), the groups' items one after the other.
constexpr int kDigestChunk = GCCNMF_RTREC_DIGEST_CHUNK_WORDS;
constexpr int kDigestMaxGroups = 3;
struct DigestGroup {
  const void *a, *b;
  size_t a_stride, b_stride;
  size_t na, nb;
  const int32_t* K;
  int atoms, count, chunks;
};
struct DigestItems {
  DigestGroup g[kDigestMaxGroups];
  int n;
};

inline int digest_chunks(size_t words) { return (int)((words + kDigestChunk - 1) / kDigestChunk); }

__device__ __forceinline__ uint64_t record_fnv(uint64_t h, uint32_t w) { return (h ^ w) * GCCNMF_RTREC_DIGEST_PRIME; }

// Item i of group g as two word sequences a[0 .. na) then b[0 .. nb); returns its atoms.
__device__ __forceinline__ int digest_item(const DigestGroup& g, int i, const uint32_t*& a, size_t& na, const uint32_t*& b, size_t& nb) {
  const int K = g.K ? g.K[i] : g.atoms;
  const size_t per = g.K ? (size_t)K : 1;
  a = reinterpret_cast<const uint32_t*>(static_cast<const char*>(g.a) + i * g.a_stride);
  b = reinterpret_cast<const uint32_t*>(static_cast<const char*>(g.b) + i * g.b_stride);
  na = g.na * per;
  nb = g.nb * per;
  return K;
}

// One thread per chunk slot: c_j = FNV-1a 64 over the chunk's words (0 for an unused slot).
__global__ void __launch_bounds__(128) record_digest_chunks_kernel(DigestItems d, uint64_t* __restrict__ chunks) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  int g = 0, k = t;
  for (; g < d.n && k >= d.g[g].count * d.g[g].chunks; ++g) k -= d.g[g].count * d.g[g].chunks;
  if (g == d.n) return;
  const uint32_t *a, *b;
  size_t na, nb;
  digest_item(d.g[g], k / d.g[g].chunks, a, na, b, nb);
  const size_t n = na + nb, w0 = (size_t)(k % d.g[g].chunks) * kDigestChunk, w1 = w0 + kDigestChunk < n ? w0 + kDigestChunk : n;
  uint64_t h = GCCNMF_RTREC_DIGEST_BASIS;
  if (w0 >= n) h = 0;
#pragma unroll 8
  for (size_t w = w0; w < (w1 < na ? w1 : na); ++w) h = record_fnv(h, __ldg(a + w));
  for (size_t w = w0 > na ? w0 : na; w < w1; ++w) h = record_fnv(h, __ldg(b + (w - na)));
  chunks[t] = h;
}

// One thread per item: the digest over (n_lo, n_hi, c_0 lo, c_0 hi, ...) and, when `atoms` is not NULL, the item's atoms.
__global__ void __launch_bounds__(128) record_digest_fold_kernel(DigestItems d, const uint64_t* __restrict__ chunks, uint64_t* __restrict__ digest,
                                                                 int32_t* __restrict__ atoms) {
  const int item = blockIdx.x * blockDim.x + threadIdx.x;
  int g = 0, i = item, c0 = 0;
  for (; g < d.n && i >= d.g[g].count; ++g) c0 += d.g[g].count * d.g[g].chunks, i -= d.g[g].count;
  if (g == d.n) return;
  const uint32_t *a, *b;
  size_t na, nb;
  const int K = digest_item(d.g[g], i, a, na, b, nb);
  const size_t n = na + nb;
  c0 += i * d.g[g].chunks;
  uint64_t h = record_fnv(record_fnv(GCCNMF_RTREC_DIGEST_BASIS, (uint32_t)n), (uint32_t)(n >> 32));
  for (size_t j = 0; j < (n + kDigestChunk - 1) / kDigestChunk; ++j) {
    const uint64_t c = chunks[c0 + j];
    h = record_fnv(record_fnv(h, (uint32_t)c), (uint32_t)(c >> 32));
  }
  digest[item] = h;
  if (atoms) atoms[item] = K;
}

// The chunk kernel, then the fold kernel: every item's digest into digest[0 ..) (and its atoms into atoms[0 ..) when not NULL).
int record_enqueue_digests(gccnmf_handle* h, const DigestItems& d, uint64_t* chunks, uint64_t* digest, int32_t* atoms, void* stream) {
  int slots = 0, items = 0;
  for (int g = 0; g < d.n; ++g) slots += d.g[g].count * d.g[g].chunks, items += d.g[g].count;
  GCCNMF_LAUNCH(h, record_digest_chunks_kernel, (slots + 127) / 128, 128, 0, stream, d, chunks);
  GCCNMF_LAUNCH(h, record_digest_fold_kernel, (items + 127) / 128, 128, 0, stream, d, chunks, digest, atoms);
  return GCCNMF_OK;
}

// The lowest of entries [0, n) whose digest is `digest` and, when K is not NULL, whose atoms are `atoms`; -1 when none is.
__host__ __device__ inline int record_find_entry(const uint64_t* digests, const int32_t* K, int n, uint64_t digest, int atoms) {
  for (int i = 0; i < n; ++i)
    if (digests[i] == digest && (!K || K[i] == atoms)) return i;
  return -1;
}

// ---- host checks.  Every record header starts with these 24 bytes; the configuration words sit at an offset of each kind's own.
struct RecordPrefix {
  uint32_t magic;
  int32_t abi_version, kind, num_sources;
  uint64_t payload_bytes;
};
static_assert(sizeof(RecordPrefix) == 24 && offsetof(gccnmf_record_header, payload_bytes) == offsetof(RecordPrefix, payload_bytes) &&
                  offsetof(gccnmf_rtrec_header, payload_bytes) == offsetof(RecordPrefix, payload_bytes),
              "shared prefix");
constexpr size_t kRecordConfigBytes = sizeof(gccnmf_record_header::config);
static_assert(sizeof(gccnmf_rtrec_header::config) == kRecordConfigBytes, "record config");

// Record i (`got`) against this engine's header (`want`): the shared prefix, then the configuration words at `config` bytes into
// both.  `what` names the calling entry in the message.
int record_check_header(gccnmf_handle* h, const char* what, int i, const void* got_header, const void* want_header, size_t config) {
  RecordPrefix got, want;
  memcpy(&got, got_header, sizeof(got));
  memcpy(&want, want_header, sizeof(want));
  GCCNMF_REQUIRE(h, got.magic == want.magic, "%s: record %d: not a stream record (magic 0x%08x)", what, i, got.magic);
  GCCNMF_REQUIRE(h, got.abi_version == want.abi_version, "%s: record %d: ABI version %d, this library is %d", what, i, got.abi_version,
                 want.abi_version);
  GCCNMF_REQUIRE(h, got.kind == want.kind, "%s: record %d: kind %d, this engine's records are kind %d", what, i, got.kind, want.kind);
  GCCNMF_REQUIRE(h, got.num_sources == want.num_sources, "%s: record %d: %d sources, this engine has %d", what, i, got.num_sources,
                 want.num_sources);
  GCCNMF_REQUIRE(h, got.payload_bytes == want.payload_bytes, "%s: record %d: payload of %llu bytes, expected %llu", what, i,
                 (unsigned long long)got.payload_bytes, (unsigned long long)want.payload_bytes);
  GCCNMF_REQUIRE(h, memcmp((const char*)got_header + config, (const char*)want_header + config, kRecordConfigBytes) == 0,
                 "%s: record %d: another configuration", what, i);
  return GCCNMF_OK;
}

}  // namespace
