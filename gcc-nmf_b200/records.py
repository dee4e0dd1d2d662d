"""Stream records: the persistent state of some streams of an engine, to be loaded into the same or another compatible engine, on any
device, in this process or after a restart.  Two kinds: the low-latency engine's (`LowLatencyEngine`, `gccnmf_llrec_*` in
include/gccnmf_b200.h) and the real-time engines' (`RealtimeEngine` and `MultiStreamRealtimeEngine` in every form, `gccnmf_rtrec_*`).

A `StreamRecord` holds one record per stream in a pinned host buffer, each a header written and checked by the library followed by
the stream's state, plus the engine's host copies of the streams' settings (which a load hands to the destination engine, so
that its later `set_params` / `set_targets` calls rewrite them unchanged).  `save(path)` / `load(path)` keep it in an .npz file.

A real-time record, and a low-latency record of an engine with a steering bank (`gccnmf_llbank_*`), names the dictionary and
steering table its slot was on by content: `content_digest` below, which the library
computes on the device and the engines compute on the host for what they were given.
"""
import numpy as np

from ._lib import (RECORD_HEADER_BYTES, RECORD_KIND_LL, RECORD_KIND_LLBANK, RECORD_KIND_RT, RECORD_MAGIC, RTREC_DIGEST_CHUNK_WORDS,
                   LLBankRecordHeader, RecordHeader, RtRecordHeader)

KINDS = {RECORD_KIND_LL: RecordHeader, RECORD_KIND_RT: RtRecordHeader, RECORD_KIND_LLBANK: LLBankRecordHeader}

_BASIS = np.uint64(0xcbf29ce484222325)
_PRIME = np.uint64(0x100000001b3)


def _fnv_columns(words):
    """FNV-1a 64 of every row of words (rows, n) uint32 -> (rows,) uint64."""
    h = np.full(words.shape[0], _BASIS, dtype=np.uint64)
    with np.errstate(over='ignore'):
        for j in range(words.shape[1]):
            h = (h ^ words[:, j].astype(np.uint64)) * _PRIME
    return h


def content_digest(*arrays):
    """The content digest of gccnmf_rtrec_header (include/gccnmf_b200.h) of the arrays' bytes one after the other, read as 32-bit
    words: FNV-1a 64 of every chunk of 1024 words, then FNV-1a 64 over (n_lo, n_hi, c_0 lo, c_0 hi, ...) -> int."""
    words = np.concatenate([np.ascontiguousarray(a).reshape(-1).view(np.uint32) for a in arrays])
    n, C = len(words), RTREC_DIGEST_CHUNK_WORDS
    full = n // C
    chunks = list(_fnv_columns(words[:full * C].reshape(full, C)))
    if n % C:
        chunks += list(_fnv_columns(words[full * C:].reshape(1, -1)))
    c = np.array(chunks, dtype=np.uint64)
    fold = np.empty(2 + 2 * len(c), dtype=np.uint32)
    fold[0], fold[1] = n & 0xFFFFFFFF, n >> 32
    fold[2::2], fold[3::2] = (c & np.uint64(0xFFFFFFFF)).astype(np.uint32), (c >> np.uint64(32)).astype(np.uint32)
    return int(_fnv_columns(fold.reshape(1, -1))[0])


def call_runs(entry, workspace_bytes, idx, rec, staging, device, stream):
    """Saves or loads the records `rec` of the streams idx (in that order): one call entry(first, count, record, record bytes,
    staging, staging bytes) per run of consecutive streams, with device staging of workspace_bytes(count) bytes, then one wait
    on `stream`.  -> the staging buffer, grown when a run needed more, for the next call."""
    import torch
    idx = np.asarray(idx)
    if len(np.unique(idx)) != len(idx):
        raise ValueError('a stream is listed twice')
    row, rb = 0, rec.data.shape[1]
    for run in np.split(idx, np.flatnonzero(np.diff(idx) != 1) + 1):
        first, count = int(run[0]), len(run)
        n = int(workspace_bytes(count))
        if staging is None or staging.numel() < n:
            staging = torch.empty(n, dtype=torch.uint8, device=device)
        entry(first, count, rec.data[row].data_ptr(), count * rb, staging.data_ptr(), staging.numel())
        row += count
    stream.synchronize()
    return staging


class StreamRecord(object):
    def __init__(self, kind, num_sources, data, mirrors):
        self.kind = int(kind)
        self.num_sources = int(num_sources)
        self.data = data                  # torch.uint8 (count, record bytes), pinned host memory
        self.mirrors = mirrors            # setting name -> numpy array, one row per stream

    @property
    def count(self):
        return int(self.data.shape[0])

    def header(self, i=0):
        """The library's header of record i: gccnmf_record_header (low-latency), gccnmf_llbank_record_header (low-latency with a
        steering bank) or gccnmf_rtrec_header (real-time)."""
        return KINDS[self.kind].from_buffer_copy(self.data[i, :RECORD_HEADER_BYTES].numpy().tobytes())

    def save(self, path):
        """Writes the records to `path` (numpy adds .npz when it is missing)."""
        np.savez(path, kind=self.kind, num_sources=self.num_sources, data=self.data.numpy(),
                 **{'mirror_' + k: v for k, v in self.mirrors.items()})


def load(path):
    """A StreamRecord written by StreamRecord.save."""
    import torch
    with np.load(path) as z:
        data = np.ascontiguousarray(z['data'], dtype=np.uint8)
        if data.ndim != 2 or data.shape[1] < RECORD_HEADER_BYTES:
            raise ValueError('%s: not a stream record file' % path)
        mirrors = {k[len('mirror_'):]: z[k].copy() for k in z.files if k.startswith('mirror_')}
        rec = StreamRecord(int(z['kind']), int(z['num_sources']), torch.from_numpy(data).pin_memory(), mirrors)
    if rec.kind not in KINDS or rec.header(0).magic != RECORD_MAGIC:
        raise ValueError('%s: not a stream record file' % path)
    return rec
