"""Stream records: the persistent state of some streams of a `LowLatencyEngine`, to be loaded into the same or another compatible
engine, on any device, in this process or after a restart (`gccnmf_llrec_*` in include/gccnmf_b200.h).

A `StreamRecord` holds one record per stream in a pinned host buffer, each a header written and checked by the library followed by
the stream's state, plus the engine's host copies of the streams' settings (which a load hands to the destination engine, so
that its later `set_params` / `set_targets` calls rewrite them unchanged).  `save(path)` / `load(path)` keep it in an .npz file.
"""
import numpy as np

from ._lib import RECORD_HEADER_BYTES, RECORD_KIND_LL, RECORD_MAGIC, RecordHeader


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
        """The library's header of record i (gccnmf_record_header)."""
        return RecordHeader.from_buffer_copy(self.data[i, :RECORD_HEADER_BYTES].numpy().tobytes())

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
    if rec.kind != RECORD_KIND_LL or rec.header(0).magic != RECORD_MAGIC:
        raise ValueError('%s: not a stream record file' % path)
    return rec
