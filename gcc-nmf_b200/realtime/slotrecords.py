"""Stream records of the real-time engines (`gccnmf_rtrec_*` in include/gccnmf_b200.h), shared by `RealtimeEngine` and every form of
`MultiStreamRealtimeEngine`: the single stream, rtm, rtsep and the bank take the same records, so a slot can move between forms.

A record names the dictionary and steering table its slot was on by content digest.  Each engine keeps the digests of what it
was given (windows, every dictionary entry with its H0, every steering entry) and checks every record against them on the host
before it calls the library, so a refusal touches neither the device nor the engine.  A load puts each slot on the lowest entry
of this engine with the record's content.
"""
import ctypes

import numpy as np

from .._lib import RECORD_KIND_RT, RECORD_MAGIC, ParameterError, RtConfig, RtRecordHeader
from ..records import StreamRecord, call_runs, content_digest

# the host mirror of a slot's settings, as a record carries it (targetTDOAIndex None travels as NaN)
PARAM_TYPES = dict(targetTDOAIndex=np.float64, epsilon=np.float64, beta=np.float64, noiseFloor=np.float64, mode=np.int64,
                   separationEnabled=bool, localizationEnabled=bool, localizationWindowSize=np.int64, active=bool)


def params_to_mirrors(params):
    """A list of per-slot settings dicts -> {name: array, one row per slot}."""
    out = {}
    for name, t in PARAM_TYPES.items():
        vals = [p[name] for p in params]
        if name == 'targetTDOAIndex':
            vals = [np.nan if v is None else v for v in vals]
        out[name] = np.array(vals, dtype=t)
    return out


def mirrors_to_params(mirrors, i):
    """Row i of a record's mirrors -> a settings dict."""
    p = {}
    for name, t in PARAM_TYPES.items():
        v = mirrors[name][i]
        if name == 'targetTDOAIndex':
            p[name] = None if np.isnan(v) else float(v)
        else:
            p[name] = bool(v) if t is bool else (int(v) if t is np.int64 else float(v))
    return p


def dictionary_digest(W, H0):
    """Digest of a dictionary entry: W (F, K_i) float32, then H0 (K_i, 2) float32 with inference (None without)."""
    W = np.ascontiguousarray(W, dtype=np.float32)
    return content_digest(W) if H0 is None else content_digest(W, np.ascontiguousarray(H0, dtype=np.float32))


def steering_digest(E):
    """Digest of a steering entry as the state stores it: E^T (D, Fp) complex64, Fp = (F + 3) & ~3, zero beyond F."""
    F, D = E.shape
    ET = np.zeros((D, (F + 3) & ~3), dtype=np.complex64)
    ET[:, :F] = np.asarray(E, dtype=np.complex64).T
    return content_digest(ET)


def windows_digest(analysisWindow, synthesisWindow):
    return content_digest(np.asarray(analysisWindow, np.float32), np.asarray(synthesisWindow, np.float32))


def payload_bytes(cfg, P):
    """Payload bytes of one record (gccnmf_rtrec_header.payload_bytes): RtDev (44), the history (D x history f64), the input ring
    and max(P, 1) output rings (2 x 8 B f32 each) and, with sources, the targets (8 i32) and status (1 i32), each 16-aligned."""
    up = lambda x: (x + 15) // 16 * 16          # noqa: E731
    ring = 4 * 2 * 8 * cfg.block_size
    sizes = [44, 8 * cfg.num_tdoas * cfg.history_length, ring] + [ring] * max(P, 1) + ([32, 4] if P else [])
    return sum(up(s) for s in sizes)


class SlotRecords(object):
    """save_streams / load_streams for an engine that provides h, torch, cfg, state, state_bytes, stream, P, `_record_dims`
    (S, P, Qd, Qe), `_slots`, `_record_digests` (windows, [(dictionary digest, K_i)], [steering digest]), `_params` (a list, one
    settings dict per slot) and `_records_loaded(slots, entries)`."""

    @property
    def record_bytes(self):
        """Bytes of one slot's record."""
        return int(self.h.lib.gccnmf_rtrec_record_bytes(ctypes.byref(self.cfg), self.P))

    def _record_call(self, name, idx, rec):
        """One library call per run of consecutive slots (in the order of idx), then one wait (records.call_runs)."""
        lib, cfg, dims = self.h.lib, ctypes.byref(self.cfg), self._record_dims
        entry = getattr(lib, 'gccnmf_rtrec_' + name)
        self._staging = call_runs(
            lambda *a: self.h.check(entry(self.h.h, cfg, *dims, self.state.data_ptr(), self.state_bytes, *a, self.stream.cuda_stream)),
            lambda count: lib.gccnmf_rtrec_workspace_bytes(cfg, *dims, count), idx, rec, getattr(self, '_staging', None), self.h.device,
            self.stream)

    def _record_slots(self, slots):
        idx = self._slots(list(range(self._record_dims[0])) if slots is None else slots)
        if len(set(idx)) != len(idx):
            raise ValueError('a slot is listed twice')
        return idx

    def save_streams(self, slots=None):
        """The persistent state of `slots` (default: all, in order) between blocks -> a StreamRecord, one record per slot.  The
        slots go on unchanged."""
        idx = self._record_slots(slots)
        rec = StreamRecord(RECORD_KIND_RT, self.P, self.torch.zeros((len(idx), self.record_bytes), dtype=self.torch.uint8).pin_memory(),
                           params_to_mirrors([self._params[s] for s in idx]))
        self._record_call('save_slots', idx, rec)
        return rec

    def _record_header(self):
        """The host part of this engine's headers (gccnmf_rtrec_header without the digests and K_i)."""
        cfg = RtConfig.from_buffer_copy(bytes(self.cfg))
        cfg.num_atoms = 0
        head = RtRecordHeader(magic=RECORD_MAGIC, abi_version=self.h.lib.gccnmf_abi_version(), kind=RECORD_KIND_RT, num_sources=self.P,
                              payload_bytes=payload_bytes(self.cfg, self.P))
        ctypes.memmove(head.config, bytes(cfg), ctypes.sizeof(cfg))
        return head

    def _record_entries(self, record):
        """Checks every record against this engine on the host -> [(dictionary entry, steering entry)] per record, the lowest
        entries with the record's content; raises ParameterError naming what differs."""
        want = self._record_header()
        windows, dicts, steers = self._record_digests
        value = lambda h, f: bytes(h.config) if f == 'config' else getattr(h, f)       # noqa: E731
        host = [f for f, _ in RtRecordHeader._fields_ if not f.endswith('_digest') and f != 'dictionary_atoms']
        entries = []
        for i in range(record.count):
            got = record.header(i)
            bad = [f for f in host if value(got, f) != value(want, f)]
            if bad:
                raise ParameterError('record %d does not fit this engine: %s differ' % (i, ', '.join(bad)))
            if got.windows_digest != windows:
                raise ParameterError('record %d: other analysis / synthesis windows' % i)
            d = [k for k, e in enumerate(dicts) if e == (got.dictionary_digest, got.dictionary_atoms)]
            if not d:
                raise ParameterError('record %d: no dictionary entry of this engine holds its dictionary (%d atoms)' % (i, got.dictionary_atoms))
            e = [k for k, s in enumerate(steers) if s == got.steering_digest]
            if not e:
                raise ParameterError('record %d: no steering entry of this engine holds its steering table' % i)
            entries.append((d[0], e[0]))
        return entries

    def load_streams(self, slots, record):
        """Record i replaces the state and settings of slots[i] from the next block on, on this engine's entries that hold the
        record's dictionary and steering table.  The record must come from a real-time engine of any form with the same
        configuration other than the number of slots, K_max and the bank, the same numSources and the same windows.  Every record
        is checked on the host before anything is loaded, so a refusal leaves the engine and the device untouched.  Each run of
        consecutive slots is one library call."""
        idx = self._record_slots(slots)
        if record.kind != RECORD_KIND_RT or record.count != len(idx):
            raise ValueError('a real-time record of %d slots is needed (got kind %d, %d slots)' % (len(idx), record.kind, record.count))
        if record.data.shape[1] != self.record_bytes:
            raise ParameterError('records of %d bytes do not fit this engine (%d bytes)' % (record.data.shape[1], self.record_bytes))
        entries = self._record_entries(record)
        self._record_call('load_slots', idx, record)
        for i, s in enumerate(idx):
            self._params[s] = mirrors_to_params(record.mirrors, i)
        self._records_loaded(idx, entries)
