"""Streaming form of the online / low-latency notebook loop (csrc/lowlatency.cu, `gccnmf_ll_*` in include/gccnmf_b200.h).

One `LowLatencyEngine` holds S independent streams on the device.  Each `process` call takes `hops * hop` new samples per stream
and returns as many finished output samples per stream; output sample p of a stream is sample p - `latency` of what
`online.performOnlineSpeechEnhancement` computes on the whole recording (samples before the stream's first frame are zero).  A
call is one stream-ordered unit on the device, optionally one CUDA graph launch.

The synthesis is a weight vector w applied to every frame in the overlap-add and a gain g applied to every output sample
(`synthesisWeights`):
  'online'      gainPerFrame=True of the batch function: w = gainFactor, g = 1
  'lowlatency'  gainPerFrame=False (the low-latency notebook, which never applies its synthesis window): w = 1, g = gainFactor
  'windowed'    applySynthesisWindow=True: w = the synthesis window, g = gainFactor
with gainFactor = 2 hop / N.  The latency is Q hop - hop - z samples, Q = ceil(N / hop) and z the first nonzero index of w; when hop
divides N that is N - hop for the first two, and 2m - hop - 1 for the asymmetric synthesis window of
lowLatencySpeechEnhancement.ipynb:382-392 (its first weight is zero).

Sources (`numSources` = P in [2, 8], `gccnmf_llsep_*`): every stream is separated into P sources, one per target TDOA index (the
reference's multi-target rule, gccNMFFunctions.py:94-143, per frame).  The targets of a frame are the P largest strict local
maxima of its running maximum (held, with status bit 0, when there are fewer), or the overrides of `set_targets`; each atom goes
to the target with the largest float32 GCC-NMF value (numpy.nanargmax), and source q is the single-target filter and synthesis fed
that mask.  `process` then returns (S, P, 2, n).  The boxcar epsilon and the single target override play no part.

Localisation window (`historyLength` = Lh in [1, 1024], `gccnmf_llhist_*`): every stream keeps the angular spectra of its last Lh
frames in a ring.  `set_localization(streams, window)` with 1 <= window <= Lh makes a stream's target (or its P targets) follow the
nanmean of its newest `window` frames, the real-time engine's rule, so the target follows a talker who moves and recovers from
silent frames; window 0 (the default, and after `reset`) is the running maximum above.  With historyLength 0 the engine is the
plain one.

Steering bank (`expJOmegaTau` a sequence of Qe tables, 1 <= Qe <= 64, `gccnmf_llbank_*`): each stream is on one table, its
client's microphone spacing; `assign_steering(streams, entries)` moves streams between tables and `load_steering(entry, E)` replaces
a table, both from the next call on and keeping everything else of the streams.  A stream on table j computes, bit for bit, what an
engine built with that table alone computes.  `init` and `reset` put streams on table 0.
"""
import ctypes

import numpy as np

from ._lib import (LLDICT_MAX_DICTIONARIES, LLBANK_MAX_STEERINGS, LLHIST_MAX_HISTORY, LLHIST_RECORD_CONFIG_HISTORY, RECORD_KIND_LL, RECORD_KIND_LLBANK, RECORD_MAGIC,
                   LLConfig, LLStreamParams, ParameterError, RecordHeader, default_handle)

SYNTHESIS_MODES = ('online', 'lowlatency', 'windowed')

EXPORT_X, EXPORT_COHERENCE, EXPORT_ANGULAR, EXPORT_ACC_MAX, EXPORT_TARGETS, EXPORT_ARGMAX, EXPORT_MASKS, EXPORT_WIENER, EXPORT_Y, \
    EXPORT_REFINED, EXPORT_STATUS, EXPORT_H, EXPORT_VALID, EXPORT_CARRY = range(14)
# export items of an engine with sources (gccnmf_llsep_export); items 4 .. 10 are then refused
EXPORT_SOURCE_TARGETS, EXPORT_SOURCE_VALUES, EXPORT_SOURCE_MASKS, EXPORT_SOURCE_WIENER, EXPORT_SOURCE_Y, EXPORT_STREAM_STATUS, \
    EXPORT_CARRIED_TARGETS, EXPORT_CALL_STATUS = range(14, 22)
# export items of an engine with historyLength > 0 (gccnmf_llhist_export)
EXPORT_HISTORY, EXPORT_HISTORY_INDEX, EXPORT_WINDOWS, EXPORT_WINDOW_MEANS = range(22, 26)
EXPORT_DICTIONARY_ASSIGNMENT = 27                               # an engine with a dictionary bank (gccnmf_lldict_export)
EXPORT_DICTIONARY_ATOMS = 28
ATOMS_OFFSET = RecordHeader.config.offset + 4 * 3                # a record header's config.num_atoms
EXPORT_ASSIGNMENT = 26                                          # an engine with a steering bank (gccnmf_llbank_export)
STATUS_FEW_PEAKS, STATUS_ALL_NAN = 1, 2
MAX_SOURCES = 8
MAX_HISTORY = LLHIST_MAX_HISTORY
MAX_STEERINGS = LLBANK_MAX_STEERINGS
MAX_DICTIONARIES = LLDICT_MAX_DICTIONARIES


def synthesisWeights(mode, synthesisWindow, hopSize):
    """(w (N) float64, g float32) of a synthesis mode (see the module docstring)."""
    N = len(synthesisWindow)
    gainFactor = hopSize / float(N) * 2
    if mode == 'online':
        return np.full(N, gainFactor), np.float32(1.0)
    if mode == 'lowlatency':
        return np.ones(N), np.float32(gainFactor)
    if mode == 'windowed':
        return np.ascontiguousarray(synthesisWindow, dtype=np.float64), np.float32(gainFactor)
    raise ValueError('synthesis must be one of %s (got %r)' % (SYNTHESIS_MODES, mode))


def latencyOf(weights, hopSize):
    """Samples between the newest input and the output emitted with it: Q hop - hop - z, Q = ceil(N / hop), z the first nonzero
    index of the weights (a frame ends in the hop that completes it, and its first z weights are zero)."""
    nz = np.flatnonzero(np.asarray(weights) != 0)
    if len(nz) == 0:
        raise ValueError('the synthesis weights are all zero')
    hop = int(hopSize)
    return -(-len(weights) // hop) * hop - hop - int(nz[0])


def batchArguments(mode):
    """The performOnlineSpeechEnhancement keywords that compute what a synthesis mode streams."""
    return {'online': dict(gainPerFrame=True), 'lowlatency': dict(gainPerFrame=False),
            'windowed': dict(gainPerFrame=False, applySynthesisWindow=True)}[mode]


class LowLatencyEngine(object):
    def __init__(self, W, expJOmegaTau, analysisWindow, synthesisWindow, hopSize, numStreams=1, hopsPerCall=1, synthesis='lowlatency',
                 targetTDOAEpsilon=1.0, numInferenceIterations=0, sparsityAlpha=0.0, epsilon=1e-16, seedValue=0, device=0, numSources=0,
                 historyLength=0):
        self.P = int(numSources)
        if self.P != 0 and not 2 <= self.P <= MAX_SOURCES:
            raise ValueError('numSources must be 0 (one enhanced target) or in [2, %d] (got %d)' % (MAX_SOURCES, self.P))
        self.Lh = int(historyLength)
        if not 0 <= self.Lh <= MAX_HISTORY:
            raise ValueError('historyLength must be in [0, %d] (got %d)' % (MAX_HISTORY, self.Lh))
        # a sequence of tables (or a (Qe, F, D) array) is a steering bank; one (F, D) table is the plain engine
        bank = isinstance(expJOmegaTau, (list, tuple)) or np.ndim(expJOmegaTau) == 3
        self.Qe = len(expJOmegaTau) if bank else 0
        if bank and not 1 <= self.Qe <= MAX_STEERINGS:
            raise ValueError('a steering bank holds 1 .. %d tables (got %d)' % (MAX_STEERINGS, self.Qe))
        if bank and len({np.shape(e) for e in expJOmegaTau}) != 1:
            raise ValueError('the tables of a steering bank must all be (F, D)')
        # a sequence of dictionaries is a dictionary bank (gccnmf_lldict_*, always with a steering bank): K = the largest K_i
        self.Qd = len(W) if isinstance(W, (list, tuple)) else 0
        if isinstance(W, (list, tuple)) and not 1 <= self.Qd <= MAX_DICTIONARIES:
            raise ValueError('a dictionary bank holds 1 .. %d dictionaries (got %d)' % (MAX_DICTIONARIES, self.Qd))
        if self.Qd and not bank:
            bank, expJOmegaTau, self.Qe = True, [expJOmegaTau], 1
        Ws = [np.ascontiguousarray(w, dtype=np.float32) for w in W] if self.Qd else None
        if self.Qd and (any(w.ndim != 2 or w.shape[0] != Ws[0].shape[0] or w.shape[1] < 1 for w in Ws)):
            raise ValueError('the dictionaries of a bank must all be (F, K_i) with K_i >= 1')
        self.h = default_handle(device)
        torch = self.torch = self.h.torch
        W = Ws[int(np.argmax([w.shape[1] for w in Ws]))] if self.Qd else np.ascontiguousarray(W, dtype=np.float32)
        E = np.ascontiguousarray(np.stack(list(expJOmegaTau)) if bank else expJOmegaTau, dtype=np.complex128)
        F, K = W.shape
        N = len(analysisWindow)
        if N != 2 * (F - 1) or E.shape[-2] != F or len(synthesisWindow) != N:
            raise ValueError('W (F, K), expJOmegaTau (F, D) and the windows (N = 2 (F - 1)) do not agree')
        self.F, self.K, self.N, self.D = F, K, N, E.shape[-1]
        self.hop, self.S, self.C = int(hopSize), int(numStreams), int(hopsPerCall)
        self.synthesis = synthesis
        self.weights, self.gain = synthesisWeights(synthesis, synthesisWindow, self.hop)
        self.latency = latencyOf(self.weights, self.hop)
        if self.latency < 0:
            raise ValueError('the synthesis weights start less than a hop before the end of the frame')
        self.cfg = LLConfig(N, self.hop, self.C, K, self.D, self.S, int(numInferenceIterations), float(sparsityAlpha), float(epsilon))
        if self.Qd:
            self.state_bytes = int(self.h.lib.gccnmf_lldict_state_bytes(ctypes.byref(self.cfg), self.P, self.Lh, self.Qd, self.Qe))
        elif self.Qe:
            self.state_bytes = int(self.h.lib.gccnmf_llbank_state_bytes(ctypes.byref(self.cfg), self.P, self.Lh, self.Qe))
        elif self.Lh:
            self.state_bytes = int(self.h.lib.gccnmf_llhist_state_bytes(ctypes.byref(self.cfg), self.P, self.Lh))
        else:
            self.state_bytes = int(self.h.lib.gccnmf_llsep_state_bytes(ctypes.byref(self.cfg), self.P) if self.P else
                                   self.h.lib.gccnmf_ll_state_bytes(ctypes.byref(self.cfg)))
        if self.state_bytes == 0:
            raise ValueError('invalid low-latency configuration (N a power of two in [32, 4096], 1 <= hop <= N, 1 <= hopsPerCall <= 64, '
                             'D a power of two in [4, 128], 1 <= numStreams <= 4096)')
        self.inference = numInferenceIterations > 0
        self.stream = torch.cuda.Stream(device=self.h.device)      # a capturable stream of its own
        self.state = torch.empty(self.state_bytes, dtype=torch.uint8, device=self.h.device)
        H0 = None
        self._seed, self._epsilon = seedValue, epsilon
        if self.inference:
            np.random.seed(seedValue)                                 # gccNMFFunctions.py:70,73, as online.py draws it
            H0 = (np.random.random((K, 2)).astype(np.float32) + epsilon).astype(np.float32)
        dev = lambda a: torch.as_tensor(np.ascontiguousarray(a)).to(self.h.device)      # noqa: E731
        self._const = [dev(W), dev(E.view(np.float64).reshape(-1, F, 2 * self.D)), dev(np.asarray(analysisWindow, np.float64)),
                       dev(self.weights), dev(H0) if H0 is not None else None]
        self._eps = np.full(self.S, float(targetTDOAEpsilon), np.float32)
        self._active = np.ones(self.S, np.int32)
        self._override = np.full(self.S, -1, np.int32)
        self._targets = np.full((self.S, max(self.P, 1)), -1, np.int32)
        self._window = np.zeros(self.S, np.int32)
        self._assign = np.zeros(self.S, np.int32)                 # bank: each stream's table
        self._dassign = np.zeros(self.S, np.int32)                # dictionary bank: each stream's dictionary
        if self.Qe:                                               # content digests of the dictionary and the tables (bank records)
            from .records import content_digest
            # (a dictionary bank keeps one digest per entry, below)
            self._dict_digest = None if self.Qd else content_digest(W, H0) if H0 is not None else content_digest(W)
            self._steer_digests = [content_digest(e) for e in E]
        self._io = {}
        self._graphs = {}
        self._exports = {}
        self._staging = None                                      # device staging of stream records
        self._header = None                                       # their header, once computed
        self.last_hops = None
        self.h.torch.cuda.current_stream(self.h.device).synchronize()
        c = self._const
        if self.Qd:
            self._dicts = [dev(w) for w in Ws]
            self._h0s = [dev(self._draw_h0(w.shape[1])) for w in Ws] if self.inference else None
            self._atoms = [w.shape[1] for w in Ws]
            from .records import content_digest
            self._dict_digests = [content_digest(w, self._draw_h0(w.shape[1])) if self.inference else content_digest(w) for w in Ws]
            with torch.cuda.stream(self.stream):
                ptr = lambda ts: (ctypes.c_void_p * self.Qd)(*[t.data_ptr() for t in ts])       # noqa: E731
                self._check(self.h.lib.gccnmf_lldict_init(self.h.h, ctypes.byref(self.cfg), self.P, self.Lh, self.Qd, self.Qe, ptr(self._dicts),
                                                          (ctypes.c_int * self.Qd)(*self._atoms), ptr(self._h0s) if self._h0s else None,
                                                          c[1].data_ptr(), c[2].data_ptr(), c[3].data_ptr(), float(self.gain), self.state.data_ptr(),
                                                          self.state_bytes, self.stream.cuda_stream))
            self._send_params(0, self.S)
            self.stream.synchronize()
            return
        with torch.cuda.stream(self.stream):
            self._check(self._fn('init')(self.h.h, ctypes.byref(self.cfg), *self._p, c[0].data_ptr(), c[1].data_ptr(), c[2].data_ptr(),
                                         c[3].data_ptr(), float(self.gain), c[4].data_ptr() if c[4] is not None else None,
                                         self.state.data_ptr(), self.state_bytes, self.stream.cuda_stream))
        self._send_params(0, self.S)
        self.stream.synchronize()

    def _check(self, status):
        self.h.check(status)

    def _draw_h0(self, K):
        """H0 (K, 2) as the plain engine with K atoms draws it."""
        np.random.seed(self._seed)
        return (np.random.random((K, 2)).astype(np.float32) + self._epsilon).astype(np.float32)

    @property
    def _p(self):
        """The num_sources argument of the gccnmf_llsep_* entries, num_sources and history_length of the gccnmf_llhist_* entries (none
        for gccnmf_ll_*)."""
        if self.Qd:
            return (self.P, self.Lh, self.Qd, self.Qe)
        return (self.P, self.Lh, self.Qe) if self.Qe else (self.P, self.Lh) if self.Lh else (self.P,) if self.P else ()

    def _fn(self, name):
        prefix = 'gccnmf_lldict_' if self.Qd else 'gccnmf_llbank_' if self.Qe else 'gccnmf_llhist_' if self.Lh else 'gccnmf_llsep_' if self.P else 'gccnmf_ll_'
        return getattr(self.h.lib, prefix + name)

    def _state(self, name, *args):
        """gccnmf_ll_<name>(h, cfg, state, state_bytes, *args), gccnmf_llsep_<name>(h, cfg, P, state, state_bytes, *args) or
        gccnmf_llhist_<name>(h, cfg, P, Lh, state, state_bytes, *args), gccnmf_llbank_<name>(h, cfg, P, Lh, Qe, state, ...)."""
        self._check(self._fn(name)(self.h.h, ctypes.byref(self.cfg), *self._p, self.state.data_ptr(), self.state_bytes, *args))

    def _streams(self, streams):
        if streams is None:
            return np.arange(self.S)
        idx = np.atleast_1d(np.asarray(streams, dtype=np.int64))
        if idx.size == 0 or idx.min() < 0 or idx.max() >= self.S:
            raise ValueError('streams outside [0, %d)' % self.S)
        return idx

    def _send_params(self, first, count):
        arr = (LLStreamParams * count)()
        for i in range(count):
            s = first + i
            arr[i] = LLStreamParams(float(self._eps[s]), int(self._active[s]), int(self._override[s]))
        self._state('set_params', first, count, arr, self.stream.cuda_stream)

    def _send_streams(self, idx):
        lo, hi = int(idx.min()), int(idx.max())
        self._send_params(lo, hi - lo + 1)
        self.stream.synchronize()

    # ------------------------------------------------------------------ settings (stream-ordered: they act from the next call)
    def set_params(self, streams=None, targetTDOAEpsilon=None, targetOverride=None):
        """Per-stream epsilon of the boxcar atom mask, and a target TDOA index that replaces the localised one (-1: none)."""
        idx = self._streams(streams)
        if targetTDOAEpsilon is not None:
            self._eps[idx] = targetTDOAEpsilon
        if targetOverride is not None:
            o = np.broadcast_to(np.asarray(targetOverride, dtype=np.int64), idx.shape)
            if o.min() < -1 or o.max() >= self.D:
                raise ValueError('targetOverride outside [0, %d) (or -1)' % self.D)
            self._override[idx] = o
        self._send_streams(idx)

    def set_targets(self, streams, targets):
        """Sources only: per stream P target TDOA indexes that replace the localised ones, -1 for a source that follows the
        localisation.  targets broadcasts to (len(streams), P)."""
        if not self.P:
            raise ValueError('set_targets needs numSources >= 2')
        idx = self._streams(streams)
        t = np.broadcast_to(np.asarray(targets, dtype=np.int64), (len(idx), self.P))
        if t.min() < -1 or t.max() >= self.D:
            raise ValueError('targets outside [0, %d) (or -1)' % self.D)
        self._targets[idx] = t
        lo, hi = int(idx.min()), int(idx.max())
        arr = np.ascontiguousarray(self._targets[lo:hi + 1], dtype=np.int32)
        self._state('set_targets', lo, hi - lo + 1, arr.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), self.stream.cuda_stream)
        self.stream.synchronize()

    def set_localization(self, streams, window):
        """Per-stream localisation window in frames: 0 is the running maximum (the default), 1 .. historyLength the nanmean of the
        stream's newest `window` angular spectra.  window broadcasts to len(streams)."""
        idx = self._streams(streams)
        w = np.broadcast_to(np.asarray(window, dtype=np.int64), idx.shape)
        if w.min() < 0 or w.max() > self.Lh:
            raise ValueError('window outside [0, %d] (historyLength %d)' % (self.Lh, self.Lh))
        if not self.Lh:
            return                                                # only window 0: the engine is the plain one
        self._window[idx] = w
        lo, hi = int(idx.min()), int(idx.max())
        arr = np.ascontiguousarray(self._window[lo:hi + 1], dtype=np.int32)
        self._state('set_window', lo, hi - lo + 1, arr.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), self.stream.cuda_stream)
        self.stream.synchronize()

    def assign_steering(self, streams, entries):
        """Steering bank: the streams use tables `entries` (broadcast to len(streams)) from the next call on; everything else of
        them stays."""
        if not self.Qe:
            raise ValueError('assign_steering needs a steering bank (expJOmegaTau a sequence of tables)')
        idx = self._streams(streams)
        e = np.broadcast_to(np.asarray(entries, dtype=np.int64), idx.shape)
        if e.min() < 0 or e.max() >= self.Qe:
            raise ValueError('steering entries outside [0, %d)' % self.Qe)
        self._assign[idx] = e
        self._send_assign(idx)

    def _send_assign(self, idx):
        lo, hi = int(idx.min()), int(idx.max())
        arr = np.ascontiguousarray(self._assign[lo:hi + 1], dtype=np.int32)
        ptr = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_int32))       # noqa: E731
        if self.Qd:
            darr = np.ascontiguousarray(self._dassign[lo:hi + 1], dtype=np.int32)
            self._state('assign', lo, hi - lo + 1, ptr(darr), ptr(arr), self.stream.cuda_stream)
        else:
            self._state('assign', lo, hi - lo + 1, ptr(arr), self.stream.cuda_stream)
        self.stream.synchronize()

    def assign_dictionary(self, streams, entries):
        """Dictionary bank: the streams use dictionaries `entries` (broadcast to len(streams)) from the next call on; everything else
        of them stays."""
        if not self.Qd:
            raise ValueError('assign_dictionary needs a dictionary bank (W a sequence of dictionaries)')
        idx = self._streams(streams)
        e = np.broadcast_to(np.asarray(entries, dtype=np.int64), idx.shape)
        if e.min() < 0 or e.max() >= self.Qd:
            raise ValueError('dictionary entries outside [0, %d)' % self.Qd)
        self._dassign[idx] = e
        self._send_assign(idx)

    def load_dictionary(self, entry, W):
        """Dictionary bank: dictionary `entry` becomes W (F, K), K <= numAtoms of the largest entry at construction, from the next call
        on, for every stream on it; with inference its H0 is drawn as the plain engine with K atoms draws it."""
        if not self.Qd:
            raise ValueError('load_dictionary needs a dictionary bank (W a sequence of dictionaries)')
        if not 0 <= int(entry) < self.Qd:
            raise ValueError('dictionary entry outside [0, %d)' % self.Qd)
        W = np.ascontiguousarray(W, dtype=np.float32)
        if W.ndim != 2 or W.shape[0] != self.F or not 1 <= W.shape[1] <= self.K:
            raise ValueError('W must be (%d, K) with 1 <= K <= %d' % (self.F, self.K))
        t = self.torch.as_tensor(W).to(self.h.device)
        h0 = self.torch.as_tensor(self._draw_h0(W.shape[1])).to(self.h.device) if self.inference else None
        self._state('load_dictionary', int(entry), t.data_ptr(), W.shape[1], h0.data_ptr() if h0 is not None else None, self.stream.cuda_stream)
        self.stream.synchronize()
        from .records import content_digest
        self._dicts[int(entry)], self._atoms[int(entry)] = t, W.shape[1]
        self._dict_digests[int(entry)] = content_digest(W, h0.cpu().numpy()) if h0 is not None else content_digest(W)
        if h0 is not None:
            self._h0s[int(entry)] = h0

    def load_steering(self, entry, expJOmegaTau):
        """Steering bank: table `entry` becomes expJOmegaTau (F, D) from the next call on, for every stream on it."""
        if not self.Qe:
            raise ValueError('load_steering needs a steering bank (expJOmegaTau a sequence of tables)')
        if not 0 <= int(entry) < self.Qe:
            raise ValueError('steering entry outside [0, %d)' % self.Qe)
        E = np.ascontiguousarray(expJOmegaTau, dtype=np.complex128)
        if E.shape != (self.F, self.D):
            raise ValueError('expJOmegaTau must be (%d, %d)' % (self.F, self.D))
        from .records import content_digest
        t = self.torch.as_tensor(E.view(np.float64)).to(self.h.device)
        self._state('load_steering', int(entry), t.data_ptr(), self.stream.cuda_stream)
        self.stream.synchronize()
        self._steer_digests[int(entry)] = content_digest(E)

    def set_active(self, streams, active):
        """An inactive stream outputs zeros and its state does not change."""
        idx = self._streams(streams)
        self._active[idx] = 1 if active else 0
        self._send_streams(idx)

    def reset(self, streams=None):
        """The streams start over (rings zeroed, running maximum -inf, no frames yet, localisation window 0); their other
        parameters stay."""
        idx = np.unique(self._streams(streams))
        self._window[idx] = 0
        self._assign[idx] = 0
        self._dassign[idx] = 0
        breaks = np.flatnonzero(np.diff(idx) != 1) + 1          # one call per contiguous run of streams
        for run in np.split(idx, breaks):
            self._state('reset_streams', int(run[0]), len(run), self.stream.cuda_stream)
        self.stream.synchronize()

    # ------------------------------------------------------------------ per-call work
    def _buffers(self, hops):
        b = self._io.get(hops)
        if b is None:
            torch = self.torch
            shape = (self.S, 2, hops * self.hop)
            oshape = (self.S, self.P, 2, hops * self.hop) if self.P else shape
            b = self._io[hops] = (torch.zeros(shape, dtype=torch.float32).pin_memory(), torch.zeros(oshape, dtype=torch.float32).pin_memory(),
                                  torch.zeros(shape, dtype=torch.float32, device=self.h.device),
                                  torch.zeros(oshape, dtype=torch.float32, device=self.h.device))
        return b

    def build_graph(self, hops=None):
        """The graph of a call of `hops` hops (default: hopsPerCall): H2D of the pinned input, the kernels, D2H of the output."""
        hops = self.C if hops is None else int(hops)
        g = self._graphs.get(hops)
        if g is None:
            in_host, out_host, in_dev, out_dev = self._buffers(hops)
            g = ctypes.c_void_p()
            self._state('graph_create', hops, in_dev.data_ptr(), out_dev.data_ptr(), in_host.data_ptr(), out_host.data_ptr(), ctypes.byref(g),
                        self.stream.cuda_stream)
            self._graphs[hops] = g
        return g

    def process(self, x, use_graph=True):
        """x (S, 2, hops * hop) float32 -> (S, 2, hops * hop) float32, or (S, P, 2, hops * hop) with sources (a copy)."""
        x = np.asarray(x, dtype=np.float32)
        if x.ndim != 3 or x.shape[0] != self.S or x.shape[1] != 2 or x.shape[2] % self.hop != 0:
            raise ValueError('x must be (%d, 2, hops * %d)' % (self.S, self.hop))
        hops = x.shape[2] // self.hop
        if not 1 <= hops <= self.C:
            raise ValueError('a call takes 1 .. %d hops (got %d)' % (self.C, hops))
        in_host, out_host, in_dev, out_dev = self._buffers(hops)
        in_host.numpy()[:] = x
        if use_graph:
            self._check(self.h.lib.gccnmf_rt_graph_launch(self.h.h, self.build_graph(hops), self.stream.cuda_stream))
        else:
            with self.torch.cuda.stream(self.stream):
                in_dev.copy_(in_host, non_blocking=True)
                self._state('process', hops, in_dev.data_ptr(), out_dev.data_ptr(), self.stream.cuda_stream)
                out_host.copy_(out_dev, non_blocking=True)
        self.stream.synchronize()
        self.last_hops = hops
        return out_host.numpy().copy()

    def export(self, what):
        """Host copy of one item of the last call (see gccnmf_ll_export / gccnmf_llsep_export); T = S hops columns, column s hops + i =
        frame i of stream s."""
        if self.last_hops is None:
            raise RuntimeError('no call yet')
        torch = self.torch
        T, F, K, D = self.S * self.last_hops, self.F, self.K, self.D
        shapes = {EXPORT_X: ((2, F, T), torch.complex64), EXPORT_COHERENCE: ((F, T), torch.complex64), EXPORT_ANGULAR: ((D, T), torch.float64),
                  EXPORT_ACC_MAX: ((D, T), torch.float64), EXPORT_TARGETS: ((T,), torch.int32), EXPORT_ARGMAX: ((K, T), torch.int32),
                  EXPORT_MASKS: ((K, T), torch.float32), EXPORT_WIENER: (((2, F, T) if self.inference else (F, T)), torch.float32),
                  EXPORT_Y: ((2, F, T), torch.complex64), EXPORT_REFINED: ((1,), torch.int32), EXPORT_STATUS: ((1,), torch.int32),
                  EXPORT_H: ((K, 2 * T), torch.float32), EXPORT_VALID: ((T,), torch.int32), EXPORT_CARRY: ((self.S, D), torch.float64)}
        P = self.P
        if P:
            shapes.update({EXPORT_SOURCE_TARGETS: ((T, P), torch.int32), EXPORT_SOURCE_VALUES: ((P, K, T), torch.float32),
                           EXPORT_SOURCE_MASKS: ((P, K, T), torch.float32),
                           EXPORT_SOURCE_WIENER: (((P, 2, F, T) if self.inference else (P, F, T)), torch.float32),
                           EXPORT_SOURCE_Y: ((P, 2, F, T), torch.complex64), EXPORT_STREAM_STATUS: ((self.S,), torch.int32),
                           EXPORT_CARRIED_TARGETS: ((self.S, P), torch.int32), EXPORT_CALL_STATUS: ((1,), torch.int32)})
        if self.Qe:
            shapes[EXPORT_ASSIGNMENT] = ((self.S,), torch.int32)
        if self.Qd:
            shapes[EXPORT_DICTIONARY_ASSIGNMENT] = ((self.S,), torch.int32)
            shapes[EXPORT_DICTIONARY_ATOMS] = ((self.Qd,), torch.int32)
        if self.Lh:
            shapes.update({EXPORT_HISTORY: ((self.S, D, self.Lh), torch.float64), EXPORT_HISTORY_INDEX: ((self.S,), torch.int32),
                           EXPORT_WINDOWS: ((self.S,), torch.int32), EXPORT_WINDOW_MEANS: ((D, T), torch.float64)})
        shape, dtype = shapes[what]
        key = (what, shape)
        buf = self._exports.get(key)
        if buf is None:
            buf = self._exports[key] = torch.zeros(shape, dtype=dtype).pin_memory()
        self._state('export', self.last_hops, int(what), buf.data_ptr(), self.stream.cuda_stream)
        self.stream.synchronize()
        return buf.numpy().copy()

    # ------------------------------------------------------------------ stream records (gccnmf_llrec_*, or gccnmf_llhist_* with history)
    def _rec(self, name):
        """gccnmf_llrec_<name> bound to (cfg, P), gccnmf_llhist_<name> bound to (cfg, P, Lh) or gccnmf_llbank_<name> bound to
        (cfg, P, Lh, Qe)."""
        fn = getattr(self.h.lib, ('gccnmf_lldict_' if self.Qd else 'gccnmf_llbank_' if self.Qe else 'gccnmf_llhist_' if self.Lh else 'gccnmf_llrec_') + name)
        hist = (self.Lh, self.Qd, self.Qe) if self.Qd else (self.Lh, self.Qe) if self.Qe else (self.Lh,) if self.Lh else ()
        if name.endswith('_bytes'):
            return lambda *a: fn(ctypes.byref(self.cfg), self.P, *hist, *a)
        return lambda *a: fn(self.h.h, ctypes.byref(self.cfg), self.P, *hist, *a)

    @property
    def record_bytes(self):
        """Bytes of one stream's record."""
        return int(self._rec('record_bytes')())

    def _record_call(self, name, streams, rec):
        """One library call per run of consecutive streams, then one wait (records.call_runs)."""
        from .records import call_runs
        entry = self._rec(name)
        self._staging = call_runs(lambda *a: self._check(entry(self.state.data_ptr(), self.state_bytes, *a, self.stream.cuda_stream)),
                                  self._rec('workspace_bytes'), self._streams(streams), rec, self._staging, self.h.device, self.stream)

    def save_streams(self, streams=None):
        """The persistent state of `streams` (default: all, in order) between calls -> a StreamRecord, one record per stream.  The
        streams go on unchanged."""
        from .records import StreamRecord
        idx = self._streams(streams)
        mirrors = dict(eps=self._eps[idx].copy(), active=self._active[idx].copy(), override=self._override[idx].copy(),
                       targets=self._targets[idx].copy())
        if self.Lh:
            mirrors['window'] = self._window[idx].copy()
        rec = StreamRecord(RECORD_KIND_LLBANK if self.Qe else RECORD_KIND_LL, self.P, self.torch.zeros((len(idx), self.record_bytes), dtype=self.torch.uint8).pin_memory(),
                           mirrors)
        self._record_call('save_streams', idx, rec)
        return rec

    def _record_header(self):
        """The header this engine's records carry (gccnmf_record_header), computed on the host: the library writes the same."""
        cfg = LLConfig.from_buffer_copy(bytes(self.cfg))
        cfg.num_streams = cfg.hops_per_call = 0
        head = RecordHeader(magic=RECORD_MAGIC, abi_version=self.h.lib.gccnmf_abi_version(), kind=RECORD_KIND_LLBANK if self.Qe else RECORD_KIND_LL,
                            num_sources=self.P,
                            payload_bytes=int(self.h.lib.gccnmf_llhist_workspace_bytes(ctypes.byref(self.cfg), self.P, self.Lh, 1)))
        ctypes.memmove(head.config, bytes(cfg), ctypes.sizeof(cfg))
        head.config[LLHIST_RECORD_CONFIG_HISTORY] = self.Lh
        d = 1469598103934665603                                    # FNV-1a 64 of the weights' bytes, then the gain's
        for b in np.ascontiguousarray(self.weights, np.float64).tobytes() + np.float32(self.gain).tobytes():
            d = ((d ^ b) * 1099511628211) & 0xFFFFFFFFFFFFFFFF
        head.synthesis_digest = d
        return head

    def load_streams(self, streams, record):
        """Record i replaces the state and settings of streams[i] from the next call on.  The record must come from an engine with
        the same configuration other than numStreams and hopsPerCall, the same synthesis, numSources and historyLength.  Every record
        is checked on the host before anything is loaded, so a refusal leaves the engine and the device untouched.  Each run of consecutive
        streams is one library call (one wait for the synthesis weights, one copy, one kernel).  With a steering bank the record must
        come from a bank engine with the same dictionary, and each stream goes onto the lowest table of this engine with the content of
        the table it was on."""
        idx = self._streams(streams)
        kind = RECORD_KIND_LLBANK if self.Qe else RECORD_KIND_LL
        if record.kind != kind or record.count != len(idx):
            raise ValueError('a low-latency record of %d streams is needed (got kind %d, %d streams)' % (len(idx), record.kind, record.count))
        if record.data.shape[1] != self.record_bytes:
            lh = record.header(0).config[LLHIST_RECORD_CONFIG_HISTORY]
            raise ParameterError('records of %d bytes (history length %d) do not fit this engine (%d bytes, history length %d)'
                                 % (record.data.shape[1], lh, self.record_bytes, self.Lh))
        if self._header is None:
            self._header = self._record_header()
        want = self._header
        head = np.frombuffer(bytes(want), np.uint8)
        data = record.data.numpy()[:, :len(head)].copy()
        if self.Qd:
            # a dictionary bank's records carry the stream's K_i in the header's num_atoms: compared below, with the dictionary
            atoms = data[:, ATOMS_OFFSET:ATOMS_OFFSET + 4].copy().view(np.int32).ravel()
            data[:, ATOMS_OFFSET:ATOMS_OFFSET + 4] = head[ATOMS_OFFSET:ATOMS_OFFSET + 4]
        for i in np.flatnonzero((data != head).any(axis=1))[:1]:
            got = record.header(int(i))
            value = lambda h, f: bytes(h.config) if f == 'config' else getattr(h, f)       # noqa: E731
            bad = [f for f, _ in RecordHeader._fields_ if value(got, f) != value(want, f)]
            raise ParameterError('record %d does not fit this engine: %s differ' % (i, ', '.join(bad)))
        if self.Qd:
            dentries, entries = np.empty(len(idx), np.int32), np.empty(len(idx), np.int32)
            for i in range(len(idx)):
                got = record.header(i)
                K = int(atoms[i])
                same = [e for e in range(self.Qd) if self._dict_digests[e] == got.dictionary_digest]
                if not same:
                    raise ParameterError('record %d: no dictionary entry of this engine holds the stream\'s dictionary' % i)
                fit = [e for e in same if self._atoms[e] == K]
                if not fit:
                    raise ParameterError('record %d: the stream\'s dictionary has %d atoms, the entry holding it %d' % (i, K, self._atoms[same[0]]))
                if got.steering_digest not in self._steer_digests:
                    raise ParameterError('record %d: no steering entry of this engine has the stream\'s table' % i)
                dentries[i], entries[i] = fit[0], self._steer_digests.index(got.steering_digest)
        elif self.Qe:
            entries = np.empty(len(idx), np.int32)
            for i in range(len(idx)):
                got = record.header(i)
                if got.dictionary_digest != self._dict_digest:
                    raise ParameterError('record %d: another dictionary' % i)
                if got.steering_digest not in self._steer_digests:
                    raise ParameterError('record %d: no steering entry of this engine has the stream\'s table' % i)
                entries[i] = self._steer_digests.index(got.steering_digest)
        self._record_call('load_streams', idx, record)
        if self.Qe:
            self._assign[idx] = entries
        if self.Qd:
            self._dassign[idx] = dentries
        m = record.mirrors
        self._eps[idx], self._active[idx], self._override[idx], self._targets[idx] = m['eps'], m['active'], m['override'], m['targets']
        if self.Lh:
            self._window[idx] = m['window']

    def _export_now(self, what):
        """A per-stream assignment item (S) i32 as the device holds it, outside a call."""
        buf = self.torch.zeros((self.S,), dtype=self.torch.int32).pin_memory()
        self._state('export', 1, int(what), buf.data_ptr(), self.stream.cuda_stream)
        self.stream.synchronize()
        return buf.numpy().copy()

    def close(self):
        if self.h.h:
            for g in self._graphs.values():
                self.h.lib.gccnmf_rt_graph_destroy(self.h.h, g)
        self._graphs = {}

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def streamSignals(signals, W, expJOmegaTau, analysisWindow, synthesisWindow, hopSize, hopsPerCall=1, synthesis='lowlatency',
                  targetTDOAEpsilon=1.0, numInferenceIterations=0, use_graph=True, device=0, numSources=0, historyLength=0,
                  localizationWindow=0, steeringEntries=None, dictionaryEntries=None, **kwargs):
    """Streams a list of stereo signals (2, n_i) through one engine, one stream each, hopsPerCall hops per call, and returns the
    outputs aligned with the input: out_i[..., p] = output sample p + latency (the batch function's targetEstimateSamplesOLA), each
    (2, n_i), or (P, 2, n_i) with numSources = P.  Shorter signals are followed by silence; the engine is flushed with `latency`
    samples of silence at the end.  historyLength / localizationWindow: every stream localises over its newest
    localizationWindow frames (see set_localization).  With a steering bank (expJOmegaTau a sequence of tables), steeringEntries
    gives each signal's table (default: table 0)."""
    sig = [np.asarray(s, dtype=np.float32) for s in signals]
    eng = LowLatencyEngine(W, expJOmegaTau, analysisWindow, synthesisWindow, hopSize, numStreams=len(sig), hopsPerCall=hopsPerCall,
                           synthesis=synthesis, targetTDOAEpsilon=targetTDOAEpsilon, numInferenceIterations=numInferenceIterations,
                           device=device, numSources=numSources, historyLength=historyLength, **kwargs)
    eng.set_localization(None, localizationWindow)
    if steeringEntries is not None:
        eng.assign_steering(None, steeringEntries)
    if dictionaryEntries is not None:
        eng.assign_dictionary(None, dictionaryEntries)
    step = eng.hop * eng.C
    total = max(s.shape[1] for s in sig) + eng.latency
    total = -(-total // step) * step
    x = np.zeros((len(sig), 2, total), np.float32)
    for i, s in enumerate(sig):
        x[i, :, :s.shape[1]] = s
    y = np.concatenate([eng.process(x[:, :, p:p + step], use_graph=use_graph) for p in range(0, total, step)], axis=-1)
    eng.close()
    return [y[i, ..., eng.latency:eng.latency + s.shape[1]] for i, s in enumerate(sig)]
