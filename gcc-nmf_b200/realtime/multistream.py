"""Many independent audio streams through one real-time engine (csrc/rt.cu, `gccnmf_rtm_*` in include/gccnmf_b200.h).

A `MultiStreamRealtimeEngine` holds S slots in one device state buffer.  The slots share the dictionary W, the steering vectors
expJOmegaTau, the analysis / synthesis windows and the inference seed H0; each slot has the rings, GCC-PHAT history, target TDOA
index and parameters one `RealtimeEngine` has, plus an `active` flag.  One audio block of every slot is one CUDA graph launch (H2D
of the (S, 2, B) pinned input -> the same kernels as one stream, each launched once for all slots -> D2H) and one stream
synchronisation.  Slot s is bit-identical to a `RealtimeEngine` fed the same blocks with the same parameters.

Join / leave without rebuilding the graph: `set_active(slots, False)` makes the kernels skip a slot (its output block is zeros, its
input block is ignored, its state stays as it was); `reset_slots(slots)` puts slots back to the state of a fresh engine.

Sources (`numSources` = P >= 2, `gccnmf_rtsep_*`): every slot is separated into P sources, one per target TDOA index (the
reference's TARGET_MODE_MULTIPLE, gccNMFFunctions.py:118-143 per block), and every call returns P output blocks per slot.  The
targets come from `set_targets` or, with localisation on, from the P largest peaks of the windowed GCC-PHAT mean (the targets of
the next block).  Source q of a slot computes bit for bit what a single-target slot computes when it is fed the exported mask of
source q as its atom mask; the P masks partition the atoms, so the P outputs sum to the separation-off output.
"""
import ctypes

import numpy as np

from .._lib import RtConfig, RtmSlotParams, default_handle
from .engine import (EXPORT_ARGMAX, EXPORT_ATOM_MASK, EXPORT_GCCPHAT, EXPORT_H, EXPORT_HISTORY, EXPORT_HISTORY_INDEX,  # noqa: F401
                     EXPORT_INPUT_SPEC, EXPORT_OUTPUT_SPEC, EXPORT_TARGET)

# export items of an engine with sources (gccnmf_rtsep_export); EXPORT_ATOM_MASK and EXPORT_OUTPUT_SPEC are then source 0's
EXPORT_TARGETS = 9                   # (P,) int32 target TDOA indexes of the next block
EXPORT_SOURCE_MASKS = 10             # (P, K, nT) float64 one-hot atom masks
EXPORT_TARGET_VALUES = 11            # (P, K, nT) float32 gccNMF[target] per atom and frame
EXPORT_SOURCE_SPECS = 12             # (P, 2, F, nT) complex64 output spectrograms
EXPORT_STATUS = 13                   # (1,) int32, bit 0 (STATUS_FEW_PEAKS): the localisation found fewer than P peaks (sticky)
STATUS_FEW_PEAKS = 1
MAX_SOURCES = 8

# gccNMFProcessor.py:190-199 -- what gccnmf_rtm_init and gccnmf_rtm_reset_slots leave in a slot
DEFAULT_SLOT_PARAMS = dict(targetTDOAIndex=10.0, epsilon=2.0, beta=1.0, noiseFloor=0.0, mode=1, separationEnabled=True,
                           localizationEnabled=False, localizationWindowSize=6, active=True)


class MultiStreamRealtimeEngine(object):
    def __init__(self, W, expJOmegaTau, analysisWindow, synthesisWindow, hopSize, blockSize, windowsPerBlock, numStreams, historyLength=128,
                 numInferenceIterations=0, sparsityAlpha=0.0, epsilon=1e-16, seedValue=0, device=0, numSources=0):
        self.P = int(numSources)
        if self.P != 0 and not 2 <= self.P <= MAX_SOURCES:
            raise ValueError('numSources must be 0 (one output per slot) or in [2, %d] (got %d)' % (MAX_SOURCES, self.P))
        self.h = default_handle(device)
        torch = self.torch = self.h.torch
        W = np.ascontiguousarray(W, dtype=np.float32)
        E = np.ascontiguousarray(expJOmegaTau, dtype=np.complex64)
        F, K = W.shape
        N = 2 * (F - 1)
        if E.shape[0] != F or len(analysisWindow) != N or len(synthesisWindow) != N:
            raise ValueError('W (F, K), expJOmegaTau (F, D) and the windows (N = 2 (F - 1)) do not agree')
        self.S = int(numStreams)
        self.F, self.K, self.N, self.D = F, K, N, E.shape[1]
        self.hop, self.B, self.nT = int(hopSize), int(blockSize), int(windowsPerBlock)
        self.cfg = RtConfig(N, self.hop, self.B, self.nT, K, self.D, int(historyLength), int(numInferenceIterations),
                            float(sparsityAlpha), float(epsilon))
        self.state_bytes = int(self.h.lib.gccnmf_rtsep_state_bytes(ctypes.byref(self.cfg), self.S, self.P) if self.P else
                               self.h.lib.gccnmf_rtm_state_bytes(ctypes.byref(self.cfg), self.S))
        if self.state_bytes == 0:
            raise ValueError('invalid real-time configuration or number of streams (%d)' % self.S)
        self.stream = torch.cuda.Stream(device=self.h.device)
        self.state = torch.empty(self.state_bytes, dtype=torch.uint8, device=self.h.device)
        H0 = None
        if numInferenceIterations > 0:          # the same seeded (K, 2) initial coefficients as RealtimeEngine
            np.random.seed(seedValue)
            H0 = (np.random.random((K, 2)).astype(np.float32) + epsilon).astype(np.float32)
        dev = lambda a: torch.as_tensor(np.ascontiguousarray(a)).to(self.h.device)      # noqa: E731
        self._const = [dev(W), dev(E.view(np.float32).reshape(F, 2 * self.D)), dev(np.asarray(analysisWindow, np.float32)),
                       dev(np.asarray(synthesisWindow, np.float32)), dev(H0) if H0 is not None else None]
        S = self.S
        per_slot = (self.P,) if self.P else ()          # outputs: (S, [P,] 2, ...)
        self.in_host = torch.zeros((S, 2, self.B), dtype=torch.float32).pin_memory()
        self.out_host = torch.zeros((S,) + per_slot + (2, self.B), dtype=torch.float32).pin_memory()
        self.in_dev = torch.zeros((S, 2, self.B), dtype=torch.float32, device=self.h.device)
        self.out_dev = torch.zeros((S,) + per_slot + (2, self.B), dtype=torch.float32, device=self.h.device)
        self.frames_in_host = torch.zeros((S, 2, N, self.nT), dtype=torch.float32).pin_memory()
        self.frames_out_host = torch.zeros((S,) + per_slot + (2, N, self.nT), dtype=torch.float32).pin_memory()
        self.frames_in_dev = torch.zeros((S, 2, N, self.nT), dtype=torch.float32, device=self.h.device)
        self.frames_out_dev = torch.zeros((S,) + per_slot + (2, N, self.nT), dtype=torch.float32, device=self.h.device)
        self._graph = None
        self._exports = {}
        self._params = [dict(DEFAULT_SLOT_PARAMS) for _ in range(S)]      # host mirror of what each slot holds
        self.reset()

    # ------------------------------------------------------------------ state
    def _check(self, status):
        self.h.check(status)

    def _abi(self, name, *args):
        """gccnmf_rtm_<name>(h, cfg, S, state, state_bytes, *args), or gccnmf_rtsep_<name>(h, cfg, S, P, ...) with sources."""
        if self.P:
            fn, head = getattr(self.h.lib, 'gccnmf_rtsep_' + name), (self.S, self.P)
        else:
            fn, head = getattr(self.h.lib, 'gccnmf_rtm_' + name), (self.S,)
        self._check(fn(self.h.h, ctypes.byref(self.cfg), *head, self.state.data_ptr(), self.state_bytes, *args))

    def _slots(self, slots):
        if isinstance(slots, slice):
            out = list(range(self.S))[slots]
        elif np.ndim(slots) == 0:
            out = [int(slots)]
        else:
            out = [int(s) for s in slots]
        for s in out:
            if not 0 <= s < self.S:
                raise IndexError('slot %d outside [0, %d)' % (s, self.S))
        return out

    @staticmethod
    def _runs(slots):
        """Sorted distinct slots -> [(first, count)] of consecutive runs."""
        runs = []
        for s in sorted(set(slots)):
            if runs and runs[-1][0] + runs[-1][1] == s:
                runs[-1][1] += 1
            else:
                runs.append([s, 1])
        return runs

    def reset(self):
        """Every slot back to a fresh state (zeroed rings and history, default parameters, active)."""
        torch = self.torch
        torch.cuda.current_stream(self.h.device).synchronize()
        c = self._const
        with torch.cuda.stream(self.stream):
            args = (c[0].data_ptr(), c[1].data_ptr(), c[2].data_ptr(), c[3].data_ptr(), c[4].data_ptr() if c[4] is not None else None,
                    self.state.data_ptr(), self.state_bytes, self.stream.cuda_stream)
            if self.P:
                self._check(self.h.lib.gccnmf_rtsep_init(self.h.h, ctypes.byref(self.cfg), self.S, self.P, *args))
            else:
                self._check(self.h.lib.gccnmf_rtm_init(self.h.h, ctypes.byref(self.cfg), self.S, *args))
        self.stream.synchronize()
        self._params = [dict(DEFAULT_SLOT_PARAMS) for _ in range(self.S)]

    def reset_slots(self, slots):
        """The given slots back to a fresh state; the others are untouched.  Stream-ordered: the graph is kept."""
        slots = self._slots(slots)
        for first, count in self._runs(slots):
            self._abi('reset_slots', first, count, self.stream.cuda_stream)
        for s in slots:
            self._params[s] = dict(DEFAULT_SLOT_PARAMS)

    def _send(self, slots, set_target):
        for first, count in self._runs(slots):
            arr = (RtmSlotParams * count)()
            for i in range(count):
                p = self._params[first + i]
                t = p['targetTDOAIndex']
                arr[i] = RtmSlotParams(float(t if t is not None else 0.0), 1 if (set_target and t is not None) else 0, float(p['epsilon']),
                                       float(p['beta']), float(p['noiseFloor']), int(p['mode']), 1 if p['separationEnabled'] else 0,
                                       1 if p['localizationEnabled'] else 0, int(p['localizationWindowSize']), 1 if p['active'] else 0)
            self._abi('set_params', first, count, arr, self.stream.cuda_stream)

    def set_params(self, slots, targetTDOAIndex=None, epsilon=2.0, beta=1.0, noiseFloor=0.0, mode=1, separationEnabled=True,
                   localizationEnabled=False, localizationWindowSize=6):
        """As RealtimeEngine.set_params, for the given slots.  Every argument is a scalar or one value per slot (in the order of
        `slots`); targetTDOAIndex None keeps the device-resident index of a slot.  The slots' `active` flags are kept."""
        slots = self._slots(slots)
        if len(set(slots)) != len(slots):
            raise ValueError('duplicate slots')
        args = dict(targetTDOAIndex=targetTDOAIndex, epsilon=epsilon, beta=beta, noiseFloor=noiseFloor, mode=mode,
                    separationEnabled=separationEnabled, localizationEnabled=localizationEnabled, localizationWindowSize=localizationWindowSize)
        for i, s in enumerate(slots):
            for name, v in args.items():
                if isinstance(v, (list, tuple, np.ndarray)):
                    if len(v) != len(slots):
                        raise ValueError('%s: %d values for %d slots' % (name, len(v), len(slots)))
                    v = v[i]
                self._params[s][name] = v
        self._send(slots, True)

    def set_active(self, slots, active):
        """Skip (False) or process (True) the given slots from the next block on."""
        slots = self._slots(slots)
        for s in slots:
            self._params[s]['active'] = bool(active)
        self._send(slots, False)

    def is_active(self, slot):
        return bool(self._params[self._slots(slot)[0]]['active'])

    def set_targets(self, slots, indexes):
        """Target TDOA indexes of the given slots' P sources from the next block on (GCCNMFProcessor.setTargetTDOAIndexes):
        indexes (len(slots), P) or one row of P for every slot, integers in [0, D); -1 keeps that source's target.  With
        localisation on, the next block's localisation replaces them again."""
        if not self.P:
            raise ValueError('set_targets needs an engine with numSources >= 2')
        slots = self._slots(slots)
        if len(set(slots)) != len(slots):
            raise ValueError('duplicate slots')
        idx = np.asarray(indexes)
        if idx.size and not np.array_equal(idx, np.round(idx)):
            raise ValueError('target TDOA indexes must be integers')
        idx = np.broadcast_to(idx.astype(np.int64), (len(slots), self.P))
        rows = dict(zip(slots, idx))
        for first, count in self._runs(slots):
            arr = np.ascontiguousarray([rows[s] for s in range(first, first + count)], dtype=np.int32)
            self._abi('set_targets', first, count, arr.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), self.stream.cuda_stream)

    # ------------------------------------------------------------------ per-block work
    def build_graph(self):
        if self._graph is None:
            g = ctypes.c_void_p()
            self._abi('graph_create', self.in_dev.data_ptr(), self.out_dev.data_ptr(), self.in_host.data_ptr(), self.out_host.data_ptr(),
                      ctypes.byref(g), self.stream.cuda_stream)
            self._graph = g
        return self._graph

    def _forced(self, forcedAtomMask):
        if forcedAtomMask is None:
            return None
        if self.P:
            raise ValueError('forcedAtomMask: the sources of an engine with numSources >= 2 take their masks from their targets')
        m = self.torch.as_tensor(np.ascontiguousarray(forcedAtomMask, dtype=np.float64).reshape(self.S, self.K, self.nT))
        self._forced_dev = m.to(self.h.device)          # kept alive until the stream has consumed it
        return self._forced_dev.data_ptr()

    def process_blocks(self, blocks, use_graph=True, forcedAtomMask=None):
        """blocks (S, 2, B) float32 (host) -> (S, 2, B) float32 view of the pinned output buffer (overwritten by the next call);
        (S, P, 2, B) with sources.  forcedAtomMask (S, K, nT) float64 replaces the per-atom TDOA decisions of every slot (kernel by
        kernel, no graph; not with sources)."""
        self.in_host.numpy()[:] = blocks
        if use_graph and forcedAtomMask is None:
            self._check(self.h.lib.gccnmf_rt_graph_launch(self.h.h, self.build_graph(), self.stream.cuda_stream))
        else:
            forced = self._forced(forcedAtomMask)
            self.torch.cuda.current_stream(self.h.device).synchronize()
            with self.torch.cuda.stream(self.stream):
                self.in_dev.copy_(self.in_host, non_blocking=True)
                self._abi('process_block', self.in_dev.data_ptr(), self.out_dev.data_ptr(), *(() if self.P else (forced,)),
                          self.stream.cuda_stream)
                self.out_host.copy_(self.out_dev, non_blocking=True)
        self.stream.synchronize()
        return self.out_host.numpy()

    def process_frames(self, windowedSamples, forcedAtomMask=None):
        """windowedSamples (S, 2, N, nT) float32 (host) -> (S, 2, N, nT) float32 ((S, P, 2, N, nT) with sources):
        GCCNMFProcessor.processFrames per slot."""
        self.frames_in_host.numpy()[:] = windowedSamples
        forced = self._forced(forcedAtomMask)
        if forced is not None:
            self.torch.cuda.current_stream(self.h.device).synchronize()
        with self.torch.cuda.stream(self.stream):
            self.frames_in_dev.copy_(self.frames_in_host, non_blocking=True)
            self._abi('process_frames', self.frames_in_dev.data_ptr(), self.frames_out_dev.data_ptr(), *(() if self.P else (forced,)),
                      self.stream.cuda_stream)
            self.frames_out_host.copy_(self.frames_out_dev, non_blocking=True)
        self.stream.synchronize()
        return self.frames_out_host.numpy()

    def export(self, slot, what):
        """Host copy of one item of slot `slot`'s state after the last block (items as RealtimeEngine.export; with sources also
        EXPORT_TARGETS .. EXPORT_STATUS)."""
        torch = self.torch
        slot = self._slots(slot)[0]
        shapes = {EXPORT_GCCPHAT: ((self.D, self.nT), torch.float32), EXPORT_TARGET: ((1,), torch.float32),
                  EXPORT_ATOM_MASK: ((self.K, self.nT), torch.float64), EXPORT_INPUT_SPEC: ((2, self.F, self.nT), torch.complex64),
                  EXPORT_OUTPUT_SPEC: ((2, self.F, self.nT), torch.complex64), EXPORT_ARGMAX: ((self.K, self.nT), torch.int32),
                  EXPORT_H: ((self.K, 2 * self.nT), torch.float32), EXPORT_HISTORY: ((self.D, self.cfg.history_length), torch.float64),
                  EXPORT_HISTORY_INDEX: ((1,), torch.int32)}
        if self.P:
            P, K, nT = self.P, self.K, self.nT
            shapes.update({EXPORT_TARGETS: ((P,), torch.int32), EXPORT_SOURCE_MASKS: ((P, K, nT), torch.float64),
                           EXPORT_TARGET_VALUES: ((P, K, nT), torch.float32), EXPORT_SOURCE_SPECS: ((P, 2, self.F, nT), torch.complex64),
                           EXPORT_STATUS: ((1,), torch.int32)})
        if what not in shapes:
            raise ValueError('unknown export item %r' % (what,))
        buf = self._exports.get(what)
        if buf is None:
            shape, dtype = shapes[what]
            buf = self._exports[what] = torch.zeros(shape, dtype=dtype).pin_memory()
        self._abi('export', slot, int(what), buf.data_ptr(), self.stream.cuda_stream)
        self.stream.synchronize()
        return buf.numpy().copy()

    def close(self):
        if self._graph is not None and self.h.h:
            self.h.lib.gccnmf_rt_graph_destroy(self.h.h, self._graph)
            self._graph = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
