"""Host side of the fused real-time block path (csrc/rt.cu, `gccnmf_rt_*` in include/gccnmf_b200.h).

One `RealtimeEngine` owns the device-resident state of one stream of audio: the 8-block input / output rings of
gccNMF/realtime/utils.py:72-116, the GCC-PHAT history and sliding-window localisation of
gccNMF/realtime/gccNMFProcessor.py:213-227, the Theano shared scalars of :196-199 -- and an instantiated CUDA graph that
takes one audio block from a pinned host buffer through H2D -> kernels -> D2H.  Per block the host does one graph
launch and one stream synchronisation; nothing else touches the device.
"""
import ctypes

import numpy as np

from .._lib import RtConfig, default_handle
from . import slotrecords

EXPORT_GCCPHAT, EXPORT_TARGET, EXPORT_ATOM_MASK, EXPORT_INPUT_SPEC, EXPORT_OUTPUT_SPEC, EXPORT_ARGMAX, EXPORT_H, EXPORT_HISTORY, \
    EXPORT_HISTORY_INDEX = range(9)

# gccNMFProcessor.py:190-199 -- what gccnmf_rt_init, gccnmf_rtm_init and gccnmf_rtm_reset_slots leave in a slot
DEFAULT_SLOT_PARAMS = dict(targetTDOAIndex=10.0, epsilon=2.0, beta=1.0, noiseFloor=0.0, mode=1, separationEnabled=True,
                           localizationEnabled=False, localizationWindowSize=6, active=True)


class RealtimeEngine(slotrecords.SlotRecords):
    def __init__(self, W, expJOmegaTau, analysisWindow, synthesisWindow, hopSize, blockSize, windowsPerBlock, historyLength=128,
                 numInferenceIterations=0, sparsityAlpha=0.0, epsilon=1e-16, seedValue=0, device=0):
        self.h = default_handle(device)
        torch = self.torch = self.h.torch
        W = np.ascontiguousarray(W, dtype=np.float32)
        E = np.ascontiguousarray(expJOmegaTau, dtype=np.complex64)
        F, K = W.shape
        N = 2 * (F - 1)
        if E.shape[0] != F or len(analysisWindow) != N or len(synthesisWindow) != N:
            raise ValueError('W (F, K), expJOmegaTau (F, D) and the windows (N = 2 (F - 1)) do not agree')
        self.F, self.K, self.N, self.D = F, K, N, E.shape[1]
        self.hop, self.B, self.nT = int(hopSize), int(blockSize), int(windowsPerBlock)
        self.cfg = RtConfig(N, self.hop, self.B, self.nT, K, self.D, int(historyLength), int(numInferenceIterations),
                            float(sparsityAlpha), float(epsilon))
        self.state_bytes = int(self.h.lib.gccnmf_rt_state_bytes(ctypes.byref(self.cfg)))
        if self.state_bytes == 0:
            raise ValueError('invalid real-time configuration')
        self.stream = torch.cuda.Stream(device=self.h.device)      # a capturable stream of its own (the legacy default stream is not)
        self.state = torch.empty(self.state_bytes, dtype=torch.uint8, device=self.h.device)
        H0 = None
        if numInferenceIterations > 0:
            # the notebook's call re-seeds on every frame (onlineSpeechEnhancement.ipynb:433 -> gccNMFFunctions.py:70,73):
            # the same (K, 2) initial coefficients for every frame
            np.random.seed(seedValue)
            H0 = (np.random.random((K, 2)).astype(np.float32) + epsilon).astype(np.float32)
        dev = lambda a: torch.as_tensor(np.ascontiguousarray(a)).to(self.h.device)      # noqa: E731
        self._const = [dev(W), dev(E.view(np.float32).reshape(F, 2 * self.D)), dev(np.asarray(analysisWindow, np.float32)),
                       dev(np.asarray(synthesisWindow, np.float32)), dev(H0) if H0 is not None else None]
        self.in_host = torch.zeros((2, self.B), dtype=torch.float32).pin_memory()
        self.out_host = torch.zeros((2, self.B), dtype=torch.float32).pin_memory()
        self.in_dev = torch.zeros((2, self.B), dtype=torch.float32, device=self.h.device)
        self.out_dev = torch.zeros((2, self.B), dtype=torch.float32, device=self.h.device)
        self.frames_in_host = torch.zeros((2, N, self.nT), dtype=torch.float32).pin_memory()
        self.frames_out_host = torch.zeros((2, N, self.nT), dtype=torch.float32).pin_memory()
        self.frames_in_dev = torch.zeros((2, N, self.nT), dtype=torch.float32, device=self.h.device)
        self.frames_out_dev = torch.zeros((2, N, self.nT), dtype=torch.float32, device=self.h.device)
        self._graph = None
        self._exports = {}
        self._record_digests = (slotrecords.windows_digest(analysisWindow, synthesisWindow), [(slotrecords.dictionary_digest(W, H0), K)],
                                [slotrecords.steering_digest(E)])
        self.reset()

    # ------------------------------------------------------------------ state
    def _check(self, status):
        self.h.check(status)

    def reset(self):
        """Zero rings / history and re-upload the constants (GCCNMFProcessor.reset, :233-236)."""
        torch = self.torch
        torch.cuda.current_stream(self.h.device).synchronize()
        c = self._const
        with torch.cuda.stream(self.stream):
            self._check(self.h.lib.gccnmf_rt_init(self.h.h, ctypes.byref(self.cfg), c[0].data_ptr(), c[1].data_ptr(), c[2].data_ptr(),
                                                  c[3].data_ptr(), c[4].data_ptr() if c[4] is not None else None,
                                                  self.state.data_ptr(), self.state_bytes, self.stream.cuda_stream))
        self.stream.synchronize()
        self._params = [dict(DEFAULT_SLOT_PARAMS)]

    def set_params(self, targetTDOAIndex=None, epsilon=2.0, beta=1.0, noiseFloor=0.0, mode=1, separationEnabled=True,
                   localizationEnabled=False, localizationWindowSize=6):
        """targetTDOAIndex=None keeps the device-resident index (loop-carried by the localisation)."""
        self._params[0].update(targetTDOAIndex=targetTDOAIndex, epsilon=epsilon, beta=beta, noiseFloor=noiseFloor, mode=mode,
                               separationEnabled=separationEnabled, localizationEnabled=localizationEnabled,
                               localizationWindowSize=localizationWindowSize)
        self._check(self.h.lib.gccnmf_rt_set_params(self.h.h, ctypes.byref(self.cfg), self.state.data_ptr(), self.state_bytes,
                                                    float(targetTDOAIndex if targetTDOAIndex is not None else 0.0),
                                                    0 if targetTDOAIndex is None else 1, float(epsilon), float(beta), float(noiseFloor), int(mode),
                                                    1 if separationEnabled else 0, 1 if localizationEnabled else 0, int(localizationWindowSize),
                                                    self.stream.cuda_stream))

    # ------------------------------------------------------------------ stream records (gccnmf_rtrec_*, slotrecords.SlotRecords)
    P = 0
    _record_dims = (1, 0, 0, 0)

    def _slots(self, slots):
        out = [int(s) for s in (slots if np.ndim(slots) else [slots])]
        if any(s != 0 for s in out):
            raise IndexError('a RealtimeEngine has the one slot 0')
        return out

    def save_streams(self):
        """The persistent state of the stream between blocks -> a StreamRecord of one record, which any real-time engine with
        this configuration (other than K_max), numSources 0, these windows and an entry holding this W, H0 and expJOmegaTau
        can load into a slot."""
        return slotrecords.SlotRecords.save_streams(self, [0])

    def load_streams(self, record):
        """The stream continues from a record of one real-time slot (of any engine form) from the next block on.  The record's
        dictionary, H0 and steering table must be this engine's."""
        return slotrecords.SlotRecords.load_streams(self, [0], record)

    def _records_loaded(self, slots, entries):
        pass

    # ------------------------------------------------------------------ per-block work
    def build_graph(self):
        if self._graph is None:
            g = ctypes.c_void_p()
            self._check(self.h.lib.gccnmf_rt_graph_create(self.h.h, ctypes.byref(self.cfg), self.state.data_ptr(), self.state_bytes,
                                                          self.in_dev.data_ptr(), self.out_dev.data_ptr(), self.in_host.data_ptr(),
                                                          self.out_host.data_ptr(), ctypes.byref(g), self.stream.cuda_stream))
            self._graph = g
        return self._graph

    def _forced(self, forcedAtomMask):
        if forcedAtomMask is None:
            return None
        m = self.torch.as_tensor(np.ascontiguousarray(forcedAtomMask, dtype=np.float64).reshape(self.K, self.nT))
        self._forced_dev = m.to(self.h.device)          # kept alive until the stream has consumed it
        return self._forced_dev.data_ptr()

    def process_block(self, block, use_graph=True, forcedAtomMask=None):
        """block (2, B) float32 (host) -> (2, B) float32 view of the pinned output buffer (overwritten by the next call):
        OverlapAddProcessor.processFrames(GCCNMFProcessor.processFrames), utils.py:99-116."""
        self.in_host.numpy()[:] = block
        if use_graph and forcedAtomMask is None:
            self._check(self.h.lib.gccnmf_rt_graph_launch(self.h.h, self.build_graph(), self.stream.cuda_stream))
        else:
            forced = self._forced(forcedAtomMask)
            self.torch.cuda.current_stream(self.h.device).synchronize()
            with self.torch.cuda.stream(self.stream):
                self.in_dev.copy_(self.in_host, non_blocking=True)
                self._check(self.h.lib.gccnmf_rt_process_block(self.h.h, ctypes.byref(self.cfg), self.state.data_ptr(), self.state_bytes,
                                                               self.in_dev.data_ptr(), self.out_dev.data_ptr(), forced, self.stream.cuda_stream))
                self.out_host.copy_(self.out_dev, non_blocking=True)
        self.stream.synchronize()
        return self.out_host.numpy()

    def process_frames(self, windowedSamples, forcedAtomMask=None):
        """windowedSamples (2, N, nT) float32 (host) -> (2, N, nT) float32: GCCNMFProcessor.processFrames (:201-231)."""
        self.frames_in_host.numpy()[:] = windowedSamples
        forced = self._forced(forcedAtomMask)
        if forced is not None:
            self.torch.cuda.current_stream(self.h.device).synchronize()
        with self.torch.cuda.stream(self.stream):
            self.frames_in_dev.copy_(self.frames_in_host, non_blocking=True)
            self._check(self.h.lib.gccnmf_rt_process_frames(self.h.h, ctypes.byref(self.cfg), self.state.data_ptr(), self.state_bytes,
                                                            self.frames_in_dev.data_ptr(), self.frames_out_dev.data_ptr(), forced,
                                                            self.stream.cuda_stream))
            self.frames_out_host.copy_(self.frames_out_dev, non_blocking=True)
        self.stream.synchronize()
        return self.frames_out_host.numpy()

    def export(self, what):
        """Host copy of one item of the state of the last block (see gccnmf_rt_export)."""
        torch = self.torch
        shapes = {EXPORT_GCCPHAT: ((self.D, self.nT), torch.float32), EXPORT_TARGET: ((1,), torch.float32),
                  EXPORT_ATOM_MASK: ((self.K, self.nT), torch.float64), EXPORT_INPUT_SPEC: ((2, self.F, self.nT), torch.complex64),
                  EXPORT_OUTPUT_SPEC: ((2, self.F, self.nT), torch.complex64), EXPORT_ARGMAX: ((self.K, self.nT), torch.int32),
                  EXPORT_H: ((self.K, 2 * self.nT), torch.float32), EXPORT_HISTORY: ((self.D, self.cfg.history_length), torch.float64),
                  EXPORT_HISTORY_INDEX: ((1,), torch.int32)}
        buf = self._exports.get(what)
        if buf is None:
            shape, dtype = shapes[what]
            buf = self._exports[what] = torch.zeros(shape, dtype=dtype).pin_memory()
        self._check(self.h.lib.gccnmf_rt_export(self.h.h, ctypes.byref(self.cfg), self.state.data_ptr(), self.state_bytes, int(what),
                                                buf.data_ptr(), self.stream.cuda_stream))
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
