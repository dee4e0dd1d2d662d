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

Bank (`W` a sequence of dictionaries and / or `expJOmegaTau` a sequence of steering tables, `gccnmf_rtbank_*`): every slot is on
one dictionary entry (its own atom count K_i <= K_max = the largest) and one steering entry (its own microphone spacing), the
reference's per-processor dictionary size / type and spacing.  `assign` moves slots between entries and `load_dictionary` /
`load_steering` rewrite an entry, from the next block on and without rebuilding the graph; the slot keeps its rings, history,
targets and parameters.  Slot s on (i, j) is bit-identical to an engine built with (W[i], expJOmegaTau[j]); its K-shaped
exports have K_i rows.
"""
import ctypes

import numpy as np

from .._lib import RtConfig, RtmSlotParams, default_handle
from . import slotrecords
from .engine import (DEFAULT_SLOT_PARAMS, EXPORT_ARGMAX, EXPORT_ATOM_MASK, EXPORT_GCCPHAT, EXPORT_H, EXPORT_HISTORY, EXPORT_HISTORY_INDEX,  # noqa: F401
                     EXPORT_INPUT_SPEC, EXPORT_OUTPUT_SPEC, EXPORT_TARGET)

# export items of an engine with sources (gccnmf_rtsep_export); EXPORT_ATOM_MASK and EXPORT_OUTPUT_SPEC are then source 0's
EXPORT_TARGETS = 9                   # (P,) int32 target TDOA indexes of the next block
EXPORT_SOURCE_MASKS = 10             # (P, K, nT) float64 one-hot atom masks
EXPORT_TARGET_VALUES = 11            # (P, K, nT) float32 gccNMF[target] per atom and frame
EXPORT_SOURCE_SPECS = 12             # (P, 2, F, nT) complex64 output spectrograms
EXPORT_STATUS = 13                   # (1,) int32, bit 0 (STATUS_FEW_PEAKS): the localisation found fewer than P peaks (sticky)
STATUS_FEW_PEAKS = 1
MAX_SOURCES = 8
EXPORT_ASSIGNMENT = 14               # (2,) int32 (dictionary, steering) entries of a slot of a bank engine
MAX_BANK_ENTRIES = 64



def check_bank_entries(values, count, num_entries, name):
    """Entries of an assign call: None, a scalar or one value per slot -> `count` ints in [-1, num_entries) (-1 keeps a slot's
    entry); anything else raises ValueError."""
    v = np.asarray(-1 if values is None else values)
    if v.size and not np.array_equal(v, np.round(v)):
        raise ValueError('%s entries must be integers' % name)
    try:
        v = np.broadcast_to(v.astype(np.int64), (count,))
    except ValueError:
        raise ValueError('%s: %d values for %d slots' % (name, v.size, count))
    if ((v < -1) | (v >= num_entries)).any():
        raise ValueError('%s entries must be in [0, %d) (or -1)' % (name, num_entries))
    return v.tolist()


def check_bank_dictionary(W, F, K_max):
    """A dictionary for a bank of K_max atoms over F bins -> float32 (F, K_i), 1 <= K_i <= K_max; anything else raises ValueError."""
    W = np.ascontiguousarray(W, dtype=np.float32)
    if W.ndim != 2 or W.shape[0] != F or not 1 <= W.shape[1] <= K_max:
        raise ValueError('dictionary (%d, 1 .. %d) expected, got %s' % (F, K_max, W.shape))
    return W


def check_bank_index(index, num_entries, name):
    if not 0 <= int(index) < num_entries:
        raise ValueError('%s entry %d outside [0, %d)' % (name, int(index), num_entries))
    return int(index)


class MultiStreamRealtimeEngine(slotrecords.SlotRecords):
    def __init__(self, W, expJOmegaTau, analysisWindow, synthesisWindow, hopSize, blockSize, windowsPerBlock, numStreams, historyLength=128,
                 numInferenceIterations=0, sparsityAlpha=0.0, epsilon=1e-16, seedValue=0, device=0, numSources=0):
        self.P = int(numSources)
        if self.P != 0 and not 2 <= self.P <= MAX_SOURCES:
            raise ValueError('numSources must be 0 (one output per slot) or in [2, %d] (got %d)' % (MAX_SOURCES, self.P))
        self.bank = isinstance(W, (list, tuple)) or isinstance(expJOmegaTau, (list, tuple))
        Ws = [np.ascontiguousarray(w, dtype=np.float32) for w in (W if isinstance(W, (list, tuple)) else [W])]
        Es = [np.ascontiguousarray(e, dtype=np.complex64) for e in (expJOmegaTau if isinstance(expJOmegaTau, (list, tuple)) else [expJOmegaTau])]
        if not Ws or not Es or (self.bank and (len(Ws) > MAX_BANK_ENTRIES or len(Es) > MAX_BANK_ENTRIES)):
            raise ValueError('a bank holds 1 .. %d dictionaries and 1 .. %d steering tables (got %d, %d)'
                             % (MAX_BANK_ENTRIES, MAX_BANK_ENTRIES, len(Ws), len(Es)))
        F = Ws[0].shape[0]
        K = max(w.shape[1] for w in Ws)
        N = 2 * (F - 1)
        D = Es[0].shape[1]
        if any(w.ndim != 2 or w.shape[0] != F for w in Ws) or any(e.ndim != 2 or e.shape != (F, D) for e in Es) or \
                len(analysisWindow) != N or len(synthesisWindow) != N:
            raise ValueError('W (F, K), expJOmegaTau (F, D) and the windows (N = 2 (F - 1)) do not agree')
        self.h = default_handle(device)
        torch = self.torch = self.h.torch
        W, E = Ws[0], Es[0]
        self.S = int(numStreams)
        self.F, self.K, self.N, self.D = F, K, N, D
        self.Qd, self.Qe = (len(Ws), len(Es)) if self.bank else (0, 0)
        self.dictionaryAtoms = [w.shape[1] for w in Ws]
        self._seed, self._epsilon, self._inference = seedValue, epsilon, int(numInferenceIterations)
        self.hop, self.B, self.nT = int(hopSize), int(blockSize), int(windowsPerBlock)
        self.cfg = RtConfig(N, self.hop, self.B, self.nT, K, self.D, int(historyLength), int(numInferenceIterations),
                            float(sparsityAlpha), float(epsilon))
        if self.bank:
            self.state_bytes = int(self.h.lib.gccnmf_rtbank_state_bytes(ctypes.byref(self.cfg), self.S, self.P, self.Qd, self.Qe))
        else:
            self.state_bytes = int(self.h.lib.gccnmf_rtsep_state_bytes(ctypes.byref(self.cfg), self.S, self.P) if self.P else
                                   self.h.lib.gccnmf_rtm_state_bytes(ctypes.byref(self.cfg), self.S))
        if self.state_bytes == 0:
            raise ValueError('invalid real-time configuration or number of streams (%d)' % self.S)
        self.stream = torch.cuda.Stream(device=self.h.device)
        self.state = torch.empty(self.state_bytes, dtype=torch.uint8, device=self.h.device)
        H0 = self._h0(K)
        dev = self._dev
        self._const = [dev(W), dev(E.view(np.float32).reshape(F, 2 * self.D)), dev(np.asarray(analysisWindow, np.float32)),
                       dev(np.asarray(synthesisWindow, np.float32)), dev(H0) if H0 is not None else None]
        if self.bank:                           # device copies of every entry, read by init
            self._dicts = [(dev(w), dev(self._h0(w.shape[1])) if H0 is not None else None) for w in Ws]
            self._steers = [dev(e.view(np.float32).reshape(F, 2 * self.D)) for e in Es]
        # content digests of the windows and of every entry, which stream records name their entries by
        self._record_digests = (slotrecords.windows_digest(analysisWindow, synthesisWindow),
                                [(slotrecords.dictionary_digest(w, self._h0(w.shape[1])), w.shape[1]) for w in Ws],
                                [slotrecords.steering_digest(e) for e in Es])
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
        self._assign = [[0, 0] for _ in range(S)]
        self._block_atoms = [None] * S          # K_i of the last block each slot computed (None: none since init / reset)
        self.reset()

    # ------------------------------------------------------------------ state
    def _h0(self, K):
        """The seeded (K, 2) initial coefficients of RealtimeEngine, or None without inference."""
        if self._inference <= 0:
            return None
        np.random.seed(self._seed)
        return (np.random.random((K, 2)).astype(np.float32) + self._epsilon).astype(np.float32)

    def _dev(self, a):
        return self.torch.as_tensor(np.ascontiguousarray(a)).to(self.h.device)

    def _check(self, status):
        self.h.check(status)

    def _abi(self, name, *args):
        """gccnmf_rtm_<name>(h, cfg, S, state, state_bytes, *args), gccnmf_rtsep_<name>(h, cfg, S, P, ...) with sources, or
        gccnmf_rtbank_<name>(h, cfg, S, P, Qd, Qe, ...) with a bank."""
        if self.bank:
            fn, head = getattr(self.h.lib, 'gccnmf_rtbank_' + name), (self.S, self.P, self.Qd, self.Qe)
        elif self.P:
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
            if self.bank:
                ptrs = lambda ts: (ctypes.c_void_p * len(ts))(*[t.data_ptr() if t is not None else None for t in ts])     # noqa: E731
                Ks = (ctypes.c_int * self.Qd)(*self.dictionaryAtoms)
                H0s = ptrs([d[1] for d in self._dicts]) if c[4] is not None else None
                self._abi('init', ptrs([d[0] for d in self._dicts]), Ks, H0s, ptrs(self._steers), c[2].data_ptr(), c[3].data_ptr(),
                          self.stream.cuda_stream)
            elif self.P:
                self._check(self.h.lib.gccnmf_rtsep_init(self.h.h, ctypes.byref(self.cfg), self.S, self.P, *args))
            else:
                self._check(self.h.lib.gccnmf_rtm_init(self.h.h, ctypes.byref(self.cfg), self.S, *args))
        self.stream.synchronize()
        self._params = [dict(DEFAULT_SLOT_PARAMS) for _ in range(self.S)]
        self._assign = [[0, 0] for _ in range(self.S)]
        self._block_atoms = [None] * self.S

    def reset_slots(self, slots):
        """The given slots back to a fresh state; the others are untouched.  Stream-ordered: the graph is kept."""
        slots = self._slots(slots)
        for first, count in self._runs(slots):
            self._abi('reset_slots', first, count, self.stream.cuda_stream)
        for s in slots:
            self._params[s] = dict(DEFAULT_SLOT_PARAMS)
            self._assign[s] = [0, 0]
            self._block_atoms[s] = None

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

    # ------------------------------------------------------------------ bank
    def _need_bank(self):
        if not self.bank:
            raise ValueError('this engine has no bank: pass sequences of dictionaries / steering tables to use one')

    def assign(self, slots, dictionary=None, steering=None):
        """Puts the given slots on dictionary entry `dictionary` and steering entry `steering` (scalars or one value per slot;
        None or -1 keeps a slot's entry) from the next block on; rings, history, targets and parameters stay."""
        self._need_bank()
        slots = self._slots(slots)
        if len(set(slots)) != len(slots):
            raise ValueError('duplicate slots')
        cols = [dict(zip(slots, check_bank_entries(v, len(slots), n, name)))
                for v, n, name in ((dictionary, self.Qd, 'dictionary'), (steering, self.Qe, 'steering'))]
        for s in slots:
            for c in range(2):
                if cols[c][s] >= 0:
                    self._assign[s][c] = cols[c][s]
        for first, count in self._runs(slots):
            d = np.ascontiguousarray([cols[0][s] for s in range(first, first + count)], dtype=np.int32)
            e = np.ascontiguousarray([cols[1][s] for s in range(first, first + count)], dtype=np.int32)
            p32 = ctypes.POINTER(ctypes.c_int32)
            self._abi('assign', first, count, d.ctypes.data_as(p32), e.ctypes.data_as(p32), self.stream.cuda_stream)

    def assignment(self, slot):
        """(dictionary, steering) entries of a slot (host mirror of EXPORT_ASSIGNMENT)."""
        self._need_bank()
        return tuple(self._assign[self._slots(slot)[0]])

    def load_dictionary(self, index, W):
        """Replaces dictionary entry `index` by W (F, K_i), K_i <= K_max, from the next block on (the seeded H0 of K_i with
        inference).  The graph is kept."""
        self._need_bank()
        W = check_bank_dictionary(W, self.F, self.K)
        index = check_bank_index(index, self.Qd, 'dictionary')
        H0 = self._h0(W.shape[1])
        entry = (self._dev(W), self._dev(H0) if H0 is not None else None)
        self.torch.cuda.current_stream(self.h.device).synchronize()
        self._abi('load_dictionary', int(index), entry[0].data_ptr(), W.shape[1], entry[1].data_ptr() if entry[1] is not None else None,
                  self.stream.cuda_stream)
        self.stream.synchronize()
        self._dicts[index] = entry
        self.dictionaryAtoms[index] = W.shape[1]
        self._record_digests[1][index] = (slotrecords.dictionary_digest(W, H0), W.shape[1])

    def load_steering(self, index, expJOmegaTau):
        """Replaces steering entry `index` by expJOmegaTau (F, D) from the next block on.  The graph is kept."""
        self._need_bank()
        E = np.ascontiguousarray(expJOmegaTau, dtype=np.complex64)
        if E.shape != (self.F, self.D):
            raise ValueError('steering table (%d, %d) expected, got %s' % (self.F, self.D, E.shape))
        index = check_bank_index(index, self.Qe, 'steering')
        entry = self._dev(E.view(np.float32).reshape(self.F, 2 * self.D))
        self.torch.cuda.current_stream(self.h.device).synchronize()
        self._abi('load_steering', int(index), entry.data_ptr(), self.stream.cuda_stream)
        self.stream.synchronize()
        self._steers[index] = entry
        self._record_digests[2][index] = slotrecords.steering_digest(E)

    # ------------------------------------------------------------------ stream records (gccnmf_rtrec_*, slotrecords.SlotRecords)
    @property
    def _record_dims(self):
        return (self.S, self.P, self.Qd, self.Qe)

    def _records_loaded(self, slots, entries):
        """After a load: the slots are on the entries the records mapped to.  _block_atoms stays: K-shaped exports describe the
        destination slot's last block until the next one."""
        for s, e in zip(slots, entries):
            self._assign[s] = list(e)

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
                self._abi('process_block', self.in_dev.data_ptr(), self.out_dev.data_ptr(), *(() if self.P and not self.bank else (forced,)),
                          self.stream.cuda_stream)
                self.out_host.copy_(self.out_dev, non_blocking=True)
        self.stream.synchronize()
        self._computed()
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
            self._abi('process_frames', self.frames_in_dev.data_ptr(), self.frames_out_dev.data_ptr(), *(() if self.P and not self.bank else (forced,)),
                      self.stream.cuda_stream)
            self.frames_out_host.copy_(self.frames_out_dev, non_blocking=True)
        self.stream.synchronize()
        self._computed()
        return self.frames_out_host.numpy()

    def _computed(self):
        """Every active slot has computed a block on its current dictionary entry."""
        if self.bank:
            for s in range(self.S):
                if self._params[s]['active']:
                    self._block_atoms[s] = self.dictionaryAtoms[self._assign[s][0]]

    def export(self, slot, what):
        """Host copy of one item of slot `slot`'s state after the last block (items as RealtimeEngine.export; with sources also
        EXPORT_TARGETS .. EXPORT_STATUS; with a bank EXPORT_ASSIGNMENT, and the K-shaped items have the K_i of the block they
        were computed in: an assign or load takes effect from the next block)."""
        torch = self.torch
        slot = self._slots(slot)[0]
        K = self.K
        if self.bank:       # K_i of the block the items were computed in, or of the slot's entry before its first block
            K = self._block_atoms[slot] or self.dictionaryAtoms[self._assign[slot][0]]
        shapes = {EXPORT_GCCPHAT: ((self.D, self.nT), torch.float32), EXPORT_TARGET: ((1,), torch.float32),
                  EXPORT_ATOM_MASK: ((K, self.nT), torch.float64), EXPORT_INPUT_SPEC: ((2, self.F, self.nT), torch.complex64),
                  EXPORT_OUTPUT_SPEC: ((2, self.F, self.nT), torch.complex64), EXPORT_ARGMAX: ((K, self.nT), torch.int32),
                  EXPORT_H: ((K, 2 * self.nT), torch.float32), EXPORT_HISTORY: ((self.D, self.cfg.history_length), torch.float64),
                  EXPORT_HISTORY_INDEX: ((1,), torch.int32)}
        if self.bank:
            shapes[EXPORT_ASSIGNMENT] = ((2,), torch.int32)
        if self.P:
            P, nT = self.P, self.nT
            shapes.update({EXPORT_TARGETS: ((P,), torch.int32), EXPORT_SOURCE_MASKS: ((P, K, nT), torch.float64),
                           EXPORT_TARGET_VALUES: ((P, K, nT), torch.float32), EXPORT_SOURCE_SPECS: ((P, 2, self.F, nT), torch.complex64),
                           EXPORT_STATUS: ((1,), torch.int32)})
        if what not in shapes:
            raise ValueError('unknown export item %r' % (what,))
        shape, dtype = shapes[what]
        buf = self._exports.get((what, shape))
        if buf is None:
            buf = self._exports[(what, shape)] = torch.zeros(shape, dtype=dtype).pin_memory()
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
