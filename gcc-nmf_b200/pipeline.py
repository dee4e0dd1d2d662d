"""Device-resident GCC-NMF pipelines: the whole hot path (STFT -> PHAT angular spectrogram ->
KL-NMF -> per-atom TDOA mask -> masked reconstruction -> iSTFT) with every intermediate kept in
HBM.  Two flows, both in the reference's stage order:

  * `separate`  -- gccNMF/runGCCNMF.py:36-52 (S targets, one-hot masks over the target TDOAs)
  * `enhance`   -- notebooks/offlineSpeechEnhancement.ipynb cells 12-41 (one target, argmax over all
                   hypothesis TDOAs, mask = within 5 % of the TDOA range of the target)

All intermediates live in persistent per-shape device buffers owned by the pipeline (allocated on the
first call of a shape, i.e. at plan time): the dict a flow returns holds views of them, valid until the
next call on the same pipeline.  Steady-state calls therefore never enter the CUDA allocator.

Only two things happen on the host, as in gccNMFFunctions.py: the D-element peak picking
(scipy.signal.argrelmax) and the plan-time constants (window, exp(-2 pi i f tau) table in float64,
seeded numpy draw of the NMF initial values -- a function of shape and seed only, gccNMFFunctions.py:70-73).

With localizationWindow=w every flow follows a moving talker instead: each frame takes its targets from the nanmean of the
angular spectrogram over its newest w frames (gccnmf_window_targets, on the device, no host wait), and the result gains
frameTargetTDOAIndexes (T, S), windowMeans (D, T) and status (bit 0: some frame held earlier targets; information, not an error).
"""
import weakref

import numpy as np

from . import gccNMFFunctions as fn
from ._lib import Handle


class _BufferOwner(object):
    """Identity token for Handle.buffer keys (an id() can be reused after garbage collection; an object cannot)."""


class GCCNMFPipeline(object):
    def __init__(self, sampleRate, windowSize, hopSize, numTDOAs, microphoneSeparationInMetres,
                 dictionarySize, numIterations, sparsityAlpha=0.0, epsilon=1e-16, seedValue=0,
                 targetTDOAWindowSizePercent=0.05, device=0, handle=None, windowFunction=np.hanning):
        self.h = handle if handle is not None else Handle(device)
        self.torch = self.h.torch
        self._token = _BufferOwner()                    # owner of this pipeline's persistent device buffers (released with it)
        weakref.finalize(self, self.h.release, self._token)
        self.sampleRate, self.N, self.hop, self.D = sampleRate, int(windowSize), int(hopSize), int(numTDOAs)
        self.micSep = microphoneSeparationInMetres
        self.K, self.I = int(dictionarySize), int(numIterations)
        self.alpha, self.eps, self.seed = float(sparsityAlpha), float(epsilon), seedValue
        self.windowPercent = targetTDOAWindowSizePercent
        self.F = self.N // 2 + 1
        self.frequenciesInHz = fn.getFrequenciesInHz(sampleRate, self.F)
        self.hypothesisTDOAs = fn.getTDOAsInSeconds(microphoneSeparationInMetres, self.D)
        self.E_host = np.ascontiguousarray(fn.getExpJOmegaTau(self.frequenciesInHz, self.hypothesisTDOAs))
        self.window = self.h.to_device(np.hanning(self.N))          # float64, librosaSTFT.py:139 (the STFT ignores windowFunction, gccNMFFunctions.py:65)
        # the iSTFT honours it (gccNMFFunctions.py:161 -> librosaSTFT.py:264-270)
        synthesis = windowFunction(self.N) if callable(windowFunction) else np.asarray(windowFunction)
        self.synthesisWindow = self.window if windowFunction is np.hanning else self.h.to_device(np.ascontiguousarray(synthesis, dtype=np.float64))
        self.E = self.h.to_device(self.E_host)
        self._init = {}
        self.stage_events = None

    # ------------------------------------------------------------------ plan-time constants
    def num_frames(self, numSamples):
        return 1 + (numSamples - self.N) // self.hop

    def nmf_init(self, T2):
        """Seeded initial (W0, H0) on the device (gccNMFFunctions.py:70-73).  W0 does not depend on T2, and H0 for T2 frames is the
        first K T2 values the seeded stream draws after W0, so one draw at the longest T2 seen so far serves every shorter clip:
        clips of any mix of lengths never redraw it."""
        key = (self.F, self.K, self.seed, self.eps)
        entry = self._init.get(key)
        if entry is None or entry[2] < T2:
            W0, H0 = fn._seededInit(self.F, T2, self.K, self.eps, self.seed)
            entry = (self.h.to_device(W0), self.h.to_device(H0).reshape(-1), T2)
            self._init = {key: entry}
        return entry[0], entry[1][:self.K * T2].view(self.K, T2)

    # ------------------------------------------------------------------ timing hooks
    def _mark(self, name):
        if self.stage_events is not None:
            ev = self.torch.cuda.Event(enable_timing=True)
            ev.record()
            self.stage_events.append((name, ev))

    def stage_times_ms(self):
        """Device time per stage in ms (a batch flow runs the per-clip stages once per clip: their times are summed)."""
        ev = self.stage_events
        times = {}
        for i in range(len(ev) - 1):
            times[ev[i + 1][0]] = times.get(ev[i + 1][0], 0.0) + ev[i][1].elapsed_time(ev[i + 1][1])
        return times

    # ------------------------------------------------------------------ shared front half
    def _front(self, samples):
        """STFT, coherence + angular spectrogram (+ async copy of its mean), KL-NMF."""
        h, torch = self.h, self.torch
        self._mark('start')
        key = self._token
        X, V = h.stft(samples, self.window, self.N, self.hop, conjugate=True, want_V=True, out_key=key)
        self._mark('stft')
        coh, ang, mean = h.phat_angspec(X, self.E, out_key=key)
        if getattr(self, '_mean_host', None) is None:
            self._mean_host = torch.empty(self.D, dtype=torch.float64, pin_memory=True)
        mean_host = self._mean_host
        mean_host.copy_(mean, non_blocking=True)
        mean_ready = torch.cuda.Event()
        mean_ready.record()
        self._mark('angular')
        W0, H0 = self.nmf_init(V.shape[1])
        W, H = h.buffer((key, 'W'), W0.shape, W0.dtype), h.buffer((key, 'H'), H0.shape, H0.dtype)
        W.copy_(W0)
        H.copy_(H0)
        h.klnmf(V, W, H, self.I, self.alpha, self.eps, update_W=True)
        self._mark('nmf')
        return dict(X=X, V=V, coherence=coh, angularSpectrogram=ang, meanAngularSpectrum=mean, W=W, H=H,
                    _mean_host=mean_host, _mean_ready=mean_ready)

    def _front_batch(self, samples):
        """_front for B clips (B, 2, n): the STFT of each clip into one (2B, F, T) spectrogram and one (B, F, 2T) V stack (the
        STFT entry takes one stereo pair per call), the angular spectrum per clip with one event for all B means, one batched
        KL-NMF over the stack.  A list of (2, n_b) recordings of any lengths: each clip's STFT into its own buffers, one ragged
        KL-NMF over them.  Returns one _front dict per clip (views of batch buffers)."""
        h, torch = self.h, self.torch
        ragged = isinstance(samples, (list, tuple))
        if ragged and not samples:
            return []
        for x in (samples if ragged else [samples[0]] if len(samples) else []):
            if x.dim() != 2 or x.shape[0] != 2:
                raise ValueError('samples must be (B, 2, n) or a list of (2, n_b), got a clip of shape %s' % (tuple(x.shape),))
        B = len(samples)
        self._mark('start')
        key = self._token
        F = self.F
        if ragged:
            Xs, Vs = [], []
            for b, x in enumerate(samples):
                T = self.num_frames(x.shape[1])
                Xb = h.buffer((key, 'clip', b, 'X'), (2, F, T), torch.complex64)
                Vb = h.buffer((key, 'clip', b, 'V'), (F, 2 * T), torch.float32)
                h.stft(x, self.window, self.N, self.hop, conjugate=True, want_V=True, out=(Xb, Vb))
                Xs.append(Xb)
                Vs.append(Vb)
        else:
            T = self.num_frames(samples.shape[2])
            X = h.buffer((key, 'batch', 'X'), (2 * B, F, T), torch.complex64)
            Vs = h.buffer((key, 'batch', 'V'), (B, F, 2 * T), torch.float32)
            for b in range(B):
                h.stft(samples[b], self.window, self.N, self.hop, conjugate=True, want_V=True, out=(X[2 * b:2 * b + 2], Vs[b]))
            Xs = [X[2 * b:2 * b + 2] for b in range(B)]
        self._mark('stft')
        means_host = getattr(self, '_means_host', None)
        if means_host is None or means_host.shape[0] != B:
            means_host = self._means_host = torch.empty((B, self.D), dtype=torch.float64, pin_memory=True)
        rs = []
        for b in range(B):
            Xb = Xs[b]
            coh, ang, mean = h.phat_angspec(Xb, self.E, out_key=(key, 'clip', b))
            means_host[b].copy_(mean, non_blocking=True)
            rs.append(dict(X=Xb, coherence=coh, angularSpectrogram=ang, meanAngularSpectrum=mean, _mean_host=means_host[b]))
        means_ready = torch.cuda.Event()
        means_ready.record()
        self._mark('angular')
        if ragged:
            W0, _ = self.nmf_init(max(V.shape[1] for V in Vs))
            W = h.buffer((key, 'batch', 'W'), (B,) + tuple(W0.shape), W0.dtype)
            W.copy_(W0.expand_as(W))
            H = []
            for b, V in enumerate(Vs):
                Hb = h.buffer((key, 'clip', b, 'H'), (self.K, V.shape[1]), torch.float32)
                Hb.copy_(self.nmf_init(V.shape[1])[1])
                H.append(Hb)
            h.klnmf_ragged(Vs, W, H, self.I, self.alpha, self.eps, update_W=True)
        else:
            W0, H0 = self.nmf_init(2 * T)
            W = h.buffer((key, 'batch', 'W'), (B,) + tuple(W0.shape), W0.dtype)
            H = h.buffer((key, 'batch', 'H'), (B,) + tuple(H0.shape), H0.dtype)
            W.copy_(W0.expand_as(W))
            H.copy_(H0.expand_as(H))
            h.klnmf_batched(Vs, W, H, self.I, self.alpha, self.eps, update_W=True)
        self._mark('nmf')
        for b, r in enumerate(rs):
            r.update(V=Vs[b], W=W[b], H=H[b], _mean_ready=means_ready)
        return rs

    def _back(self, r, masks, key=None):
        h = self.h
        key = self._token if key is None else key
        S = masks.shape[0]
        est = h.masked_recon_phase(masks, r['X'], r['W'], r['H'], out_key=key)
        self._mark('recon')
        F, T = est.shape[2:]
        y = h.istft_ola(est.reshape(S * 2, F, T), self.synthesisWindow, self.N, self.hop,
                        gain=np.float32(self.hop / float(self.N) * 2), center=True, conjugate=True, out_key=key)
        self._mark('istft')
        r['targetCoefficientMasks'] = masks
        r['targetSpectrogramEstimates'] = est
        r['targetSignalEstimates'] = y.reshape(S, 2, -1)
        return r

    def _pick_targets(self, r, numTargets):
        r['_mean_ready'].synchronize()
        mean = r['_mean_host'].numpy().copy()
        idx = fn.estimateTargetTDOAIndexesFromAngularSpectrum(mean, self.micSep, self.D, numTargets)
        r['targetTDOAIndexes'] = [int(i) for i in idx]
        return r['targetTDOAIndexes']

    # ------------------------------------------------------------------ flows
    def enhance(self, samples, collect_stage_times=False, localizationWindow=None):
        """samples (2, n) f32 cuda -> dict of device tensors (enhancement flow, one target; per frame with a localizationWindow)."""
        self.stage_events = [] if collect_stage_times else None
        return self._enhance_back(self._front(samples), self._token, localizationWindow)

    def _window_targets(self, r, numTargets, localizationWindow, key):
        """Each frame's targets from the window means of the clip's angular spectrogram, on the device."""
        targets, means, status = self.h.window_targets(r['angularSpectrogram'], localizationWindow, numTargets, out_key=key)
        self._mark('localize')
        r.update(frameTargetTDOAIndexes=targets, windowMeans=means, status=status)
        return targets

    def _tdoas_device(self):
        if getattr(self, '_tdoas_dev', None) is None:
            self._tdoas_dev = self.h.to_device(np.ascontiguousarray(self.hypothesisTDOAs, dtype=np.float64))
        return self._tdoas_dev

    def _enhance_back(self, r, key, localizationWindow=None):
        h = self.h
        if localizationWindow is not None:
            targets = self._window_targets(r, 1, localizationWindow, key)
        argmax, refined = h.tdoa_argmax(r['coherence'], self.E, r['W'], out_key=key)
        self._mark('gccnmf')
        if localizationWindow is None:
            target = self._pick_targets(r, 1)[0]
        r['refinedDecisions'] = int(refined.item())
        if r['refinedDecisions'] > h.lib.gccnmf_tdoa_argmax_refine_capacity(self.K, argmax.shape[1]):
            _, argmax = h.tdoa_gccnmf(r['coherence'], self.E, r['W'], want_values=False, want_argmax=True)   # exact float64 kernel
        window = (self.hypothesisTDOAs[-1] - self.hypothesisTDOAs[0]) * self.windowPercent
        if localizationWindow is None:
            lut = fn.getTargetTDOALookup(self.hypothesisTDOAs, target, window)
            mask = h.argmax_mask(argmax, h.to_device(lut.astype(np.uint8)), out_key=key)
        else:
            mask = h.argmax_mask_frames(argmax, self._tdoas_device(), targets.reshape(-1), window, out_key=key)
        self._mark('mask')
        r['argMaxGCCNMF'] = argmax
        return self._back(r, mask[None], key)

    def separate(self, samples, numTargets, collect_stage_times=False, localizationWindow=None):
        """samples (2, n) f32 cuda -> dict of device tensors (runGCCNMF.py flow, numTargets sources; source q is the q-th target
        from the left in each frame with a localizationWindow)."""
        self.stage_events = [] if collect_stage_times else None
        return self._separate_back(self._front(samples), numTargets, self._token, localizationWindow)

    def _separate_back(self, r, numTargets, key, localizationWindow=None):
        h = self.h
        if localizationWindow is None:
            idx = self._pick_targets(r, numTargets)
            E_sel = h.to_device(np.ascontiguousarray(self.E_host[:, idx]))
            values, _ = h.tdoa_gccnmf(r['coherence'], E_sel, r['W'], want_values=True, want_argmax=False)
        else:
            targets = self._window_targets(r, numTargets, localizationWindow, key)
            values = h.target_gccnmf(r['coherence'], self.E, r['W'], targets, out_key=key)
        self._mark('gccnmf')
        masks, flag = h.coeff_mask(values)
        self._mark('mask')
        r['targetTDOAGCCNMFs'] = values
        r['_all_nan_flag'] = flag
        return self._back(r, masks, key)

    # ------------------------------------------------------------------ batches of clips
    def enhance_batch(self, samples, collect_stage_times=False, localizationWindow=None):
        """samples (B, 2, n) f32 cuda, or a list of B (2, n_b) f32 cuda recordings of any lengths -> list of B dicts, clip b's
        bit-identical to enhance(samples[b], localizationWindow=localizationWindow).  The KL-NMF runs once for the whole batch;
        the other stages run per clip.  Valid until the next batch call."""
        self.stage_events = [] if collect_stage_times else None
        rs = self._front_batch(samples)
        if rs and localizationWindow is None:
            rs[0]['_mean_ready'].synchronize()          # one host wait for all B means before peak picking
        return [self._enhance_back(r, (self._token, 'clip', b), localizationWindow) for b, r in enumerate(rs)]

    def separate_batch(self, samples, numTargets, collect_stage_times=False, localizationWindow=None):
        """samples (B, 2, n) f32 cuda or a list of (2, n_b) recordings -> list of B dicts, clip b's bit-identical to
        separate(samples[b], numTargets, localizationWindow=localizationWindow)."""
        self.stage_events = [] if collect_stage_times else None
        rs = self._front_batch(samples)
        if rs and localizationWindow is None:
            rs[0]['_mean_ready'].synchronize()
        return [self._separate_back(r, numTargets, (self._token, 'clip', b), localizationWindow) for b, r in enumerate(rs)]

    # ------------------------------------------------------------------ the whole flow as ONE C-ABI call
    def run_fused(self, samples, numTargets=0, localizationWindow=None):
        """gccnmf_separate: every stage enqueued by one library call, target picking on the device, no host synchronisation
        until the caller reads a result.  numTargets = 0: enhancement flow (one target); >= 1: runGCCNMF.py separation.
        Returns dict(W, H, targetSignalEstimates (S, 2, n_out), targetTDOAIndexes (device i32), status (device i32)).
        With a localizationWindow, gccnmf_separate_tracked: targets per frame, and the dict has frameTargetTDOAIndexes (T, S) and
        windowMeans (D, T) in place of targetTDOAIndexes."""
        import ctypes
        from ._lib import PipelineConfig, _ptr
        h, torch = self.h, self.torch
        n = samples.shape[1]
        T = self.num_frames(n)
        S = max(1, numTargets)
        window = (self.hypothesisTDOAs[-1] - self.hypothesisTDOAs[0]) * self.windowPercent
        cfg = PipelineConfig(self.N, self.hop, self.D, self.K, self.I, int(numTargets), self.alpha, self.eps, float(window))
        key = (self._token, 'fused', int(numTargets))
        W0, H0 = self.nmf_init(2 * T)
        W, H = h.buffer((key, 'W'), W0.shape, W0.dtype), h.buffer((key, 'H'), H0.shape, H0.dtype)
        W.copy_(W0)
        H.copy_(H0)
        tdoas = self._tdoas_device()
        length = int(h.lib.gccnmf_istft_length(self.N, self.hop, T, 1))
        y = h.buffer((key, 'y'), (S, 2, length), torch.float32)
        status = h.buffer((key, 'status'), (1,), torch.int32)
        if localizationWindow is not None:
            w = int(localizationWindow)
            frame_targets = h.buffer((key, 'frame_targets'), (T, S), torch.int32)
            means = h.buffer((key, 'window_means'), (self.D, T), torch.float64)
            ws = h.workspace('pipeline', h.lib.gccnmf_pipeline_tracked_workspace_bytes(ctypes.byref(cfg), w, n))
            h.check(h.lib.gccnmf_separate_tracked(h.h, ctypes.byref(cfg), w, _ptr(samples), n, _ptr(self.window), _ptr(self.E), _ptr(tdoas), _ptr(W),
                                                  _ptr(H), _ptr(y), _ptr(frame_targets), _ptr(means), _ptr(status), _ptr(ws), ws.numel(), h.stream))
            return dict(W=W, H=H, targetSignalEstimates=y, frameTargetTDOAIndexes=frame_targets, windowMeans=means, status=status)
        targets = h.buffer((key, 'targets'), (S,), torch.int32)
        ws = h.workspace('pipeline', h.lib.gccnmf_pipeline_workspace_bytes(ctypes.byref(cfg), n))
        h.check(h.lib.gccnmf_separate(h.h, ctypes.byref(cfg), _ptr(samples), n, _ptr(self.window), _ptr(self.E), _ptr(tdoas), _ptr(W), _ptr(H),
                                      _ptr(y), _ptr(targets), _ptr(status), _ptr(ws), ws.numel(), h.stream))
        return dict(W=W, H=H, targetSignalEstimates=y, targetTDOAIndexes=targets, status=status)

    @staticmethod
    def raise_on_status(status, tracked=False):
        """The conditions the reference turns into exceptions (call after synchronising).  tracked: bit 0 of a tracked flow (a
        frame held earlier targets) is not one of them."""
        st = int(status.item())
        if st & 1 and not tracked:
            raise ValueError('did not find enough peaks in the angular spectrum')          # gccNMFFunctions.py:102-104
        if st & 2:
            raise ValueError('All-NaN slice encountered')                                  # numpy.nanargmax, :138
        if st & 4:
            raise RuntimeError('all-TDOA argmax: more near-tie decisions than the refinement list holds; use enhance(), which falls '
                               'back to the exact float64 kernel')

    def run_fused_host(self, samples_host, numTargets=0, out_host=None, check=True, localizationWindow=None):
        """Pinned (or pageable) host samples in -> host float32 (S, 2, n_out) signal estimates out, through ONE library call
        (gccnmf_separate, or gccnmf_separate_tracked with a localizationWindow): H2D copy, the whole flow enqueued without host
        synchronisation, D2H copy, one stream synchronise."""
        torch = self.torch
        s = samples_host if isinstance(samples_host, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(samples_host, dtype=np.float32))
        r = self.run_fused(s.to(self.h.device, non_blocking=True), numTargets, localizationWindow)
        y = r['targetSignalEstimates']
        if out_host is None:
            out_host = torch.empty(y.shape, dtype=torch.float32, pin_memory=True)
        if getattr(self, '_status_host', None) is None:
            self._status_host = torch.zeros(1, dtype=torch.int32, pin_memory=True)
        out_host.copy_(y, non_blocking=True)
        self._status_host.copy_(r['status'], non_blocking=True)
        torch.cuda.current_stream(self.h.device).synchronize()
        if check:
            self.raise_on_status(self._status_host, tracked=localizationWindow is not None)
        return out_host

    # ------------------------------------------------------------------ host-buffer entry (what e2e times)
    def enhance_host(self, samples_host, out_host=None):
        """Pinned (or pageable) host samples in -> host float32 (1, 2, n_out) signal estimates out."""
        torch = self.torch
        s = samples_host if isinstance(samples_host, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(samples_host, dtype=np.float32))
        r = self.enhance(s.to(self.h.device, non_blocking=True))
        y = r['targetSignalEstimates']
        if out_host is None:
            out_host = torch.empty(y.shape, dtype=torch.float32, pin_memory=True)
        out_host.copy_(y, non_blocking=True)
        torch.cuda.current_stream(self.h.device).synchronize()
        return out_host

    def separate_host(self, samples_host, numTargets, out_host=None):
        torch = self.torch
        s = samples_host if isinstance(samples_host, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(samples_host, dtype=np.float32))
        r = self.separate(s.to(self.h.device, non_blocking=True), numTargets)
        y = r['targetSignalEstimates']
        if out_host is None:
            out_host = torch.empty(y.shape, dtype=torch.float32, pin_memory=True)
        out_host.copy_(y, non_blocking=True)
        torch.cuda.current_stream(self.h.device).synchronize()
        if int(r['_all_nan_flag'].item()):
            raise ValueError('All-NaN slice encountered')
        return out_host
