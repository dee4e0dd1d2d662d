"""Host model of the target decisions of the low-latency engine with a localisation window (csrc/lowlatency.cu,
ll_hist_targets_kernel / ll_hist_src_targets_kernel, gccnmf_llhist_*), stateful across calls, next to ll_sources.py.

Per frame of a stream, valid or not (a frame is valid when it starts at or after the stream's first sample and the stream is
active):
  - a valid frame updates the running maximum (NaN propagates and sticks) and writes its angular column into the (D, Lh) float64
    ring at the write index, which then moves on mod Lh;
  - with window w >= 1 the frame's mean is the newest-first float64 nanmean of the newest w ring columns (rt_sources.window_mean,
    the loop of rt_exact.localize without its float32 input), NaN where all are NaN; with w = 0 it is NaN;
  - P = 0: the target is numpy.argmax of the mean (w >= 1) or of the running maximum (w = 0), or the override when it is >= 0;
  - P >= 2: on a valid frame, the P largest strict local maxima of that same vector (ll_sources.pick_peaks) become the targets, or
    the targets stay and status bit 0 is set; the column targets are the targets or the source overrides.
init / reset zero the ring and set the index and the window to 0; reset keeps the overrides.
"""
import numpy as np

from .ll_sources import STATUS_FEW_PEAKS, default_targets, pick_peaks
from .rt_sources import window_mean


class WindowTargets(object):
    """One stream's decisions.  frame(angular column (D,), valid) -> (mean (D,), targets: () int for P = 0, (P,) with sources)."""

    def __init__(self, D, Lh, P=0):
        self.D, self.Lh, self.P = D, Lh, P
        self.override = -1 if P == 0 else np.full(P, -1, np.int32)
        self.reset()

    def reset(self):
        self.carry = np.full(self.D, -np.inf)
        self.ring = np.zeros((self.D, self.Lh))
        self.index = 0
        self.window = 0
        self.targets = default_targets(self.D, self.P) if self.P else None
        self.status = 0

    def frame(self, ang, valid=True):
        if valid:
            v = np.asarray(ang, np.float64)
            with np.errstate(invalid='ignore'):
                self.carry = np.where((v > self.carry) | np.isnan(v), v, self.carry)
            self.ring[:, self.index] = v
            self.index = (self.index + 1) % self.Lh
        mean = window_mean(self.ring, self.index, self.window) if self.window else np.full(self.D, np.nan)
        x = mean if self.window else self.carry
        if not self.P:
            return mean, np.int32(self.override if self.override >= 0 else np.argmax(x))
        if valid:
            picked = pick_peaks(x, self.P)
            if picked is None:
                self.status |= STATUS_FEW_PEAKS
            else:
                self.targets = picked
        return mean, np.where(self.override >= 0, self.override, self.targets).astype(np.int32)
