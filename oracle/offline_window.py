"""Host model of the offline window targets (csrc/tracking.cu, gccnmf_window_targets) and of the per-frame enhancement mask
(gccnmf_argmax_mask_frames), built from the engines' models.

  window_means   frame t: rt_sources.window_mean over the clip's columns 0 .. t, so the window is cut at the start of the clip
                 (newest first, float64, NaN skipped, NaN when every term is NaN)
  frame_targets  frame t: ll_sources.pick_peaks(means[:, t], P), or, with fewer than P peaks, the targets of the latest earlier
                 frame that had P (ll_sources.default_targets before any such frame) and status bit 0
  mask_frames    frame t: offline_exact.argmax_mask with offline_exact.tdoa_lut of the frame's target
"""
import numpy as np

from .ll_sources import STATUS_FEW_PEAKS, default_targets, pick_peaks
from .offline_exact import argmax_mask, tdoa_lut
from .rt_sources import window_mean


def window_means(angular, window):
    """angular (D, T) float64 -> means (D, T) float64."""
    A = np.asarray(angular, np.float64)
    return np.stack([window_mean(A[:, :t + 1], t + 1, window) for t in range(A.shape[1])], axis=1).reshape(A.shape)


def frame_targets(means, P):
    """means (D, T) -> (targets (T, P) int32, status)."""
    D, T = means.shape
    last = default_targets(D, P)
    targets = np.empty((T, P), np.int32)
    status = 0
    for t in range(T):
        picked = pick_peaks(means[:, t], P)
        if picked is None:
            status |= STATUS_FEW_PEAKS
        else:
            last = picked
        targets[t] = last
    return targets, status


def window_targets(angular, window, P):
    """angular (D, T) float64 -> (means (D, T), targets (T, P) int32, status)."""
    means = window_means(angular, window)
    targets, status = frame_targets(means, P)
    return means, targets, status


def mask_frames(argmax, tdoas, targets, window):
    """argmax (K, T), tdoas (D,), targets (T,) -> mask (K, T) float32."""
    argmax = np.asarray(argmax)
    return np.stack([argmax_mask(argmax[:, t], tdoa_lut(tdoas, targets[t], window)) for t in range(argmax.shape[1])], axis=1)
