"""Host model of the source stages of the real-time path with P target TDOAs per stream (csrc/rt.cu, gccnmf_rtsep_*), in the
kernel's orders, next to the single-target model in rt_exact.py.

source_masks      the winner per atom and frame among the target rows of the atoms contraction, numpy.argmax's order (a NaN
                  first, then the larger value, then the lower source), as P one-hot float64 masks
localize_sources  rt_localize with P sources: the history push and windowed nanmean of rt_exact.localize, then the P largest
                  strict local maxima (estimateTargetTDOAIndexesFromAngularSpectrum, the host function the device picker is
                  tested against) as the next targets, or the previous targets and status bit 0 when there are fewer peaks
"""
import numpy as np

from . import rt_exact as rx

F64 = np.float64
STATUS_FEW_PEAKS = 1


def source_masks(C, targets):
    """C (nT, D, K) float32 from rx.atoms, targets (P,) -> (masks (P, K, nT) float64 0 / 1, values (P, K, nT) float32)."""
    targets = [int(t) for t in targets]
    values = np.ascontiguousarray(np.asarray(C, np.float32)[:, targets, :].transpose(1, 2, 0))     # (P, K, nT)
    winner = np.argmax(values, axis=0)
    masks = (winner[None] == np.arange(len(targets))[:, None, None]).astype(F64)
    return masks, values


def window_mean(hist, index, window):
    """The nanmean rt_localize takes: the newest min(max(window, 1), length) columns before `index`, newest first."""
    D, L = hist.shape
    w = min(max(int(window), 1), L)
    s = np.zeros(D, F64)
    n = np.zeros(D, np.int64)
    for j in range(w):
        v = hist[:, (index - 1 - j) % L]
        ok = v == v
        s = s + np.where(ok, v, 0.0)
        n = n + ok
    with np.errstate(all='ignore'):
        return np.where(n > 0, s / np.maximum(n, 1), np.nan)


def localize_sources(hist, index, gcc, window, enabled, targets, P):
    """Returns (hist, index, targets (P,) int32, status bit) after one block's localisation."""
    from gcc_nmf_b200.gccNMFFunctions import estimateTargetTDOAIndexesFromAngularSpectrum
    hist, index, _ = rx.localize(hist, index, gcc, window, False, 0.0)
    targets = np.asarray(targets, np.int32).copy()
    status = 0
    if enabled:
        mean = window_mean(hist, index, window)
        try:
            targets = np.asarray(estimateTargetTDOAIndexesFromAngularSpectrum(mean, 0.1, len(mean), P), np.int32)
        except ValueError:
            status = STATUS_FEW_PEAKS
    return hist, index, targets, status
