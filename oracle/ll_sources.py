"""Host model of the target decisions of the low-latency engine with P sources per stream (csrc/lowlatency.cu,
ll_src_targets_kernel, gccnmf_llsep_*), stateful across calls, next to the schedule model in ll_stream.py.

Per whole frame of a stream: the running maximum of the angular spectrum is updated from the carried one (NaN propagates and
sticks), then the P largest strict local maxima of that running maximum, ascending, become the stream's targets; with fewer than
P peaks the targets stay and status bit 0 is set (sticky until reset).  The frame's column targets are the targets, or a source's
override where it is >= 0.  After init / reset the targets are floor((2 q + 1) D / (2 P)).

The peak rule is written out as select_peaks (csrc/common.cuh) counts it; with distinct peak values it is the reference's
estimateTargetTDOAIndexesFromAngularSpectrum(numSources=P) (pinned in tests/test_ll_sources_cpu.py).
"""
import numpy as np

STATUS_FEW_PEAKS = 1
STATUS_ALL_NAN = 2


def default_targets(D, P):
    return np.array([(2 * q + 1) * D // (2 * P) for q in range(P)], np.int32)


def pick_peaks(x, P):
    """The P largest strict interior maxima of x in ascending index order, or None when there are fewer than P.  Of two equal
    peak values the higher index ranks higher (argsort(kind='stable'))."""
    x = np.asarray(x, np.float64)
    D = len(x)
    with np.errstate(invalid='ignore'):
        peaks = [d for d in range(1, D - 1) if x[d] > x[d - 1] and x[d] > x[d + 1]]
    if len(peaks) < P:
        return None
    chosen = [d for d in peaks if sum(1 for e in peaks if x[e] > x[d] or (x[e] == x[d] and e > d)) < P]
    return np.array(sorted(chosen), np.int32)


class SourceTargets(object):
    """One stream's decisions.  frame(angular column (D,)) -> (running maximum (D,), column targets (P,))."""

    def __init__(self, D, P):
        self.D, self.P = D, P
        self.override = np.full(P, -1, np.int32)
        self.reset()

    def reset(self):
        """Back to an empty stream; the overrides stay."""
        self.carry = np.full(self.D, -np.inf)
        self.targets = default_targets(self.D, self.P)
        self.status = 0

    def set_override(self, targets):
        self.override = np.asarray(targets, np.int32).copy()

    def frame(self, ang):
        v = np.asarray(ang, np.float64)
        with np.errstate(invalid='ignore'):
            self.carry = np.where((v > self.carry) | np.isnan(v), v, self.carry)
        picked = pick_peaks(self.carry, self.P)
        if picked is None:
            self.status |= STATUS_FEW_PEAKS
        else:
            self.targets = picked
        return self.carry.copy(), self.column_targets()

    def column_targets(self):
        return np.where(self.override >= 0, self.override, self.targets).astype(np.int32)
