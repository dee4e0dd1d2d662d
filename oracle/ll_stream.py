"""Host model of the streaming schedule of the low-latency engine (gcc-nmf_b200/csrc/lowlatency.cu): the input ring, the running
maximum carried across calls, the N-sample output ring and the emit.  It is fed per-frame quantities (the angular spectrum and the
synthesised frames of every whole frame) and reproduces, call by call, what the engine emits; the batch loop is the reference it
must match whatever the call sizes are.
"""
import numpy as np


def latency(weights, hop):
    """Q hop - hop - z: Q = ceil(N / hop) hops per frame, z the first nonzero weight."""
    nz = np.flatnonzero(np.asarray(weights) != 0)
    return -(-len(weights) // hop) * hop - hop - int(nz[0])


def frames_of(samples, n_frames, N, hop):
    """(channels, n) -> (n_frames, channels, N): the whole frames the batch loop cuts."""
    return np.stack([samples[:, j * hop:j * hop + N] for j in range(n_frames)])


class StreamModel(object):
    """One stream; the output ring accumulates in float32 after every add, as the notebook's float32 output array does (float64
    with accumulate=np.float64).  push(x (2, c hop), frame_fn) calls frame_fn(frames (c', 2, N)) for the c' whole frames this call completes,
    which returns (angular (D, c'), synthesised frames (c', 2, N)); returns the c hop output samples."""

    def __init__(self, N, hop, weights, gain, D, accumulate=np.float32):
        self.Q = -(-N // hop)
        self.N, self.hop, self.w, self.g = N, hop, np.asarray(weights, np.float64), gain
        self.z = int(np.flatnonzero(self.w != 0)[0])
        self.in_ring = np.zeros((2, (self.Q - 1) * hop), np.float32)
        self.out_ring = np.zeros((2, N), accumulate)
        self.carry = np.full(D, -np.inf)
        self.hops = 0
        self.accumulate = accumulate

    def push(self, x, frame_fn):
        N, hop = self.N, self.hop
        c = x.shape[1] // hop
        stage = np.concatenate([self.in_ring, x], axis=1)
        js = [self.hops + i + 1 - self.Q for i in range(c)]
        whole = [i for i in range(c) if js[i] >= 0]
        ang, frames, targets = None, None, []
        if whole:
            ang, frames = frame_fn(np.stack([stage[:, i * hop:i * hop + N] for i in whole]), [js[i] for i in whole])
        out = np.zeros((2, c * hop), np.float32)
        k = 0
        for i in range(c):
            base = (js[i] * hop) % N
            if js[i] >= 0:
                v = ang[:, k]
                self.carry = np.where((v > self.carry) | np.isnan(v), v, self.carry)
                targets.append(int(np.argmax(self.carry)))
                pos = (base + np.arange(self.z, N)) % N
                terms = self.w[self.z:] * frames[k][:, self.z:].astype(np.float64)
                if self.accumulate is np.float32:
                    self.out_ring[:, pos] = (self.out_ring[:, pos].astype(np.float64) + terms).astype(np.float32)
                else:
                    self.out_ring[:, pos] += terms
                k += 1
            pos = (base + self.z + np.arange(hop)) % N
            out[:, i * hop:(i + 1) * hop] = (self.out_ring[:, pos] * self.g).astype(np.float32)
            self.out_ring[:, pos] = 0
        self.in_ring = stage[:, c * hop:]
        self.hops += c
        self.targets = targets
        return out


def stream(samples, N, hop, weights, gain, D, frame_fn, schedule, accumulate=np.float32):
    """Runs a whole signal (2, n), n a multiple of hop, with calls of schedule[i % len] hops; returns (output (2, n), targets)."""
    m = StreamModel(N, hop, weights, gain, D, accumulate)
    outs, targets = [], []
    p, i = 0, 0
    while p < samples.shape[1]:
        c = min(schedule[i % len(schedule)], (samples.shape[1] - p) // hop)
        outs.append(m.push(samples[:, p:p + c * hop], frame_fn))
        targets += m.targets
        p += c * hop
        i += 1
    return np.concatenate(outs, axis=1), targets
