"""Host model of the low-latency engine's coefficient inference (ll_infer_kernel / ll_dict_infer_kernel, csrc/lowlatency.cu), and
the column groups of a bank engine's call.  Test infrastructure only.

The engine keeps H (K, 2T) with channel c of frame t in column c T + t, every column starting from H0[:, c].  Both contractions
of an iteration are a lane-strided float32 fmaf chain from 0.f followed by the xor butterfly, and the update is
H * (num / ((colsum + alpha) + eps)); the column sums are ll_dict_kernel's sequential float32 sums over f.  Every piece comes
from oracle/rt_exact.py and oracle/offline_exact.py, so the model adds no arithmetic of its own and is bit-exact.
"""
import numpy as np

from oracle.offline_exact import magnitudes
from oracle.rt_exact import butterfly, column_sums, lane_fma_chains

F32 = np.float32


def infer(X, W, H0, iterations, alpha, epsilon):
    """H (K, 2T) float32 after `iterations` H-only KL updates of every column of X (2, F, T), column c T + t from H0[:, c]."""
    W = np.asarray(W, F32)
    F, K = W.shape
    V = magnitudes(X, 2)                                                           # (F, 2T), column c T + t
    T = V.shape[1] // 2
    H = np.repeat(np.asarray(H0, F32), T, axis=1)                                  # (K, 2T)
    denom = (column_sums(W) + F32(alpha)) + F32(epsilon)
    with np.errstate(all='ignore'):
        for _ in range(iterations):
            wh = butterfly(lane_fma_chains(W.T[:, :, None], H[:, None, :], K))     # (F, 2T) over k
            R = (V / wh).astype(F32)
            num = butterfly(lane_fma_chains(W[:, :, None], R[:, None, :], F))     # (K, 2T) over f
            H = (H * (num / denom[:, None])).astype(F32)
    return H


def column_groups(hops, steering=None, dictionary=None):
    """{(dictionary entry, table entry): columns} of a call of `hops` hops per stream, from the exported per-stream assignments
    (None: every stream on entry 0).  Column t is frame t % hops of stream t // hops; only groups with columns are listed."""
    n = len(steering if steering is not None else dictionary)
    s = np.zeros(n, np.int64) if steering is None else np.asarray(steering, np.int64)
    d = np.zeros(n, np.int64) if dictionary is None else np.asarray(dictionary, np.int64)
    col_stream = np.arange(n * hops) // hops
    out = {}
    for key in sorted(set(zip(d.tolist(), s.tolist()))):
        out[key] = np.flatnonzero((d[col_stream] == key[0]) & (s[col_stream] == key[1]))
    return out


def split_h(H, cols, K):
    """Rows < K of columns `cols` of both channels of an engine's H (Kmax, 2T), as the model lays them out: (K, 2 len(cols))."""
    T = H.shape[1] // 2
    return np.concatenate([H[:K, cols], H[:K, T + np.asarray(cols)]], axis=1)
