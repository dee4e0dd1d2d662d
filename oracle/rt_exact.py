"""Host model of one block of the real-time path (csrc/rt.cu), stage by stage, in the reduction orders DESIGN §4.5 fixes.

Every function takes the device's exported output of the previous stage (teacher forcing), so an error in one stage does not
spread into the next.  Where the kernel's order is fixed (coherence, realGCC, the gccPHAT nanmean, the inference chains, the
atoms contraction, the localisation) the model reproduces it bit for bit; the analysis FFT, the float64 filter sums and the
float32 inverse FFT are modelled in float64 and compared with a bound.

The one piece numpy lacks is a float32 fused multiply-add.  `fma32` gets it by round-to-odd: a * b of two float32 is exact in
float64, the float64 sum s = a * b + c is corrected to the odd neighbour when it was inexact (TwoSum error e != 0), and since
53 >= 24 + 2 the float32 rounding of that odd value is the correctly rounded fma.  No GPU is needed here.
"""
import numpy as np

WARP = 32
F32, F64 = np.float32, np.float64


# ------------------------------------------------------------------------------------------------ exact float32 arithmetic
def fma32(a, b, c):
    """Correctly rounded float32 a * b + c, elementwise (C fmaf / CUDA fmaf)."""
    p = np.asarray(a, F32).astype(F64) * np.asarray(b, F32).astype(F64)          # exact: 24 + 24 bits
    c = np.asarray(c, F32).astype(F64)
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)                                                  # TwoSum: s + e == p + c exactly
    bits = s.view(np.int64)
    fix = (e != 0) & ((bits & 1) == 0) & np.isfinite(s)
    step = np.where((e > 0) == (s > 0), 1, -1)                                     # one ulp toward e (bit patterns are sign-magnitude)
    return np.where(fix, bits + step, bits).view(F64).astype(F32)


def fma32_naive(a, b, c):
    """float32(float64(a) * b + c): double rounding, wrong where the float64 sum lands on a float32 midpoint."""
    return (np.asarray(a, F32).astype(F64) * np.asarray(b, F32).astype(F64) + np.asarray(c, F32).astype(F64)).astype(F32)


def butterfly(lanes):
    """Value every lane holds after `for (o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(~0u, s, o)`; axis 0 is the lane."""
    s = np.array(lanes)
    idx = np.arange(WARP)
    for o in (16, 8, 4, 2, 1):
        s = s + s[idx ^ o]
    return s[0]


def lane_fma_chains(a, b, n):
    """Per lane l: acc = fmaf(a[i], b[i], acc) over i = l, l + 32, ... < n from 0.f; a, b have the contracted index first.
    Returns (32, ...) lane partials.  Zero padding appends fmaf(0, 0, acc) = acc."""
    steps = -(-n // WARP)
    pad = steps * WARP - n
    a = np.concatenate([np.asarray(a, F32), np.zeros((pad,) + a.shape[1:], F32)])
    b = np.concatenate([np.asarray(b, F32), np.zeros((pad,) + b.shape[1:], F32)])
    acc = np.zeros((WARP,) + np.broadcast_shapes(a.shape[1:], b.shape[1:]), F32)
    for i in range(steps):
        acc = fma32(a[i * WARP:(i + 1) * WARP], b[i * WARP:(i + 1) * WARP], acc)
    return acc


# ------------------------------------------------------------------------------------------------ A: analysis
def analysis(frames, win_a):
    """frames (2, N, nT) raw float32 samples -> X (2, F, nT) complex64: float64 rfft of the float32 product frame . window."""
    x = (np.asarray(frames, F32) * np.asarray(win_a, F32)[None, :, None]).astype(F64)
    return np.fft.rfft(x, axis=1).astype(np.complex64)


def coherence(X):
    """rt_coherence of X[0], X[1] (F, nT) in kernel order -> (re, im) float32."""
    a, b = X[0], X[1]
    ax, ay, bx, by = (np.real(a).astype(F32), np.imag(a).astype(F32), np.real(b).astype(F32), np.imag(b).astype(F32))
    with np.errstate(all='ignore'):
        re = ax * bx + ay * by
        im = ay * bx - ax * by
        ma = np.sqrt(ax.astype(F64) ** 2 + ay.astype(F64) ** 2).astype(F32)
        mb = np.sqrt(bx.astype(F64) ** 2 + by.astype(F64) ** 2).astype(F32)
        ia, ib = F32(1) / ma, F32(1) / mb
        re, im = re * ia, im * ia
        re, im = re * ib, im * ib
    return re, im


def real_gcc(X, E):
    """G (nT, D, F) float32 = fsub(fmul(c.x, e.x), fmul(c.y, e.y)) with E (F, D) complex64."""
    re, im = coherence(X)                                              # (F, nT)
    ex, ey = np.real(E).astype(F32), np.imag(E).astype(F32)           # (F, D)
    with np.errstate(all='ignore'):
        G = re.T[:, None, :] * ex.T[None] - im.T[:, None, :] * ey.T[None]
    return G.astype(F32)


def gccphat(G):
    """(D, nT) float32: per lane a float64 sum (and count) of the non-NaN G over f = lane (mod 32), the xor butterfly on both,
    then float(sum / count), NaN for count 0."""
    nT, D, F = G.shape
    steps = -(-F // WARP)
    g = np.full((nT, D, steps * WARP), np.nan, F32)
    g[:, :, :F] = G
    g = g.reshape(nT, D, steps, WARP)
    ok = g == g
    s = np.zeros((WARP, nT, D), F64)
    for i in range(steps):                                             # sequential per lane, in f order
        s = s + np.where(ok[:, :, i, :], g[:, :, i, :].astype(F64), 0.0).transpose(2, 0, 1)
    n = ok.sum(axis=2).transpose(2, 0, 1)
    s, n = butterfly(s), butterfly(n)
    with np.errstate(all='ignore'):
        out = np.where(n > 0, (s / np.maximum(n, 1)).astype(F32), F32(np.nan))
    return out.T.astype(F32)


# ------------------------------------------------------------------------------------------------ I: coefficient inference
def seeded_H0(K, epsilon, seed=0):
    """The (K, 2) initial coefficients RealtimeEngine / MultiStreamRealtimeEngine upload."""
    np.random.seed(seed)
    return (np.random.random((K, 2)).astype(F32) + epsilon).astype(F32)


def magnitudes(X):
    """|X| (F, 2 nT) float32, column 2 t + channel: float(sqrt(double re^2 + double im^2))."""
    r, i = np.real(X).astype(F64), np.imag(X).astype(F64)
    m = np.sqrt(r * r + i * i).astype(F32)                             # (2, F, nT)
    return np.ascontiguousarray(m.transpose(1, 2, 0).reshape(m.shape[1], -1))


def column_sums(W):
    """colsum(W) (K,) float32, a sequential float32 sum over f."""
    s = np.zeros(W.shape[1], F32)
    for f in range(W.shape[0]):
        s = s + W[f]
    return s


def infer(X, W, H0, iterations, alpha, epsilon):
    """H (K, 2 nT) float32 after `iterations` of rt_inf_ratio / rt_inf_update, every column starting from H0[:, channel]."""
    W = np.asarray(W, F32)
    F, K = W.shape
    V = magnitudes(X)
    J = V.shape[1]
    H = np.tile(np.asarray(H0, F32), (1, J // 2))
    denom = (column_sums(W) + F32(alpha)) + F32(epsilon)
    with np.errstate(all='ignore'):
        for _ in range(iterations):
            wh = butterfly(lane_fma_chains(W.T[:, :, None], H[:, None, :], K))          # (F, J) over k
            R = (V / wh).astype(F32)
            num = butterfly(lane_fma_chains(W[:, :, None], R[:, None, :], F))          # (K, J) over f
            H = (H * (num / denom[:, None])).astype(F32)
    return H


# ------------------------------------------------------------------------------------------------ B: atoms
def atoms(G, W):
    """C (nT, D, K) float32: one fmaf chain per output over f = 0 .. F-1 from 0.f."""
    nT, D, F = G.shape
    W = np.asarray(W, F32)
    acc = np.zeros((nT, D, W.shape[1]), F32)
    for f in range(F):
        acc = fma32(G[:, :, f, None], W[f][None, None, :], acc)
    return acc


def argmax_over_tdoa(C):
    """(K, nT) int32 argmax over d in numpy's order (a NaN wins, then the larger value, then the lower index)."""
    return np.argmax(C, axis=1).T.astype(np.int32)


def atom_mask(argmax, target, epsilon, beta, noise_floor, mode):
    """(K, nT) float64, rt_atoms_kernel's mask of a given argmax: int - float32 target promotes to float64."""
    dist = np.abs(np.asarray(argmax, F64) - F64(F32(target)))
    eps, beta, nf = F64(F32(epsilon)), F64(F32(beta)), F32(noise_floor)
    if mode == 0:
        return np.where(dist < eps, 1.0, 0.0)
    return np.exp(-np.power(dist / eps, beta)) / F64(F32(1) + nf) + F64(nf)


def atom_mask_ulp_bound(argmax, target, epsilon, beta):
    """float64 ulps a window-mode mask may differ by: 4 for exp, the division and the addition, plus CUDA pow's 2 ulps on
    x = (dist / eps)^beta amplified by the condition number x of exp(-x)."""
    x = np.power(np.abs(np.asarray(argmax, F64) - F64(F32(target))) / F64(F32(epsilon)), F64(F32(beta)))
    return 4.0 + 2.0 * x


# ------------------------------------------------------------------------------------------------ C, D: filter and synthesis
def row_sums(W):
    """recV (F,) float32 = float(sequential float64 sum over k)."""
    return np.cumsum(np.asarray(W, F64), axis=1)[:, -1].astype(F32)


def filter_spectrum(X, W, hmask, H=None, separation=True):
    """Y (2, F, nT) complex128 in float64 (not rounded): tfMask X with tfMask = (W . mask) / recV, or per channel
    (W . (H mask)) / (W . H) with inference.  Separation off: X."""
    X = np.asarray(X, np.complex64).astype(np.complex128)
    if not separation:
        return X
    W = np.asarray(W, F32).astype(F64)
    with np.errstate(all='ignore'):
        if H is None:
            tf = (W @ hmask) / row_sums(W).astype(F64)[:, None]                        # (F, nT)
            return X * tf[None]
        H = np.asarray(H, F32).astype(F64)
        Y = np.empty_like(X)
        for c in range(2):
            h = H[:, c::2]                                                             # (K, nT)
            Y[c] = X[c] * ((W @ (h * hmask)) / (W @ h))
    return Y


def synthesis(Y, win_s):
    """(2, N, nT) float64: irfft(Y) . synthesis window (irfft ignores the imaginary parts of bins 0 and N/2)."""
    N = len(win_s)
    return np.fft.irfft(np.asarray(Y).astype(np.complex128), n=N, axis=1) * np.asarray(win_s, F32).astype(F64)[None, :, None]


# ------------------------------------------------------------------------------------------------ localisation
def localize(hist, index, gcc, window, enabled, target):
    """rt_localize: push the (D, nT) gccPHAT columns into the (D, history_length) float64 ring at `index`, then the nanmean
    over the newest min(max(window, 1), length) columns, newest first, and its argmax.  Returns (hist, index, target)."""
    hist = np.array(hist, F64)
    D, L = hist.shape
    nT = gcc.shape[1]
    for t in range(nT):
        hist[:, (index + t) % L] = np.asarray(gcc[:, t], F32).astype(F64)
    index = (index + nT) % L
    w = min(max(int(window), 1), L)
    s = np.zeros(D, F64)
    n = np.zeros(D, np.int64)
    for j in range(w):
        v = hist[:, (index - 1 - j) % L]
        ok = v == v
        s = s + np.where(ok, v, 0.0)
        n = n + ok
    with np.errstate(all='ignore'):
        mean = np.where(n > 0, s / np.maximum(n, 1), np.nan)
    if enabled:
        target = F32(np.argmax(mean))
    return hist, index, F32(target)


# ------------------------------------------------------------------------------------------------ comparisons
def ulps32(device, model):
    """|device - model| in float32 ulps of the model value (complex: per part); NaN where both are NaN counts 0."""
    device, model = np.asarray(device), np.asarray(model)
    if np.iscomplexobj(model):
        return np.maximum(ulps32(np.real(device), np.real(model)), ulps32(np.imag(device), np.imag(model)))
    d, m = device.astype(F64), model.astype(F64)
    unit = np.spacing(np.abs(m).astype(F32)).astype(F64)
    with np.errstate(all='ignore'):
        u = np.abs(d - m) / unit
    both_nan = np.isnan(d) & np.isnan(m)
    return np.where(both_nan, 0.0, np.where(np.isnan(d) | np.isnan(m), np.inf, u))


def ulps64(device, model):
    d, m = np.asarray(device, F64), np.asarray(model, F64)
    with np.errstate(all='ignore'):
        u = np.abs(d - m) / np.spacing(np.abs(m))
    return np.where(np.isnan(d) & np.isnan(m), 0.0, np.where(np.isnan(d) | np.isnan(m), np.inf, u))
