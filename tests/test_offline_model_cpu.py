"""CPU: the host model of the offline stage kernels (oracle/offline_exact.py) checked on its own, against float64 sums, exact
rational arithmetic, numpy's own expressions and the float32 oracle."""
from fractions import Fraction

import numpy as np
import pytest

from oracle import gccnmf_oracle as orc
from oracle import offline_exact as ox
from oracle import rt_exact as rx

F32, F64 = np.float32, np.float64
COHERENCE_BAR = 16 * 2.0 ** -24


def test_fma64_is_correctly_rounded():
    rng = np.random.default_rng(1)
    a = rng.standard_normal(3000)
    b = rng.standard_normal(3000).astype(F32).astype(F64)
    c = rng.standard_normal(3000) * 10.0 ** rng.integers(-20, 4, 3000)
    c[:1000] = -(a[:1000] * b[:1000])                          # heavy cancellation: the product's low part is the answer
    got = ox.fma64(a, b, c)
    for x, y, z, g in zip(a, b, c, got):
        assert g == float(Fraction(x) * Fraction(y) + Fraction(z)), (x, y, z)
    assert np.any(got != a * b + c)                             # the plain expression is not what the device computes


@pytest.mark.parametrize('K', [1, 7, 16, 129, 300])
def test_fma_chain_against_float64(K):
    rng = np.random.default_rng(K)
    A = rng.random((K, 6, 1)).astype(F32)
    B = (rng.random((K, 1, 5)) * (rng.random((K, 1, 5)) < 0.7)).astype(F32)
    got = ox.fma_chain(A, B, K).astype(F64)
    ref = np.einsum('kab,kab->ab', *np.broadcast_arrays(A.astype(F64), B.astype(F64)))
    mag = np.einsum('kab,kab->ab', *np.broadcast_arrays(np.abs(A).astype(F64), np.abs(B).astype(F64)))
    assert np.all(np.abs(got - ref) <= K * 2.0 ** -24 * mag)
    # the chain is sequential: the first steps agree with a float32 loop written out by hand
    acc = np.zeros((6, 5), F32)
    for k in range(K):
        acc = rx.fma32(A[k], B[k], acc)
    assert np.array_equal(acc, ox.fma_chain(A, B, K))


@pytest.mark.parametrize('K', [1, 5, 127, 128, 129, 1024, 1031])
def test_rowsum_model_against_float64(K):
    rng = np.random.default_rng(K)
    W = (rng.random((9, K)) ** 3).astype(F32)
    got = ox.rowsum(W).astype(F64)
    ref = W.astype(F64).sum(axis=1)
    steps = -(-K // ox.ROWSUM_THREADS)
    assert np.all(np.abs(got - ref) <= (steps + 10) * 2.0 ** -24 * np.abs(W).astype(F64).sum(axis=1))
    if K <= 128:    # at most one element per thread: the warp sums are the butterflies of the plain values
        lanes = np.zeros((128, 9), F32)
        lanes[:K] = W.T
        warps = np.zeros((32, 9), F32)
        warps[:4] = [rx.butterfly(lanes[w * 32:(w + 1) * 32]) for w in range(4)]
        assert np.array_equal(got.astype(F32), rx.butterfly(warps))


def test_coherence_model_against_numpy():
    rng = np.random.default_rng(7)
    n = 1 << 18
    X = (rng.standard_normal((2, 1, n)) + 1j * rng.standard_normal((2, 1, n))).astype(np.complex64)
    X *= (10.0 ** rng.integers(-6, 7, (2, 1, n))).astype(F32)
    X[0, 0, :16] = 0                                             # 0/0 -> NaN in both
    X[1, 0, 16:32] = 0
    model, ref = ox.coherence(X), ox.numpy_coherence(X)
    assert np.array_equal(np.isnan(model), np.isnan(ref))
    ok = ~np.isnan(ref)
    d = np.maximum(np.abs(model.real - ref.real), np.abs(model.imag - ref.imag))[ok]
    equal = float(np.mean((model.view(F32) == ref.view(F32))[np.repeat(ok, 2, axis=-1)]))
    print('coherence model vs numpy: max |d| = %d * 2^-24, %.1f %% of parts bit-equal' % (round(d.max() * 2 ** 24), 100 * equal))
    assert d.max() <= COHERENCE_BAR
    # and the model is the rt path's coherence (one formula for both)
    re, im = rx.coherence(X[:, 0])
    assert np.array_equal(model[0].real, re, equal_nan=True) and np.array_equal(model[0].imag, im, equal_nan=True)


def _nanargmax_cases():
    nan, inf = np.nan, np.inf
    cols = [[nan, -inf], [nan, -inf, -inf], [-inf, nan], [nan, 1.0], [1.0, nan], [nan, nan, 2.0], [2.0, 2.0], [0.0, -0.0],
            [-0.0, 0.0], [-inf, -inf], [inf, inf, nan], [1.0, nan, 1.0], [-1.0, nan, -inf, -1.0], [nan, nan], [nan]]
    S = max(len(c) for c in cols)
    G = np.full((S, len(cols)), nan, F32)
    for j, c in enumerate(cols):
        G[:len(c), j] = c
        if len(c) < S and not all(np.isnan(c)):
            G[len(c):, j] = -inf
    return G


def test_nanargmax_model_against_numpy():
    G = _nanargmax_cases()
    rng = np.random.default_rng(3)
    R = rng.integers(-2, 3, (5, 4000)).astype(F32)
    R[rng.random(R.shape) < 0.15] = np.nan
    R[rng.random(R.shape) < 0.1] = -np.inf
    for A in (G, R):
        masks, flag = ox.coeff_mask(A[:, :, None])
        all_nan = np.isnan(A).all(axis=0)
        assert flag == int(all_nan.any())
        assert not masks[:, all_nan].any()
        want = np.nanargmax(A[:, ~all_nan], axis=0)
        assert np.array_equal(np.argmax(masks[:, ~all_nan, 0], axis=0), want)
        assert np.array_equal(masks[:, ~all_nan, 0].sum(axis=0), np.ones(int((~all_nan).sum()), F32))
    assert ox.coeff_mask(np.array([[[np.nan]], [[-np.inf]]], F32))[0][:, 0, 0].tolist() == [1.0, 0.0]


@pytest.mark.parametrize('n_fft,hop', [(32, 8), (64, 48), (256, 64), (128, 128)])
def test_ola_model_against_oracle_istft(n_fft, hop):
    """Fed the oracle's own float32 frames, the unfused model is the oracle's istft bit for bit; the fused one (the device's
    DFMA) stays within one float32 ulp per add."""
    from scipy import fftpack
    rng = np.random.default_rng(n_fft + hop)
    F, T = n_fft // 2 + 1, 9
    spec = (rng.standard_normal((F, T)) + 1j * rng.standard_normal((F, T))).astype(np.complex64)
    frames = np.stack([fftpack.ifft(np.concatenate((spec[:, i].conj(), spec[-2:0:-1, i]))).real for i in range(T)])
    assert frames.dtype == F32
    w = np.hanning(n_fft)
    y = ox.ola(frames[None], w, hop, True, 1.0, fused=False)[0]
    assert np.array_equal(y, orc.istft(spec, hop, n_fft, np.hanning, center=True))
    yf = ox.ola(frames[None], w, hop, True, 1.0)[0]
    assert float(rx.ulps32(yf, y).max()) <= -(-n_fft // hop)


def test_ifft_model_matches_oracle_frames():
    from scipy import fftpack
    rng = np.random.default_rng(5)
    n, T = 64, 4
    spec = (rng.standard_normal((1, n // 2 + 1, T)) + 1j * rng.standard_normal((1, n // 2 + 1, T))).astype(np.complex64)
    model = ox.ifft_frames(spec, n, conjugate=True)[0]
    for i in range(T):
        col = spec[0, :, i].copy()
        col[0] = col[0].real                                    # the oracle's rebuild drops these imaginary parts too
        col[-1] = col[-1].real
        ref = fftpack.ifft(np.concatenate((col.conj(), col[-2:0:-1])).astype(np.complex128)).real
        assert np.abs(model[i] - ref).max() <= 1e-14 * np.abs(ref).max()


def _kernel_rule(x, S):
    """select_peaks written out as the kernel counts: a peak is kept when fewer than S peaks are larger, or equal and later."""
    D = len(x)
    peak = [0 < d < D - 1 and x[d] > x[d - 1] and x[d] > x[d + 1] for d in range(D)]
    kept = [d for d in range(D) if peak[d] and sum(1 for e in range(D) if peak[e] and (x[e] > x[d] or (x[e] == x[d] and e > d))) < S]
    return kept, sum(peak)


def test_stable_peak_rule():
    rng = np.random.default_rng(11)
    ties = 0
    for _ in range(3000):
        D = int(rng.integers(2, 70))
        x = rng.integers(0, 6, D).astype(F64)
        if rng.random() < 0.2:
            x[rng.integers(0, D)] = rng.choice([np.nan, np.inf, -np.inf])
        S = int(rng.integers(1, 5))
        got, n = ox.pick_targets(x, S)
        kept, peaks = _kernel_rule(x, S)
        assert n == peaks
        assert got.tolist() == kept + [0] * (S - len(kept))
        vals = x[argrelmax_list(x)]
        if len(set(vals.tolist())) == len(vals) and peaks >= S:   # distinct peak values: the reference's default argsort agrees
            assert got.tolist() == [int(i) for i in orc.estimateTargetTDOAIndexesFromAngularSpectrum(x, 0.1, D, S)]
        else:
            ties += 1
    assert ties > 100


def argrelmax_list(x):
    from scipy.signal import argrelmax
    with np.errstate(invalid='ignore'):
        return argrelmax(x)[0]


def test_nearest_or_within():
    r = np.array([1.0, 1.0 + 2.0 ** -24, 1.0 + 2.0 ** -24 + 2.0 ** -40, 1e-17, np.nan])
    d = np.array([1.0, 1.0, 1.0 + 2.0 ** -23, 0.0, np.nan], F32)
    assert ox.nearest_or_within(d, r, 0.0).tolist() == [True, True, True, False, True]
    assert ox.nearest_or_within(np.array([1.0 + 2 ** -23], F32), np.array([1.0 + 2.0 ** -24]), 0.0).tolist() == [False]
    assert ox.nearest_or_within(np.array([1.0 + 2 ** -23], F32), np.array([1.0 + 2.0 ** -24]), 1e-12).tolist() == [True]
    assert ox.nearest_or_within(d[3:4], r[3:4], 1e-16).tolist() == [True]
