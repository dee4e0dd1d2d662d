"""CPU: the bit-exact host model of a real-time block (oracle/rt_exact.py) -- its float32 fma against libm, its reduction orders
on cases small enough to follow by hand, and the whole model against the numpy restatement of the reference processor."""
import ctypes
import ctypes.util

import numpy as np
import pytest

from oracle import rt_exact as rx

F32 = np.float32


@pytest.fixture(scope='module')
def libm_fmaf():
    libm = ctypes.CDLL(ctypes.util.find_library('m') or 'libm.so.6')
    f = libm.fmaf
    f.argtypes = [ctypes.c_float] * 3
    f.restype = ctypes.c_float

    def fmaf(a, b, c):
        return np.array([f(float(x), float(y), float(z)) for x, y, z in zip(a, b, c)], F32)
    return fmaf


def _bits(x):
    return np.asarray(x, F32).view(np.uint32)


def _double_rounding_cases(rng, n):
    """Triples whose exact a * b + c lies within 2^-60 of a float32 midpoint, so float64 rounds it ONTO the midpoint:
    above it with an even c (the naive formula rounds down to c), below it with an odd c (it rounds up).  Scaled by powers
    of two and mirrored in sign."""
    out = []
    for above in (True, False):
        if above:   # a b = 2^-24 (1 + 2^-36): the exact sum is c + ulp/2 + 2^-60 for c in [1, 2)
            a, b = 2.0 ** -24 * (1 + 2.0 ** -12), 1 - 2.0 ** -12 + 2.0 ** -24
        else:       # a b = 2^-24 (1 - 2^-32): the exact sum is c + ulp/2 - 2^-56
            a, b = 2.0 ** -24 * (1 + 2.0 ** -16), 1 - 2.0 ** -16
        mant = rng.integers(0, 1 << 23, n) & ~1 | (0 if above else 1)           # even / odd last bit
        c = (np.uint32(127 << 23) | mant.astype(np.uint32)).view(F32)           # [1, 2)
        e = rng.integers(-20, 20, n).astype(np.float64)
        sign = np.where(rng.random(n) < 0.5, -1.0, 1.0)
        out.append((np.full(n, a) * 2 ** e * sign, np.full(n, b), c.astype(np.float64) * 2 ** e * sign))
    return tuple(np.concatenate(v).astype(F32) for v in zip(*out))


def test_fma_emulator_fixes_double_rounding(libm_fmaf):
    # the case spelled out: exact sum 1 + 2^-24 + 2^-60 -> fmaf 1 + 2^-23, naive float64 then float32 -> 1.0
    a, b, c = F32(2.0 ** -24 * (1 + 2.0 ** -12)), F32(1 - 2.0 ** -12 + 2.0 ** -24), F32(1.0)
    assert float(a) == 2.0 ** -24 * (1 + 2.0 ** -12) and float(b) == 1 - 2.0 ** -12 + 2.0 ** -24
    assert libm_fmaf([a], [b], [c])[0] == F32(1 + 2.0 ** -23)
    assert rx.fma32(a, b, c) == F32(1 + 2.0 ** -23)
    assert rx.fma32_naive(a, b, c) == F32(1.0)
    a, b, c = _double_rounding_cases(np.random.default_rng(0), 2000)
    ref = libm_fmaf(a, b, c)
    assert np.array_equal(_bits(rx.fma32(a, b, c)), _bits(ref))
    assert not np.any(_bits(rx.fma32_naive(a, b, c)) == _bits(ref))       # every constructed case defeats the naive formula


def test_fma_emulator_matches_libm_on_random_cancelling_and_special_triples(libm_fmaf):
    rng = np.random.default_rng(1)
    n = 60000
    a = (rng.standard_normal(n) * 2.0 ** rng.integers(-30, 30, n)).astype(F32)
    b = (rng.standard_normal(n) * 2.0 ** rng.integers(-30, 30, n)).astype(F32)
    c = (rng.standard_normal(n) * 2.0 ** rng.integers(-60, 60, n)).astype(F32)
    half = n // 2                                                          # c ~ -a b: catastrophic cancellation
    c[:half] = (-(a[:half].astype(np.float64) * b[:half]) * (1 + 2.0 ** -20 * rng.standard_normal(half))).astype(F32)
    # signed zeros, and subnormal products and addends
    z = np.array([0.0, -0.0, 0.0, -0.0, 1.0, -1.0, 0.0, -0.0], F32)
    sa = np.concatenate([z, (rng.random(2000) * 2.0 ** -70).astype(F32), np.full(2000, 2.0 ** -126, F32)])
    sb = np.concatenate([z[::-1], (rng.random(2000) * 2.0 ** -70).astype(F32), (rng.random(2000) * 0.5).astype(F32)])
    sc = np.concatenate([np.array([-0.0, -0.0, 0.0, 0.0, 0.0, 0.0, -0.0, 0.0], F32),
                         rng.integers(1, 1 << 23, 2000).astype(np.uint32).view(F32) * np.where(rng.random(2000) < 0.5, -1, 1).astype(F32),
                         -rng.integers(1, 1 << 23, 2000).astype(np.uint32).view(F32)])
    a, b, c = np.concatenate([a, sa]), np.concatenate([b, sb]), np.concatenate([c, sc])
    ref = libm_fmaf(a, b, c)
    got = rx.fma32(a, b, c)
    bad = np.flatnonzero(_bits(got) != _bits(ref))
    assert bad.size == 0, [(float(a[i]), float(b[i]), float(c[i]), float(got[i]), float(ref[i])) for i in bad[:5]]
    assert np.any(np.abs(ref[n:]) < 2.0 ** -126) and np.any(np.signbit(ref[:8]))      # subnormal results and a -0 were exercised


def test_butterfly_order_by_hand():
    # lanes 0, 1, 3 = 2^24, 1, 1: the butterfly adds lane 1 + lane 3 (= 2) at o = 2 and then 2^24 + 2 exactly at o = 1; a
    # sequential float32 sum loses both ones (2^24 + 1 rounds to 2^24, twice)
    s = np.zeros(32, F32)
    s[0], s[1], s[3] = 2.0 ** 24, 1.0, 1.0
    assert rx.butterfly(s) == F32(2.0 ** 24 + 2)
    seq = F32(0)
    for v in s:
        seq = F32(seq + v)
    assert seq == F32(2.0 ** 24)
    # lane-strided chains: K = 40 -> lanes 0..7 see k = l and l + 32, the others k = l only
    a = np.ones((40, 1), F32)
    b = np.zeros((40, 1), F32)
    b[0], b[32], b[5] = 2.0 ** 24, 1.0, 3.0
    acc = rx.lane_fma_chains(a, b, 40)
    assert acc.shape == (32, 1) and acc[0, 0] == F32(2.0 ** 24) and acc[5, 0] == 3 and acc[1:5].sum() == 0


def test_gccphat_order_by_hand():
    """The lane-strided float64 nanmean against the kernel's loops written out scalar by scalar."""
    rng = np.random.default_rng(2)
    nT, D, F = 2, 3, 75
    G = (rng.standard_normal((nT, D, F)) * 10.0 ** rng.integers(-8, 8, (nT, D, F))).astype(F32)
    G[0, 1, ::7] = np.nan
    G[1, 2, :] = np.nan
    out = rx.gccphat(G)
    for t in range(nT):
        for d in range(D):
            sums, cnt = [0.0] * 32, [0] * 32
            for lane in range(32):
                for f in range(lane, F, 32):
                    v = G[t, d, f]
                    if v == v:
                        sums[lane] += float(v)
                        cnt[lane] += 1
            for o in (16, 8, 4, 2, 1):
                sums = [sums[i] + sums[i ^ o] for i in range(32)]
                cnt = [cnt[i] + cnt[i ^ o] for i in range(32)]
            want = F32(sums[0] / cnt[0]) if cnt[0] else F32(np.nan)
            assert np.array_equal(out[d, t], want, equal_nan=True), (t, d)


def test_localize_ring_by_hand():
    """History of length 5 fed 4 columns per block: the write wraps inside a block, and a window longer than the history is the
    whole history.  NaN columns are skipped by the nanmean."""
    D, L = 3, 5
    hist, idx, tgt = np.zeros((D, L)), 0, np.float32(1)
    cols = [np.array([[1, 2, 3, 4], [0, 0, 0, 9], [5, 5, 5, 5]], F32), np.array([[np.nan, 1, 1, 1], [8, 8, 8, 8], [0, 0, 0, 0]], F32)]
    hist, idx, tgt = rx.localize(hist, idx, cols[0], 3, True, tgt)
    assert idx == 4 and tgt == 2                                     # means of columns 3, 2, 1: [3, 3, 5]
    hist, idx, tgt = rx.localize(hist, idx, cols[1], 200, True, tgt)
    assert idx == 3
    assert np.array_equal(hist[0], [1, 1, 1, 4, np.nan], equal_nan=True)
    assert tgt == 1                                                  # whole ring: [7/4, 41/5, 1]
    _, _, kept = rx.localize(hist, idx, cols[1], 2, False, tgt)
    assert kept == tgt


@pytest.mark.parametrize('tag,nT,mode', [('w1', 1, 2), ('b4', 4, 0), ('w4', 4, 2)])
def test_model_against_reference_processor_fixture(golden, tag, nT, mode):
    """The model's stages chained (no device) against realtime_mini, the unmodified reference processor on numpy arithmetic.
    The per-atom TDOA decisions must agree wherever the float64 gap between the two best TDOAs exceeds the float32 error bound
    of the two contractions, F 2^-22 sum_f |W[f, k]| (|realGCC| <= 1); the localisation decisions everywhere; the GCC-PHAT
    columns to float32 rounding; the output frames, where every decision agrees, to 1e-5 of their peak."""
    from oracle import gccnmf_oracle as orc
    g = golden('realtime_mini')
    sr, N, K, D = [int(v) for v in g['params']]
    W = g['W']
    F = W.shape[0]
    ref = orc.GCCNMFProcessorOracle(sr, N, nT, W, D, float(g['micSep']))
    win = ref.windowFunction[:, 0]
    idx0, eps, beta, nf = [float(v) for v in g['targetRange']]
    hist, hidx, target = np.zeros((D, 128)), 0, F32(idx0)
    bound = F * 2.0 ** -22 * np.abs(W).sum(axis=0)                  # (K,)
    checked = 0
    for i in range(g[tag + '_frames'].shape[0]):
        frames = g[tag + '_frames'][i]
        X = rx.analysis(frames, win)
        G = rx.real_gcc(X, ref.expJOmegaTau)
        gcc = rx.gccphat(G)
        np.testing.assert_allclose(gcc, g[tag + '_gccphat'][i], rtol=0, atol=2e-6)
        am = rx.argmax_over_tdoa(rx.atoms(G, W))
        C64 = np.einsum('tdf,fk->tdk', G.astype(np.float64), W.astype(np.float64))
        top2 = np.sort(C64, axis=1)[:, -2:, :]
        clear = (top2[:, 1] - top2[:, 0] > bound[None]).T             # (K, nT)
        assert np.array_equal(am[clear], g[tag + '_argmax'][i][clear])
        checked += int(clear.sum())
        mask = rx.atom_mask(am, target, eps, beta, nf, 0 if mode == 0 else 1)
        if np.array_equal(am, g[tag + '_argmax'][i]):
            np.testing.assert_allclose(mask, g[tag + '_hmask'][i], rtol=1e-15, atol=0)
            y = rx.synthesis(rx.filter_spectrum(X, W, mask), win)
            assert np.abs(y - g[tag + '_y'][i]).max() <= 1e-5 * np.abs(g[tag + '_y'][i]).max()
        hist, hidx, target = rx.localize(hist, hidx, gcc, 6, True, target)
        assert target == g[tag + '_target'][i]
    assert checked >= 0.9 * g[tag + '_frames'].shape[0] * K * nT, checked
