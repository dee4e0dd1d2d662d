"""CPU: the bit-exact host model of the low-latency coefficient inference (oracle/ll_exact.py) -- against the real-time model on the
same columns, against a per-column scalar restatement of ll_infer_kernel, against float64, and on digital silence."""
import numpy as np
import pytest

from oracle import ll_exact as lx
from oracle import rt_exact as rx

F32, F64 = np.float32, np.float64
WARP = 32


def _case(F, K, T, seed):
    rng = np.random.default_rng(seed)
    W = (rng.random((F, K)) + 0.01).astype(F32)
    X = (rng.standard_normal((2, F, T)) + 1j * rng.standard_normal((2, F, T))).astype(np.complex64)
    H0 = rx.seeded_H0(K, 1e-16, seed)
    return W, X, H0


def _bits_equal(a, b):
    return a.shape == b.shape and np.array_equal(np.asarray(a, F32).view(np.uint32), np.asarray(b, F32).view(np.uint32))


def _warp_sum(W_rows, x, n):
    """One warp's reduction as ll_infer_kernel runs it: lane l chains acc = fmaf(W_rows[i], x[i], acc) over i = l, l + 32, ... < n
    from 0.f, then `s += shfl_xor(s, o)` for o = 16 .. 1; lane 0's value.  W_rows (n, m) reduces m outputs at once."""
    lanes = []
    for lane in range(WARP):
        acc = np.zeros(W_rows.shape[1], F32)
        for i in range(lane, n, WARP):
            acc = rx.fma32(W_rows[i], np.full(W_rows.shape[1], x[i], F32), acc)
        lanes.append(acc)
    for o in (16, 8, 4, 2, 1):
        lanes = [(lanes[l] + lanes[l ^ o]).astype(F32) for l in range(WARP)]
    return lanes[0]


def _scalar_column(W, v, h0, iterations, alpha, eps):
    F, K = W.shape
    h = np.array(h0, F32)
    cs = np.zeros(K, F32)
    for f in range(F):
        cs = (cs + W[f]).astype(F32)
    with np.errstate(all='ignore'):
        for _ in range(iterations):
            a = _warp_sum(W.T, h, K)                                   # (F,): warp per bin over k
            r = (v / a).astype(F32)
            num = _warp_sum(W, r, F)                                   # (K,): warp per atom over f
            h = (h * (num / ((cs + F32(alpha)) + F32(eps)))).astype(F32)
    return h


@pytest.mark.parametrize('F', [17, 129])
@pytest.mark.parametrize('K', [1, 31, 32, 33, 100])
def test_model_equals_the_real_time_model_on_permuted_columns(F, K):
    T = 5
    W, X, H0 = _case(F, K, T, seed=K + F)
    for iterations, alpha in ((1, 0.0), (3, 0.5)):
        got = lx.infer(X, W, H0, iterations, alpha, 1e-16)
        rt = rx.infer(X, W, H0, iterations, alpha, 1e-16)                   # column 2 t + c
        want = rt.reshape(K, T, 2).transpose(0, 2, 1).reshape(K, 2 * T)    # column c T + t
        assert _bits_equal(got, want)


@pytest.mark.parametrize('F', [17, 129])
@pytest.mark.parametrize('K', [1, 31, 32, 33, 100])
def test_model_equals_a_per_column_scalar_loop(F, K):
    T = 3
    W, X, H0 = _case(F, K, T, seed=3 * K + F)
    iterations, alpha, eps = 2, 0.5, 1e-16
    got = lx.infer(X, W, H0, iterations, alpha, eps)
    r, i = np.real(X).astype(F64), np.imag(X).astype(F64)
    V = np.sqrt(r * r + i * i).astype(F32)                                   # (2, F, T)
    for c in range(2):
        for t in range(T):
            h = _scalar_column(W, V[c, :, t], H0[:, c], iterations, alpha, eps)
            assert _bits_equal(got[:, c * T + t], h), (c, t)


@pytest.mark.parametrize('F,K', [(17, 1), (17, 100), (129, 33), (129, 256), (513, 256)])
def test_model_is_within_float32_rounding_of_float64(F, K):
    T = 4
    W, X, H0 = _case(F, K, T, seed=F * K)
    for iterations, alpha in ((1, 0.0), (2, 0.5), (7, 0.0)):
        got = lx.infer(X, W, H0, iterations, alpha, 1e-16).astype(F64)
        V = np.abs(X.astype(np.complex128))
        V = np.concatenate([V[0], V[1]], axis=1)                             # (F, 2T)
        W64 = W.astype(F64)
        H = np.repeat(H0.astype(F64), T, axis=1)
        for _ in range(iterations):
            H = H * ((W64.T @ (V / (W64 @ H))) / ((W64.sum(axis=0) + alpha) + 1e-16)[:, None])
        # every sum is of positive terms: a relative error of a few units per chain step and butterfly level, per iteration
        u = 2.0 ** -24
        bound = iterations * (-(-K // WARP) + -(-F // WARP) + 16) * 4 * u
        assert np.all(np.abs(got - H) <= bound * np.abs(H)), (iterations, np.max(np.abs(got - H) / np.abs(H)) / u)


def test_silent_column_is_finite_after_one_iteration_and_nan_after_two():
    F, K, T = 129, 33, 4
    W, X, H0 = _case(F, K, T, seed=11)
    X[:, :, 1] = 0                                   # a silent frame
    X[1, :, 3] = 0                                   # a silent channel
    silent = [1, T + 1, T + 3]
    for alpha in (0.0, 0.5):
        one = lx.infer(X, W, H0, 1, alpha, 1e-16)
        assert np.isfinite(one).all()
        assert (one[:, silent] == 0).all()           # R = 0 / (W H0) = 0, so H = H0 * 0
        for it in (2, 3):
            h = lx.infer(X, W, H0, it, alpha, 1e-16)
            assert np.isnan(h[:, silent]).all()      # W H = 0, R = 0 / 0
            others = np.setdiff1d(np.arange(2 * T), silent)
            assert np.isfinite(h[:, others]).all()


def test_column_groups():
    steer = np.array([2, 0, 2, 1])
    dic = np.array([1, 1, 0, 1])
    g = lx.column_groups(3, steer, dic)
    assert sorted(g) == [(0, 2), (1, 0), (1, 1), (1, 2)]
    assert g[(1, 2)].tolist() == [0, 1, 2]
    assert g[(0, 2)].tolist() == [6, 7, 8]
    assert g[(1, 1)].tolist() == [9, 10, 11]
    assert lx.column_groups(2, steering=np.array([1, 0]))[(0, 1)].tolist() == [0, 1]
    assert lx.column_groups(1, dictionary=np.array([0, 0]))[(0, 0)].tolist() == [0, 1]
    H = np.arange(4 * 6, dtype=F32).reshape(4, 6)           # K 4, T 3
    assert lx.split_h(H, [0, 2], 2).tolist() == [[0, 2, 3, 5], [6, 8, 9, 11]]
