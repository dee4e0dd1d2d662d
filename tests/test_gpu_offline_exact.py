"""GPU: the offline stage kernels (csrc/stft.cu, csrc/gcc.cu, the masked reconstruction of csrc/gcc_tc.cu, the peak picking of
csrc/pipeline.cu) element by element against the host model of oracle/offline_exact.py, each from the device's output of the
stage before.  Every kernel form is mirrored on the host (stft_form, istft_form, angspec_form, recon_width) and the coverage
tests check that the case lists reach each form with a partial last block.
  X (STFT)           each float32 part the nearest float32 of the float64 FFT, or a neighbour within 1e-12 sum |w x| of the frame
  V, coherence, y (OLA), SIMT reconstruction, wiener filters, online targets, boxcar atom mask, masks, peak picking   bit-exact
  iFFT frames        float64 irfft, max |d| <= FRAMES_BAR x the frame's peak
  angular, mean      float64 sums within 2 F 2^-53 sum |terms| (mean: (T + 16) 2^-53 mean |ang|), same NaN pattern
  tdoa values        nearest float32 of the float64 sum or a neighbour within its float64 bound, >= 99.9 % bit-equal
  tensor-core recon  (8e-6 + 4e-8 3K/16) sum_k W (H M) + 1 float32 ulp per part
Measured worst values are printed by the last test (run with -s)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import offline_exact as ox  # noqa: E402
from oracle import rt_exact as rx  # noqa: E402

F32, F64, C64 = np.float32, np.float64, np.complex64
FRAMES_BAR = 1e-6          # 4x the worst measured on the H100 (2.4e-7)
ANGULAR_FACTOR = 2.0      # x F 2^-53 sum |terms|: 4x the worst measured (0.52)
STATS = {'stft_bit_equal': [0, 0], 'frames_err': 0.0, 'angular_ratio': 0.0, 'mean_ratio': 0.0, 'values_bit_equal': [0, 0],
         'recon_tc_ratio': 0.0, 'coherence_numpy': 0.0, 'mask_ulps': 0.0}


@pytest.fixture(scope='module')
def h():
    from gcc_nmf_b200._lib import default_handle
    return default_handle()


def _t(h, a):
    return h.to_device(np.ascontiguousarray(a))


def bits_equal(device, model):
    """Bit for bit, signed zeros included; any NaN matches any NaN."""
    d = np.ascontiguousarray(device)
    m = np.ascontiguousarray(model)
    if np.iscomplexobj(m):
        d, m = d.view(F32), m.view(F32)
    assert d.dtype == m.dtype and d.shape == m.shape, (d.dtype, m.dtype, d.shape, m.shape)
    nan = np.isnan(d) & np.isnan(m)
    udt = np.uint32 if d.dtype == F32 else np.uint64
    same = (d.view(udt) == m.view(udt)) | nan
    return bool(same.all()), np.argwhere(~same)[:4].tolist()


# ------------------------------------------------------------------------------------------------ host mirrors of the forms
def stft_form(n, C, T):
    """gccnmf_stft: FB 8 if T >= 8 and its shared memory fits 160 KiB, else 4 on the same terms, else 1."""
    F = n // 2 + 1
    smem = lambda fb: n * 16 + C * F * fb * 8   # noqa: E731
    return 8 if T >= 8 and smem(8) <= 160 * 1024 else 4 if T >= 4 and smem(4) <= 160 * 1024 else 1


def istft_form(n, T):
    F = n // 2 + 1
    smem = lambda fb: n * 8 + 2 * F * fb * 8   # noqa: E731
    return 8 if T >= 8 and smem(8) <= 160 * 1024 else 4 if T >= 4 and smem(4) <= 160 * 1024 else 1


def angspec_form(D):
    """(DPL, BF) of phat_angspec_kernel."""
    return (1, 32) if D <= 32 else (2, 16) if D <= 64 else (4, 8)


def recon_width(F):
    """gccnmf_masked_recon_planes: the first of the widths whose tiles waste the fewest F columns (strict <)."""
    bn, best = 128, 1 << 30
    for w in (128, 176, 208, 256):
        waste = -(-F // w) * w - F
        if waste < best:
            best, bn = waste, w
    return bn


def recon_tc(S, F, T, K):
    return S >= 1 and K % 8 == 0 and K >= 64 and F >= 64 and T >= 64


# ------------------------------------------------------------------------------------------------ STFT
def _stft_cases():
    cases = []
    for i, log2n in enumerate(range(5, 13)):
        n = 1 << log2n
        for C in (1, 2):
            cases.append((n, C, 13, n // 4, (i + C) % 2, n // 8, 0))          # 8q + 5 frames: a partial last block in every form
    cases += [(64, 2, T, hop, T % 2, extra, 0) for T, hop, extra in
              ((1, 64, 5), (3, 1, 0), (4, 16, 3), (7, 71, 70), (8, 64, 0), (9, 16, 15))]
    cases += [(4096, 1, 7, 1024, 0, 100, 0), (2048, 2, 6, 512, 1, 0, 0), (2048, 2, 4, 512, 1, 0, 0), (32, 1, 29, 39, 0, 38, 0),
              (256, 2, 45, 64, 1, 9, 24), (256, 1, 3, 256, 0, 0, 3)]                # last column: row padding of the samples
    return cases


STFT_CASES = _stft_cases()


def test_stft_cases_cover_every_form():
    forms = {(stft_form(n, C, T), C, T % stft_form(n, C, T) != 0) for n, C, T, *_ in STFT_CASES}
    for fb in (8, 4):
        for C in (1, 2):
            assert (fb, C, True) in forms, (fb, C)
    assert {(1, 1), (1, 2)} <= {(f, c) for f, c, _ in forms}
    assert stft_form(4096, 1, 13) == 4 and stft_form(4096, 2, 13) == 1 and stft_form(2048, 2, 13) == 4
    assert {n for n, *_ in STFT_CASES} == {1 << k for k in range(5, 13)}
    assert {hop for n, C, T, hop, *_ in STFT_CASES if n == 64} >= {1, 16, 64, 71}
    assert any(pad for *_, pad in STFT_CASES) and {1, 3, 4, 7, 8, 9} <= {T for _, _, T, *_ in STFT_CASES}


@pytest.mark.parametrize('n,C,T,hop,conj,extra,pad', STFT_CASES)
def test_stft(h, n, C, T, hop, conj, extra, pad):
    import torch
    rng = np.random.default_rng(n * 7 + C * 3 + T)
    L = n + hop * (T - 1) + extra
    x = (rng.standard_normal((C, L)) * 0.3).astype(F32)
    if T > 2:
        x[:, hop:hop + n // 3] *= F32(1e-3)                                  # a quiet stretch: weak bins next to loud ones
    window = np.hanning(n)
    F = n // 2 + 1
    if pad:
        buf = torch.zeros((C, L + pad), dtype=torch.float32, device=h.device)
        buf[:, :L] = torch.from_numpy(x).to(h.device)
        X = torch.empty((C, F, T), dtype=torch.complex64, device=h.device)
        V = torch.empty((F, C * T), dtype=torch.float32, device=h.device)
        wd = _t(h, window)
        h.check(h.lib.gccnmf_stft(h.h, buf.data_ptr(), L + pad, C, L, wd.data_ptr(), n, hop, conj, X.data_ptr(), V.data_ptr(), h.stream))
    else:
        X, V = h.stft(_t(h, x), _t(h, window), n, hop, conjugate=bool(conj), want_V=True)
    X, V = X.cpu().numpy(), V.cpu().numpy()
    ref, slack = ox.stft(x, window, n, hop, conj)
    for part in (np.real, np.imag):
        ok = ox.nearest_or_within(part(X), part(ref), slack[None, None, :])
        assert ok.all(), (np.argwhere(~ok)[:4].tolist(), int((~ok).sum()))
    STATS['stft_bit_equal'][0] += int(np.sum(X.view(F32) == np.ascontiguousarray(ref.astype(C64)).view(F32)))
    STATS['stft_bit_equal'][1] += X.size * 2
    same, where = bits_equal(V, ox.magnitudes(X, C))
    assert same, where


def test_stft_channel_one_is_not_channel_zero(h):
    """Both halves of the packed transform: a silent left channel leaves the right one's spectrum intact and vice versa."""
    rng = np.random.default_rng(2)
    x = np.zeros((2, 64 + 16 * 8), F32)
    x[1] = rng.standard_normal(x.shape[1])
    X = h.stft(_t(h, x), _t(h, np.hanning(64)), 64, 16, conjugate=True).cpu().numpy()
    ref, slack = ox.stft(x, np.hanning(64), 64, 16, 1)
    for c in (0, 1):
        for part in (np.real, np.imag):
            assert np.all(ox.nearest_or_within(part(X[c]), part(ref[c]), slack[None, :])), (c, part)


# ------------------------------------------------------------------------------------------------ iSTFT
def _istft_cases():
    cases = []
    for i, log2n in enumerate(range(5, 13)):
        n = 1 << log2n
        T = 11 if n < 4096 else 6
        cases.append((n, (1, 2, 3, 6)[i % 4], T, (n // 4, n // 2, n, n + 5)[i % 4], i % 2, (i // 2) % 2))
    cases += [(32, 3, 2, 3, 1, 1), (64, 1, 7, 16, 1, 0), (64, 2, 8, 3, 0, 1), (64, 3, 9, 32, 1, 1), (128, 1, 1, 32, 1, 1),
              (128, 3, 1, 32, 0, 1), (256, 6, 19, 69, 1, 0), (4096, 3, 3, 1024, 1, 1), (2048, 2, 5, 512, 1, 1)]
    return cases


ISTFT_CASES = _istft_cases()


def test_istft_cases_cover_every_form():
    forms = {(istft_form(n, T), B % 2, T % istft_form(n, T) != 0) for n, B, T, *_ in ISTFT_CASES}
    for fb in (8, 4):
        assert (fb, 1, True) in forms and (fb, 0, True) in forms, fb
    assert {(1, 0), (1, 1)} <= {(f, b) for f, b, _ in forms}
    assert istft_form(4096, 11) == 1 and {n for n, *_ in ISTFT_CASES} == {1 << k for k in range(5, 13)}
    assert any(T == 1 and c for _, _, T, _, c, _ in ISTFT_CASES) and any(not c for *_, c, _ in ISTFT_CASES)
    assert any(hop > n for n, _, _, hop, *_ in ISTFT_CASES) and any(n % hop for n, _, _, hop, *_ in ISTFT_CASES)


@pytest.mark.parametrize('n,B,T,hop,center,conj', ISTFT_CASES)
def test_istft(h, n, B, T, hop, center, conj):
    import torch
    rng = np.random.default_rng(n + 13 * B + T)
    F = n // 2 + 1
    spec = (rng.standard_normal((B, F, T)) + 1j * rng.standard_normal((B, F, T))).astype(C64)   # DC and Nyquist imaginary parts too
    window = np.hanning(n)
    gain = F32(hop / float(n) * 2) if hop < n else F32(0.75)
    length = ox.istft_length(n, hop, T, center)
    ws_bytes = h.lib.gccnmf_istft_workspace_bytes(B, n, T)
    ws = torch.full((ws_bytes // 4,), float('nan'), dtype=torch.float32, device=h.device)
    y = torch.empty((B, max(length, 0)), dtype=torch.float32, device=h.device)
    sd, wd = _t(h, spec), _t(h, window)
    h.check(h.lib.gccnmf_istft_ola(h.h, sd.data_ptr(), B, n, hop, T, wd.data_ptr(), float(gain), center, conj,
                                   y.data_ptr() if length > 0 else None, ws.data_ptr(), ws_bytes, h.stream))
    if length <= 0:
        assert length == 0 and torch.isnan(ws).all()                       # nothing to do: no launch
        return
    frames = ws[:B * T * n].reshape(B, T, n).cpu().numpy()
    ref = ox.ifft_frames(spec, n, conj)
    peak = np.abs(ref).max(axis=2, keepdims=True)
    err = np.abs(frames - ref) / peak
    STATS['frames_err'] = max(STATS['frames_err'], float(err.max()))
    assert float(err.max()) <= FRAMES_BAR, float(err.max())
    same, where = bits_equal(y.cpu().numpy(), ox.ola(frames, window, hop, center, gain))
    assert same, where


# ------------------------------------------------------------------------------------------------ coherence + angular spectrogram
SUBSETS = ('all', 'coherence', 'angular', 'mean')


def _angspec_cases():
    Ds = (0, 1, 3, 31, 32, 33, 64, 65, 100, 128)
    Fs = (5, 33, 65, 129, 200, 513, 2049)
    Ts = (1, 15, 16, 17, 333)
    cases = []
    for i, D in enumerate(Ds):
        for j in range(2):
            F, T = Fs[(i + 3 * j) % len(Fs)], Ts[(2 * i + j) % len(Ts)]
            if F * T > 200000:
                T = 17
            cases.append((D, F, T, (i + j) % 2, SUBSETS[(i + 2 * j) % 4] if D else 'coherence', ('plain', 'special')[j]))
    cases += [(128, 2049, 333, 0, 'all', 'plain'), (65, 513, 333, 0, 'all', 'special'), (33, 129, 17, 1, 'mean', 'plain'),
              (100, 200, 15, 0, 'angular', 'special'), (1, 65, 17, 0, 'all', 'special'), (20, 33, 31, 0, 'mean', 'special')]
    return cases


ANGSPEC_CASES = _angspec_cases()


def test_angspec_cases_cover_every_form():
    seen = set()
    for D, F, T, is_coh, subset, kind in ANGSPEC_CASES:
        if not D:
            continue
        dpl, bf = angspec_form(D)
        if D % 32 and F % bf and T % 16:
            seen.add((dpl, is_coh))
    assert seen >= {(1, 0), (2, 0), (4, 0)} and {1 for *_, c, _, _ in ANGSPEC_CASES if c}, seen
    assert {s for *_, s, _ in ANGSPEC_CASES} == set(SUBSETS)
    assert {D for D, *_ in ANGSPEC_CASES} >= {0, 1, 3, 31, 32, 33, 64, 65, 100, 128}


def _steering(F, D, seed):
    rng = np.random.default_rng(seed)
    freq = np.linspace(0, 8000, F)
    tau = np.sort(rng.uniform(-3e-4, 3e-4, D))
    return np.exp(np.outer(freq, -2j * np.pi * tau))


def _mixture(F, T, kind, seed):
    rng = np.random.default_rng(seed)
    X = (rng.standard_normal((2, F, T)) + 1j * rng.standard_normal((2, F, T))).astype(C64)
    if kind == 'special':
        X[0, F // 2, :: 3] = 0                                              # zero bins
        if T > 2:
            X[1, :, 1] = 0                                                  # one silent channel for a whole frame
        X[:, :, -1] *= F32(1e-40)                                           # subnormal
        if T > 3:
            X[:, :, T // 2] *= F32(1e18)
            X[1, 1 % F, 2] = complex(-0.0, 0.0)
    return X


@pytest.mark.parametrize('D,F,T,is_coh,subset,kind', ANGSPEC_CASES)
def test_phat_angspec(h, D, F, T, is_coh, subset, kind):
    seed = D * 1000 + F + T
    X = _mixture(F, T, kind, seed)
    E = _steering(F, D, seed) if D else None
    coh_in = ox.coherence(X) if is_coh else None
    Xd = _t(h, coh_in if is_coh else X)
    want = dict(want_coherence=subset in ('all', 'coherence'), want_angular=subset in ('all', 'angular'),
                want_mean=subset in ('all', 'mean'))
    coh, ang, mean = h.phat_angspec(Xd, _t(h, E) if D else None, **want)
    model = coh_in if is_coh else ox.coherence(X)
    if want['want_coherence']:
        same, where = bits_equal(coh.cpu().numpy(), model)
        assert same, where
        if not is_coh:
            ref = ox.numpy_coherence(X)
            fin = np.isfinite(ref) & np.isfinite(model)
            d = float(max(np.abs(model.real - ref.real)[fin].max(initial=0), np.abs(model.imag - ref.imag)[fin].max(initial=0)))
            STATS['coherence_numpy'] = max(STATS['coherence_numpy'], d)
            assert d <= 16 * 2.0 ** -24
    else:
        assert coh is None
    if not D:
        assert ang is None and mean is None
        return
    ref, bound = ox.angular(model, E)
    bound = bound * (ANGULAR_FACTOR / 4.0)
    if want['want_angular']:
        a = ang.cpu().numpy()
        assert np.array_equal(np.isnan(a), np.isnan(ref))
        fin = ~np.isnan(ref)
        r = np.abs(a - ref)[fin] / np.maximum(bound[fin], 1e-300)
        STATS['angular_ratio'] = max(STATS['angular_ratio'], float(r.max(initial=0)))
        assert np.all(np.abs(a - ref)[fin] <= bound[fin])
    if want['want_mean']:
        m = mean.cpu().numpy()
        src = ang.cpu().numpy() if want['want_angular'] else ref
        mref, mb = ox.mean_bound(src)
        if not want['want_angular']:
            mb = mb + np.where(np.isnan(bound), 0, bound).sum(axis=1) / T
        assert np.array_equal(np.isnan(m), np.isnan(mref))
        fin = ~np.isnan(mref)
        STATS['mean_ratio'] = max(STATS['mean_ratio'], float((np.abs(m - mref)[fin] / np.maximum(mb[fin], 1e-300)).max(initial=0)))
        assert np.all(np.abs(m - mref)[fin] <= mb[fin])


def test_phat_angspec_rejects_129_tdoas(h):
    from gcc_nmf_b200._lib import GCCNMFError
    X = _mixture(9, 5, 'plain', 0)
    with pytest.raises(GCCNMFError, match='UNSUPPORTED|numTDOAs'):
        h.phat_angspec(_t(h, X), _t(h, _steering(9, 129, 0)))


# ------------------------------------------------------------------------------------------------ GCC-NMF per TDOA
VALUE_CASES = [(1, 1, 1, 5), (2, 7, 7, 77), (3, 129, 9, 100), (5, 300, 513, 61), (8, 128, 8, 33), (3, 72, 513, 247)]
ARGMAX_CASES = [(4, 7, 9, 50), (8, 128, 1, 31), (16, 129, 8, 21), (32, 1, 7, 13), (64, 300, 9, 9), (128, 129, 513, 37), (128, 7, 65, 1)]


def test_tdoa_cases_are_ragged():
    for D, K, F, T in VALUE_CASES + ARGMAX_CASES:
        assert (T * D) % 128 or K % 128, (D, K, F, T)
    assert any(T * D > 256 for D, K, F, T in VALUE_CASES + ARGMAX_CASES)
    assert {D for D, *_ in ARGMAX_CASES} == {4, 8, 16, 32, 64, 128}
    assert {K for _, K, *_ in VALUE_CASES + ARGMAX_CASES} >= {1, 7, 128, 129, 300}
    assert {F for _, _, F, _ in VALUE_CASES + ARGMAX_CASES} >= {1, 7, 8, 9, 513}


def _gcc_inputs(D, K, F, T, seed, nan_frames=False):
    rng = np.random.default_rng(seed)
    X = (rng.standard_normal((2, F, T)) + 1j * rng.standard_normal((2, F, T))).astype(C64)
    coh = ox.coherence(X)
    if nan_frames:
        coh[F // 2, ::7] = np.nan
    W = ((rng.random((F, K)) ** 3) + 1e-3).astype(F32)
    return coh, _steering(F, D, seed), W


@pytest.mark.parametrize('D,K,F,T', VALUE_CASES)
def test_tdoa_gccnmf_values(h, D, K, F, T):
    coh, E, W = _gcc_inputs(D, K, F, T, D * 31 + K)
    values, argmax = h.tdoa_gccnmf(_t(h, coh), _t(h, E), _t(h, W), want_values=True, want_argmax=False)
    assert argmax is None
    v = values.cpu().numpy()
    ref, slack = ox.tdoa_values(coh, E, W)
    ok = ox.nearest_or_within(v, ref, slack)
    assert ok.all(), (np.argwhere(~ok)[:4].tolist(), int((~ok).sum()))
    equal = int(np.sum(v == ref.astype(F32)))
    STATS['values_bit_equal'][0] += equal
    STATS['values_bit_equal'][1] += v.size
    assert equal >= 0.999 * v.size, equal / v.size


@pytest.mark.parametrize('D,K,F,T', ARGMAX_CASES)
def test_tdoa_gccnmf_argmax(h, D, K, F, T):
    coh, E, W = _gcc_inputs(D, K, F, T, D * 17 + K, nan_frames=T > 7)
    _, argmax = h.tdoa_gccnmf(_t(h, coh), _t(h, E), _t(h, W), want_values=False, want_argmax=True)
    ref, _ = ox.tdoa_values(coh, E, W)
    assert np.array_equal(argmax.cpu().numpy(), ox.tdoa_argmax(ref))


# ------------------------------------------------------------------------------------------------ masks
def _nan_inf_mix(S, K, T, seed):
    rng = np.random.default_rng(seed)
    G = rng.integers(-3, 4, (S, K, T)).astype(F32)                          # small integers: many ties
    G[rng.random(G.shape) < 0.05] = np.inf
    G[rng.random(G.shape) < 0.1] = -np.inf
    G[rng.random(G.shape) < 0.05] = 0.0
    G[rng.random(G.shape) < 0.05] = -0.0
    G[0, 0, :] = np.nan                                                     # NaN first
    G[S // 2, 1, :] = np.nan                                                # NaN in the middle
    G[S - 1, 2, :] = np.nan                                                 # NaN last
    G[:, 3, ::2] = -np.inf
    G[0, 3, ::2] = np.nan                                                   # NaN before -inf: nanargmax picks the NaN's index
    G[:, 4, 1::3] = np.nan                                                  # all-NaN columns
    return G


@pytest.mark.parametrize('S', [1, 2, 3, 8, 17])
def test_coeff_mask(h, S):
    G = _nan_inf_mix(S, 37, 29, S)
    masks, flag = h.coeff_mask(_t(h, G))
    m, f = ox.coeff_mask(G)
    same, where = bits_equal(masks.cpu().numpy(), m)
    assert same, where
    assert int(flag.item()) == f == 1
    clean = G.copy()
    clean[:, np.isnan(G).all(axis=0)] = 0
    _, flag = h.coeff_mask(_t(h, clean))
    assert int(flag.item()) == 0


def test_coeff_mask_nan_before_minus_inf(h):
    """numpy.nanargmax ranks NaN as -inf: [nan, -inf] and [nan, -inf, -inf] choose index 0, and the column is not all-NaN."""
    from gcc_nmf_b200 import gccNMFFunctions as fn
    G = np.full((3, 1, 4), -np.inf, F32)
    G[0, 0, :] = np.nan
    G[1:, 0, 1] = [5.0, np.nan]
    G[2, 0, 2] = np.nan
    masks, flag = h.coeff_mask(_t(h, G))
    assert int(flag.item()) == 0
    assert np.argmax(masks.cpu().numpy()[:, 0], axis=0).tolist() == np.nanargmax(G[:, 0], axis=0).tolist() == [0, 1, 0, 0]
    two = np.array([[[np.nan]], [[-np.inf]]], F32)
    assert fn.getTargetCoefficientMasks(two, 2)[:, 0, 0].tolist() == [1.0, 0.0]


def test_argmax_mask(h):
    rng = np.random.default_rng(4)
    D = 37
    a = rng.integers(-3, D + 3, (129, 71)).astype(np.int32)
    lut = (rng.random(D) < 0.4).astype(np.uint8)
    m = h.argmax_mask(_t(h, a), _t(h, lut))
    same, where = bits_equal(m.cpu().numpy(), ox.argmax_mask(a, lut))
    assert same, where


# ------------------------------------------------------------------------------------------------ masked reconstruction
def _recon_inputs(S, F, T, K, seed, fractional):
    rng = np.random.default_rng(seed)
    X = (rng.standard_normal((2, F, T)) + 1j * rng.standard_normal((2, F, T))).astype(C64)
    X[0, F // 3, ::5] = 0
    X[1, F - 1, 1::4] = complex(-0.0, -0.0)
    X[0, 0, 2::7] = complex(-0.0, 0.0)
    X[1, F // 2, 3::6] = complex(np.nan, 0.0)
    W = ((rng.random((F, K)) ** 3) + 1e-3).astype(F32)
    H = (rng.random((K, 2 * T)) + 1e-3).astype(F32)
    masks = rng.random((S, K, T)).astype(F32) if fractional else (rng.random((S, K, T)) < 0.5).astype(F32)
    return masks, X, W, H


SIMT_CASES = [(1, 5, 3, 1, 0), (2, 130, 129, 17, 1), (3, 257, 130, 33, 0), (1, 129, 257, 16, 1), (2, 64, 64, 64, 0)]
TC_CASES = [(1, 65, 64, 64), (2, 65, 127, 72), (5, 513, 129, 64), (1, 513, 300, 1024), (2, 1025, 301, 72), (1, 200, 128, 1024),
            (2, 200, 301, 64)]


def test_recon_cases_cover_every_width():
    assert all((F % 128 or T % 128 or K % 16) for S, F, T, K, _ in SIMT_CASES[:4])
    assert {(1, 5, 3, 1)} <= {(S, F, T, K) for S, F, T, K, _ in SIMT_CASES} and {f for *_, f in SIMT_CASES} == {0, 1}
    assert any(F % 128 and T % 128 and K % 16 for S, F, T, K, _ in SIMT_CASES)
    widths = {(recon_width(F), T % 128 != 0, T % 4 != 0) for S, F, T, K in TC_CASES}
    for w in (128, 176, 208):
        assert (w, True, False) in widths or (w, True, True) in widths, w
    assert {w for w, _, _ in widths} == {128, 176, 208} and any(t for _, _, t in widths)
    assert recon_width(1025) == recon_width(200) == 208 and recon_width(513) == 176 and recon_width(65) == 128
    assert all(recon_width(F) != 256 for F in range(1, 5000))               # the 256 width can never be chosen


@pytest.mark.parametrize('S,F,T,K,frac', SIMT_CASES)
def test_masked_recon_simt(h, S, F, T, K, frac):
    masks, X, W, H = _recon_inputs(S, F, T, K, S * 100 + F + K, frac)
    out = h.masked_recon_phase(_t(h, masks), _t(h, X), _t(h, W), _t(h, H), tensor_cores=False).cpu().numpy()
    same, where = bits_equal(out, ox.recon_simt(masks, X, W, H))
    assert same, where


def _check_tc(out, masks, X, W, H):
    ref, bre, bim = ox.recon_bound(masks, X, W, H)
    for part, b in ((np.real, bre), (np.imag, bim)):
        d, r = part(out).astype(F64), part(ref)
        assert np.array_equal(np.isnan(d), np.isnan(r))
        fin = ~np.isnan(r)
        err = np.abs(d - r)[fin]
        STATS['recon_tc_ratio'] = max(STATS['recon_tc_ratio'], float((err / b[fin]).max()))
        bad = err > b[fin]
        assert not bad.any(), (int(bad.sum()), float((err / b[fin]).max()))


@pytest.mark.parametrize('S,F,T,K', TC_CASES)
def test_masked_recon_tensor_cores(h, S, F, T, K):
    assert recon_tc(S, F, T, K) and h.lib.gccnmf_masked_recon_workspace_bytes(S, F, T, K) > 256
    masks, X, W, H = _recon_inputs(S, F, T, K, S * 100 + F + K, (T + K) % 2)
    out = h.masked_recon_phase(_t(h, masks), _t(h, X), _t(h, W), _t(h, H), tensor_cores=True).cpu().numpy()
    _check_tc(out, masks, X, W, H)


def test_masked_recon_tensor_cores_unaligned(h):
    """X and out one complex64 into larger allocations: T % 4 == 0 still takes the scalar epilogue."""
    import torch
    S, F, T, K = 2, 200, 128, 72
    masks, X, W, H = _recon_inputs(S, F, T, K, 9, 1)
    Xbuf = torch.zeros(X.size + 1, dtype=torch.complex64, device=h.device)
    Xbuf[1:] = torch.from_numpy(X.reshape(-1)).to(h.device)
    obuf = torch.full((S * 2 * F * T + 1,), float('nan'), dtype=torch.complex64, device=h.device)
    md, Wd, Hd = _t(h, masks), _t(h, W), _t(h, H)
    nbytes = h.lib.gccnmf_masked_recon_workspace_bytes(S, F, T, K)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=h.device)
    h.check(h.lib.gccnmf_masked_recon_phase(h.h, md.data_ptr(), Xbuf.data_ptr() + 8, Wd.data_ptr(), Hd.data_ptr(), S, F, T, K,
                                            obuf.data_ptr() + 8, ws.data_ptr(), nbytes, h.stream))
    o = obuf.cpu().numpy()
    assert np.isnan(o[0])                                                     # nothing written before the output
    _check_tc(o[1:].reshape(S, 2, F, T), masks, X, W, H)


# ------------------------------------------------------------------------------------------------ online / Wiener-like filters
WIENER_CASES = [(5, 1, 1), (65, 127, 7), (513, 129, 129), (65, 129, 1024), (5, 127, 128), (513, 1, 1024)]


@pytest.mark.parametrize('F,T,K', WIENER_CASES)
def test_wiener_apply(h, F, T, K):
    rng = np.random.default_rng(F + T + K)
    W = ((rng.random((F, K)) ** 3) + 1e-3).astype(F32)
    W[F // 2] = 0                                                           # row sum 0: division by zero
    mask = rng.random((K, T)).astype(F32) * (rng.random((K, T)) < 0.7)
    X = (rng.standard_normal((2, F, T)) + 1j * rng.standard_normal((2, F, T))).astype(C64)
    Y, wf = h.wiener_apply(_t(h, mask), _t(h, W), _t(h, X), want_filter=True)
    Ym, wm = ox.wiener_apply(mask, W, X)
    for d, m in ((wf.cpu().numpy(), wm), (Y.cpu().numpy(), Ym)):
        same, where = bits_equal(d, m)
        assert same, where
    H = (rng.random((K, 2 * T)) + 1e-3).astype(F32)
    Y, wf = h.wiener_apply_h(_t(h, mask), _t(h, W), _t(h, H), _t(h, X), want_filter=True)
    Ym, wm = ox.wiener_apply_h(mask, W, H, X)
    for d, m in ((wf.cpu().numpy(), wm), (Y.cpu().numpy(), Ym)):
        same, where = bits_equal(d, m)
        assert same, where


@pytest.mark.parametrize('D,T', [(3, 1), (64, 127), (100, 129), (1, 17)])
def test_online_targets(h, D, T):
    rng = np.random.default_rng(D + T)
    A = rng.integers(-4, 5, (D, T)).astype(F64) + 0.5 * (rng.random((D, T)) < 0.3)   # ties in time and across TDOAs
    A[:, 0] = np.nan if T > 1 else A[:, 0]
    A[D // 2, T // 2] = np.nan
    A[:, T - 1] = np.nan if T > 2 else A[:, T - 1]
    A[-1, ::4] = -np.inf
    acc, targets = h.online_targets(_t(h, A))
    am, tm = ox.online_targets(A)
    same, where = bits_equal(acc.cpu().numpy(), am)
    assert same, where
    assert np.array_equal(targets.cpu().numpy(), tm)


@pytest.mark.parametrize('mode', [0, 1])
@pytest.mark.parametrize('per_frame', [False, True])
def test_atom_mask(h, mode, per_frame):
    rng = np.random.default_rng(mode * 2 + per_frame)
    K, T, D = 129, 127, 64
    a = rng.integers(0, D, (K, T)).astype(np.int32)
    targets = rng.integers(0, D, T).astype(np.int32) if per_frame else None
    eps, beta, nf = 3.0, 1.7, 0.05
    m = h.atom_mask(_t(h, a), _t(h, targets) if per_frame else None, 17.0, eps, mode, beta, nf).cpu().numpy()
    ref = ox.atom_mask(a, targets, 17.0, eps, mode, beta, nf)
    if mode == 0:
        same, where = bits_equal(m, ref)
        assert same, where
    else:
        mu = targets[None, :] if per_frame else 17.0
        u = rx.ulps32(m, ref)
        STATS['mask_ulps'] = max(STATS['mask_ulps'], float(u.max()))
        assert np.all(u <= rx.atom_mask_ulp_bound(a, mu, eps, beta)), float(u.max())


# ------------------------------------------------------------------------------------------------ peak picking and the fused flow
@pytest.mark.parametrize('D', [3, 5, 64, 1024])
def test_pick_targets_stable_rule(h, D):
    import torch
    rng = np.random.default_rng(D)
    for trial in range(12):
        x = rng.integers(0, 4, D).astype(F64)                               # equal peaks straddle the S boundary
        if trial % 3 == 1:
            x[rng.integers(0, D, max(1, D // 16))] = np.nan
        if trial % 3 == 2:
            x[rng.integers(0, D)] = np.inf
            x[rng.integers(0, D)] = -np.inf
        S = int(rng.integers(1, min(D, 6) + 1))
        targets = torch.full((S,), -1, dtype=torch.int32, device=h.device)
        status = torch.zeros(1, dtype=torch.int32, device=h.device)
        xd = _t(h, x)
        h.check(h.lib.gccnmf_pick_targets(h.h, xd.data_ptr(), D, S, targets.data_ptr(), status.data_ptr(), h.stream))
        want, peaks = ox.pick_targets(x, S)
        assert targets.cpu().tolist() == want.tolist(), (D, trial, S)
        assert int(status.item()) == (1 if peaks < S else 0)


def _pipeline(D=33, K=72):
    from gcc_nmf_b200.pipeline import GCCNMFPipeline
    return GCCNMFPipeline(16000, 256, 64, D, 0.1, K, 3)


def test_separate_ragged_matches_staged():
    """D = 33, S = 3, K = 72, T = 247: the fused call equals the staged pipeline (host peak picking) bit for bit."""
    import torch
    from gcc_nmf_b200.synth import synthetic_stereo
    pipe = _pipeline()
    x = pipe.h.to_device(synthetic_stereo(1.0, seed=5, num_sources=3))
    assert pipe.num_frames(x.shape[1]) == 247
    staged = pipe.separate(x, 3)
    # the stages after peak picking, from the staged run's own outputs
    E_sel = ox.gather_steering(pipe.E_host, staged['targetTDOAIndexes'])
    values = staged['targetTDOAGCCNMFs'].cpu().numpy()
    ref, slack = ox.tdoa_values(staged['coherence'].cpu().numpy(), E_sel, staged['W'].cpu().numpy())
    assert ox.nearest_or_within(values, ref, slack).all()
    m, flag = ox.coeff_mask(values)
    assert flag == 0 and bits_equal(staged['targetCoefficientMasks'].cpu().numpy(), m)[0]
    y, W, H = (staged[k].clone() for k in ('targetSignalEstimates', 'W', 'H'))
    fused = pipe.run_fused(x, 3)
    torch.cuda.synchronize()
    assert int(fused['status'].item()) == 0
    assert fused['targetTDOAIndexes'].cpu().tolist() == staged['targetTDOAIndexes']
    assert torch.equal(fused['W'], W) and torch.equal(fused['H'], H)
    assert torch.equal(fused['targetSignalEstimates'], y)


def test_separate_digital_silence_sets_status():
    """A zero stretch of N + hop samples makes one frame all zero: NaN coherence, a NaN mean angular spectrum (no peaks, bit 0)
    and all-NaN GCC-NMF columns (bit 1); the drop-in raises at peak picking."""
    import torch
    from gcc_nmf_b200.synth import synthetic_stereo
    pipe = _pipeline()
    x = synthetic_stereo(0.5, seed=6, num_sources=3)
    x[:, 2000:2000 + 256 + 64 + 10] = 0
    xd = pipe.h.to_device(x)
    fused = pipe.run_fused(xd, 3)
    torch.cuda.synchronize()
    assert int(fused['status'].item()) & 3 == 3
    with pytest.raises(ValueError):
        pipe.separate(xd, 3)


def test_zz_report_measured():
    print('\noffline exactness, measured: %s' % {k: (v[0] / max(v[1], 1) if isinstance(v, list) else v) for k, v in STATS.items()})
