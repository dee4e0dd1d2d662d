"""GPU: the offline flows that follow a moving talker (gccnmf_window_targets, gccnmf_target_gccnmf, gccnmf_argmax_mask_frames,
gccnmf_separate_tracked and the localizationWindow keyword of GCCNMFPipeline), bit for bit and NaN-equal:
  - the window means, frame targets and status against oracle/offline_window.py fed the device's own angular spectrogram, at
    D 16 / 64 / 128, P 1 / 2 / 3 / 8, w 1 / 6 / 64 / T / T + 5, with digital silence and inputs scaled by 2^+-20;
  - the per-frame contraction against the all-TDOA values gathered at each frame's targets, and its masks against numpy's rule;
  - the tracked stage chain fed the static targets in every frame against separate / enhance, byte for byte;
  - a talker who moves half way: the frame targets reach the new TDOA within w frames, the static flow keeps one target;
  - run_fused with a window against the Python tracked flow, the batch and ragged flows against the solo tracked flow;
  - every refusal leaves the launch count where it was."""
import ctypes

import numpy as np
import pytest

from oracle import offline_window as ow

pytestmark = pytest.mark.gpu

SR = 16000


@pytest.fixture(scope='module')
def h():
    from gcc_nmf_b200._lib import default_handle
    return default_handle()


def bytes_equal(a, b):
    import torch
    if a.is_complex():
        a, b = torch.view_as_real(a), torch.view_as_real(b)
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8))


def np_(t):
    return t.cpu().numpy()


def pipeline(h, N=256, hop=128, D=16, K=32, iters=20, micSep=0.1):
    from gcc_nmf_b200.pipeline import GCCNMFPipeline
    return GCCNMFPipeline(SR, N, hop, D, micSep, K, iters, handle=h)


# ------------------------------------------------------------------------------------------------ window targets
def stereo(variant, seconds=1.0, seed=21):
    from gcc_nmf_b200.synth import synthetic_stereo
    x = synthetic_stereo(seconds, SR, seed=seed, num_sources=3)
    if variant == 'silence_start':
        x[:, :3000] = 0
    elif variant == 'silence_middle':
        x[:, 6000:7500] = 0
    elif variant == 'silence_channel':
        x[1, 4000:9000] = 0
    return x


VARIANTS = ['plain', 'silence_start', 'silence_middle', 'silence_channel']


def angular(h, pipe, x):
    X = h.stft(h.to_device(np.ascontiguousarray(x, np.float32)), pipe.window, pipe.N, pipe.hop)
    _, ang, _ = h.phat_angspec(X, pipe.E)
    return ang


@pytest.mark.parametrize('D', [16, 64, 128])
@pytest.mark.parametrize('variant', VARIANTS)
def test_window_targets_match_the_oracle(h, D, variant):
    pipe = pipeline(h, D=D)
    x = stereo(variant)
    ang = angular(h, pipe, x)
    A = np_(ang)
    T = A.shape[1]
    if variant != 'plain':
        assert np.isnan(A).all(axis=0).any()              # the silence reaches whole frames
    held = 0
    for w in (1, 6, 64, T, T + 5):
        ref_means = ow.window_means(A, w)
        for P in (1, 2, 3, 8):
            targets, means, status = h.window_targets(ang, w, P)
            ref_targets, ref_status = ow.frame_targets(ref_means, P)
            assert np.array_equal(np_(means), ref_means, equal_nan=True), (w, P)
            assert np.array_equal(np_(targets), ref_targets), (w, P)
            assert int(status.item()) == ref_status, (w, P)
            held += ref_status
            if variant == 'plain' and P <= 2:
                for scale in (2.0 ** 20, 2.0 ** -20):          # PHAT is scale-free: the same decisions on scaled input
                    ang_s = angular(h, pipe, x * np.float32(scale))
                    t_s, m_s, st_s = h.window_targets(ang_s, w, P)
                    assert np.array_equal(np_(t_s), ref_targets) and int(st_s.item()) == ref_status, (scale, w, P)
                    ref_s = ow.window_targets(np_(ang_s), w, P)
                    assert np.array_equal(np_(m_s), ref_s[0], equal_nan=True) and np.array_equal(np_(t_s), ref_s[1])
    if variant != 'plain':
        assert held > 0                                     # silent frames hold


def test_window_targets_without_means(h):
    pipe = pipeline(h, D=64)
    ang = angular(h, pipe, stereo('silence_middle'))
    for w, P in ((1, 1), (9, 3), (500, 2)):
        t1, _, s1 = h.window_targets(ang, w, P)
        t1 = t1.clone()
        t2, m2, s2 = h.window_targets(ang, w, P, want_means=False)
        assert m2 is None and np.array_equal(np_(t1), np_(t2)) and int(s1.item()) == int(s2.item())


def test_window_targets_at_the_longest_clip(h):
    """T = 18747 frames (configs[3]'s length): the hold scan runs 19 chunks; w = T adds every earlier frame."""
    rng = np.random.default_rng(7)
    D, T = 64, 18747
    A = np.exp(-0.5 * ((np.arange(D)[:, None] - 20 - 20 * (np.arange(T)[None] > T // 2)) / 2.0) ** 2) + 0.05 * rng.standard_normal((D, T))
    A[:, :40] = np.nan
    A[:, 9000:9100] = 1.0
    ang = h.to_device(A)
    from oracle.rt_sources import window_mean
    for w in (6, 1024, T):
        targets, means, status = h.window_targets(ang, w, 2)
        M = np_(means)
        for t in list(range(0, 50)) + list(range(8990, 9200, 7)) + [T - 1]:
            assert np.array_equal(M[:, t], window_mean(A[:, :t + 1], t + 1, w), equal_nan=True), (w, t)
        ref_targets, ref_status = ow.frame_targets(M, 2)
        assert np.array_equal(np_(targets), ref_targets) and int(status.item()) == ref_status == 1


# ------------------------------------------------------------------------------------------------ contraction and masks
def test_contraction_is_the_all_tdoa_values_gathered(h):
    from oracle import offline_exact as ox
    pipe = pipeline(h, D=32)
    W = pipe.separate(h.to_device(stereo('plain')), 2)['W'].clone()
    X = h.stft(h.to_device(stereo('silence_middle')), pipe.window, pipe.N, pipe.hop)
    coh, _, _ = h.phat_angspec(X, pipe.E)
    T = coh.shape[1]
    allv, _ = h.tdoa_gccnmf(coh, pipe.E, W, want_values=True, want_argmax=False)
    allv = np_(allv)
    rng = np.random.default_rng(3)
    for P in (1, 3, 8):
        targets = rng.integers(0, 32, (T, P)).astype(np.int32)
        values = np_(h.target_gccnmf(coh, pipe.E, W, h.to_device(targets)))
        ref = np.stack([allv[targets[:, q], :, np.arange(T)].T for q in range(P)])
        assert np.array_equal(values, ref, equal_nan=True), P
        masks, flag = h.coeff_mask(h.to_device(values))
        m_ref, f_ref = ox.coeff_mask(values)
        assert np.array_equal(np_(masks), m_ref) and int(flag.item()) == f_ref == 1, P     # the silent frames are all NaN


def test_argmax_mask_frames_match_the_oracle(h):
    pipe = pipeline(h, D=64)
    rng = np.random.default_rng(4)
    K, T = 40, 77
    argmax = rng.integers(-1, 66, (K, T)).astype(np.int32)
    targets = rng.integers(0, 64, T).astype(np.int32)
    tdoas = np.ascontiguousarray(pipe.hypothesisTDOAs, np.float64)
    for window in (0.0, 2e-5, 4e-5, 1.0):
        mask = h.argmax_mask_frames(h.to_device(argmax), h.to_device(tdoas), h.to_device(targets), window)
        assert np.array_equal(np_(mask), ow.mask_frames(argmax, tdoas, targets, window)), window


# ------------------------------------------------------------------------------------------------ constant targets
def test_constant_targets_give_the_static_bytes(h):
    import torch
    pipe = pipeline(h, N=512, hop=128, D=64, K=64)
    x = h.to_device(stereo('plain', 1.5))
    keep = lambda r: {k: (v.clone() if hasattr(v, 'clone') else v) for k, v in r.items()}
    st = keep(pipe.separate(x, 3))
    T = st['coherence'].shape[1]
    tiled = h.to_device(np.tile(np.asarray(st['targetTDOAIndexes'], np.int32), (T, 1)))
    values = h.target_gccnmf(st['coherence'], pipe.E, st['W'], tiled)
    masks, _ = h.coeff_mask(values)
    r = pipe._back(dict(X=st['X'], W=st['W'], H=st['H']), masks, key=(pipe._token, 'constant'))
    assert bytes_equal(values, st['targetTDOAGCCNMFs']) and bytes_equal(masks, st['targetCoefficientMasks'])
    for k in ('targetSpectrogramEstimates', 'targetSignalEstimates'):
        assert bytes_equal(r[k], st[k]), k
    en = keep(pipe.enhance(x))
    tiled = h.to_device(np.full(T, en['targetTDOAIndexes'][0], np.int32))
    window = (pipe.hypothesisTDOAs[-1] - pipe.hypothesisTDOAs[0]) * pipe.windowPercent
    mask = h.argmax_mask_frames(en['argMaxGCCNMF'], pipe._tdoas_device(), tiled, window)
    assert bytes_equal(mask[None], en['targetCoefficientMasks'])
    r = pipe._back(dict(X=en['X'], W=en['W'], H=en['H']), mask[None], key=(pipe._token, 'constant'))
    for k in ('targetSpectrogramEstimates', 'targetSignalEstimates'):
        assert bytes_equal(r[k], en[k]), k
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ a talker who moves
def moving_mix(seconds=6.0, seed=5):
    """Source 0 (gain 1) at delays (0, 3) samples, then (3, 0) from the middle on; source 1 (gain 0.5) at (1, 1) throughout.  After
    the jump each channel also gets its own independent noise."""
    from scipy.signal import lfilter
    n = int(seconds * SR)
    rng = np.random.default_rng(seed)
    src = [lfilter([1.0], [1.0, -0.9], rng.standard_normal(n)) for _ in range(2)]
    x = np.zeros((2, n))
    half = n // 2
    for ch, (d0, d1) in enumerate(((0, 3), (3, 0))):
        x[ch, d0:half] += src[0][:half - d0]
        x[ch, half + d1:] += src[0][half:n - d1]
        x[ch, 1:] += 0.5 * src[1][:n - 1]
    x[:, half:] += 0.05 * rng.standard_normal((2, n - half))
    x *= 0.1 / x.std()
    return x.astype(np.float32), half


@pytest.mark.parametrize('numTargets', [0, 2])
def test_tracking_follows_the_jump(h, numTargets):
    from oracle.ll_sources import pick_peaks
    pipe = pipeline(h, N=1024, hop=256, D=64, K=64)
    x, half = moving_mix()
    xd = h.to_device(x)
    w = 64
    if numTargets:
        static = pipe.separate(xd, numTargets)
    else:
        static = pipe.enhance(xd)
    static_targets = list(static['targetTDOAIndexes'])
    A = np_(static['angularSpectrogram'])
    T = A.shape[1]
    jump = -(-half // pipe.hop)                                 # the first frame that starts after the jump
    before = jump - pipe.N // pipe.hop                          # the first frame that reaches past it
    P = max(numTargets, 1)
    old = pick_peaks(np.mean(A[:, :before], axis=1), 1)[0]
    new = pick_peaks(np.mean(A[:, jump:], axis=1), 1)[0]
    assert abs(int(old) - int(new)) > 10
    tracked = pipe.separate(xd, numTargets, localizationWindow=w) if numTargets else pipe.enhance(xd, localizationWindow=w)
    ft = np_(tracked['frameTargetTDOAIndexes'])
    assert ft.shape == (T, P)
    near = lambda row, tau: bool(np.any(np.abs(row.astype(int) - int(tau)) <= 1))
    assert all(near(ft[t], new) for t in range(jump + w, T)), ft[jump:, :]
    assert all(near(ft[t], old) for t in range(8, before)), ft[:before, :]
    if P == 1:          # the static flow has one target for the whole clip: it misses the talker on one side of the jump
        wrong = sum(1 for t in range(T) if not near(np.asarray(static_targets), new if t >= jump else old))
        assert wrong >= min(before, T - jump)


# ------------------------------------------------------------------------------------------------ fused call
@pytest.mark.parametrize('numTargets', [0, 1, 3])
def test_fused_equals_python_tracked_flow(h, numTargets):
    import torch
    pipe = pipeline(h, N=512, hop=128, D=64, K=64)
    x, _ = moving_mix(3.0, seed=8)
    x[:, :2000] = 0                                              # silent start: frames on the default targets, status bit 0
    xd = h.to_device(x)
    for w in (1, 6, 64):
        py = pipe.separate(xd, numTargets, localizationWindow=w) if numTargets else pipe.enhance(xd, localizationWindow=w)
        py = {k: (v.clone() if hasattr(v, 'clone') else v) for k, v in py.items()}
        fused = pipe.run_fused(xd, numTargets, localizationWindow=w)
        torch.cuda.synchronize()
        st = int(py['status'].item())
        if numTargets:
            st |= 2 * int(py['_all_nan_flag'].item())
        elif py['refinedDecisions'] > h.lib.gccnmf_tdoa_argmax_refine_capacity(pipe.K, py['coherence'].shape[1]):
            st |= 4
        assert int(fused['status'].item()) == st and st & 1, (w, st)
        for k in ('W', 'H', 'targetSignalEstimates', 'frameTargetTDOAIndexes', 'windowMeans'):
            assert bytes_equal(fused[k], py[k]), (w, k)
    if numTargets:      # the silent frames' all-NaN mask columns (bit 1) raise as in the static flow
        with pytest.raises(ValueError, match='All-NaN'):
            pipe.run_fused_host(x, numTargets, localizationWindow=6)
        host = pipe.run_fused_host(x, numTargets, localizationWindow=6, check=False)
    else:               # bit 0 alone does not raise in a tracked flow
        host = pipe.run_fused_host(x, numTargets, localizationWindow=6)
    assert np.array_equal(np.asarray(host), np_(pipe.run_fused(xd, numTargets, localizationWindow=6)['targetSignalEstimates']), equal_nan=True)


# ------------------------------------------------------------------------------------------------ batch flows
TRACKED_KEYS = ['W', 'H', 'angularSpectrogram', 'frameTargetTDOAIndexes', 'windowMeans', 'status', 'targetCoefficientMasks',
                'targetSpectrogramEstimates', 'targetSignalEstimates']


@pytest.mark.parametrize('flow', ['enhance', 'separate'])
@pytest.mark.parametrize('ragged', [False, True])
def test_batch_flows_equal_solo_tracked(h, flow, ragged):
    from gcc_nmf_b200.synth import synthetic_stereo
    pipe = pipeline(h, N=512, hop=128, D=64, K=64)
    w = 16
    if ragged:
        xs = [moving_mix(2.0, seed=9)[0], synthetic_stereo(1.3, SR, seed=41, num_sources=3), moving_mix(3.1, seed=10)[0]]
        clips = [h.to_device(x) for x in xs]
        batch_in = clips
    else:
        xs = [moving_mix(2.0, seed=s)[0] for s in (11, 12, 13)]
        batch_in = h.to_device(np.stack(xs))
        clips = [batch_in[b] for b in range(len(xs))]
    keep = lambda r: {k: (v.clone() if hasattr(v, 'clone') else v) for k, v in r.items()}
    if flow == 'enhance':
        batch = [keep(r) for r in pipe.enhance_batch(batch_in, localizationWindow=w)]
        singles = [keep(pipe.enhance(c, localizationWindow=w)) for c in clips]
    else:
        batch = [keep(r) for r in pipe.separate_batch(batch_in, 2, localizationWindow=w)]
        singles = [keep(pipe.separate(c, 2, localizationWindow=w)) for c in clips]
    assert len(batch) == len(xs)
    for b in range(len(xs)):
        for k in TRACKED_KEYS:
            assert bytes_equal(batch[b][k], singles[b][k]), (flow, ragged, b, k)


# ------------------------------------------------------------------------------------------------ refusals
def test_refusals_enqueue_nothing(h):
    import torch
    from gcc_nmf_b200._lib import GCCNMF_ERR_INVALID_ARGUMENT, GCCNMF_ERR_WORKSPACE, PipelineConfig, _ptr
    lib, hh, s = h.lib, h.h, h.stream
    D, T, K = 16, 50, 8
    ang = h.to_device(np.random.default_rng(0).random((D, T)))
    targets = torch.zeros((T, D + 1), dtype=torch.int32, device=h.device)
    status = torch.zeros(1, dtype=torch.int32, device=h.device)
    means = torch.empty((D, T), dtype=torch.float64, device=h.device)
    a, t, st, m = _ptr(ang), _ptr(targets), _ptr(status), _ptr(means)
    before = h.launches
    bad = [
        lambda: lib.gccnmf_window_targets(hh, a, D, T, 0, 1, m, t, st, s),
        lambda: lib.gccnmf_window_targets(hh, a, D, T, -3, 1, m, t, st, s),
        lambda: lib.gccnmf_window_targets(hh, a, D, T, 4, 0, m, t, st, s),
        lambda: lib.gccnmf_window_targets(hh, a, D, T, 4, D + 1, m, t, st, s),
        lambda: lib.gccnmf_window_targets(hh, a, 2, T, 4, 1, m, t, st, s),
        lambda: lib.gccnmf_window_targets(hh, a, 1025, T, 4, 1, m, t, st, s),
        lambda: lib.gccnmf_window_targets(hh, a, D, 1 << 30, 4, 2, m, t, st, s),
        lambda: lib.gccnmf_window_targets(hh, a, D, 0, 4, 2, m, t, st, s),
        lambda: lib.gccnmf_window_targets(hh, None, D, T, 4, 1, m, t, st, s),
        lambda: lib.gccnmf_window_targets(hh, a, D, T, 4, 1, m, None, st, s),
        lambda: lib.gccnmf_window_targets(hh, a, D, T, 4, 1, m, t, None, s),
        lambda: lib.gccnmf_target_gccnmf(hh, t, 9, 1 << 20, a, D, m, 4096, t, 1, m, s),
        lambda: lib.gccnmf_target_gccnmf(hh, t, 9, 1 << 29, a, D, m, 1, t, 4, m, s),
        lambda: lib.gccnmf_target_gccnmf(hh, None, 9, T, a, D, m, K, t, 1, m, s),
        lambda: lib.gccnmf_argmax_mask_frames(hh, t, K, T, a, 1025, t, 1e-5, m, m, s),
        lambda: lib.gccnmf_argmax_mask_frames(hh, t, K, T, a, D, t, 1e-5, None, m, s),
        lambda: lib.gccnmf_argmax_mask_frames(hh, None, K, T, a, D, t, 1e-5, m, m, s),
    ]
    for i, call in enumerate(bad):
        assert call() == GCCNMF_ERR_INVALID_ARGUMENT, i
        assert h.launches == before, i
    # the fused call: every buffer is sized from the configuration the good call passes (the pipeline's N and hop)
    pipe = pipeline(h, D=D, K=K)
    n = 8000
    x = h.to_device(stereo('plain', 0.5))
    Tf = lib.gccnmf_stft_num_frames(n, pipe.N, pipe.hop)
    assert Tf == pipe.num_frames(n) and Tf * 2 <= targets.numel()
    W0, H0 = pipe.nmf_init(2 * Tf)
    W, H = W0.clone(), H0.clone()
    assert tuple(W.shape) == (pipe.F, K) and tuple(H.shape) == (K, 2 * Tf)
    y = torch.zeros((2, 2, lib.gccnmf_istft_length(pipe.N, pipe.hop, Tf, 1)), dtype=torch.float32, device=h.device)
    tdoas = pipe._tdoas_device()

    small = torch.empty(1 << 20, dtype=torch.uint8, device=h.device)

    def fused(w=8, S=2, K_=K, N=pipe.N, ws=small, samples=_ptr(x), frame_targets=t):
        cfg = PipelineConfig(N, pipe.hop, D, K_, 2, S, 0.0, 1e-16, 1e-5)
        return lib.gccnmf_separate_tracked(hh, ctypes.byref(cfg), w, samples, n, _ptr(pipe.window), _ptr(pipe.E), _ptr(tdoas), _ptr(W), _ptr(H),
                                           _ptr(y), frame_targets, None, st, _ptr(ws), ws.numel() if ws is not None else 0, s)

    cases = [(dict(w=0), GCCNMF_ERR_INVALID_ARGUMENT), (dict(w=-1), GCCNMF_ERR_INVALID_ARGUMENT), (dict(S=D + 1), GCCNMF_ERR_INVALID_ARGUMENT),
             (dict(K_=1 << 25), GCCNMF_ERR_INVALID_ARGUMENT), (dict(samples=None), GCCNMF_ERR_INVALID_ARGUMENT),
             (dict(frame_targets=None), GCCNMF_ERR_INVALID_ARGUMENT), (dict(N=n + 1), GCCNMF_ERR_INVALID_ARGUMENT),
             (dict(ws=None), GCCNMF_ERR_WORKSPACE), (dict(ws=torch.empty(1024, dtype=torch.uint8, device=h.device)), GCCNMF_ERR_WORKSPACE)]
    assert 2 * (1 << 25) * Tf >= 1 << 31                        # S K T of the K_ case overflows int32
    for i, (kw, err) in enumerate(cases):
        assert fused(**kw) == err, (i, kw)
        assert h.launches == before, (i, kw)
    cfg = PipelineConfig(pipe.N, pipe.hop, D, K, 2, 2, 0.0, 1e-16, 1e-5)
    ws = torch.empty(lib.gccnmf_pipeline_tracked_workspace_bytes(ctypes.byref(cfg), 8, n), dtype=torch.uint8, device=h.device)
    assert fused(ws=ws) == 0 and h.launches > before             # the same arguments with a large enough workspace run
    torch.cuda.synchronize()
    from gcc_nmf_b200._lib import ParameterError
    with pytest.raises(ParameterError):
        pipe.separate(x, 2, localizationWindow=0)
    with pytest.raises(ParameterError):
        pipe.run_fused(x, 2, localizationWindow=0)
