"""GPU: the streamed online / low-latency loop (lowlatency.py, csrc/lowlatency.cu) against performOnlineSpeechEnhancement on the
whole signal, bit for bit with zero inference iterations; chunking, stream independence, reset, inactive streams, graph against
kernel-by-kernel, the gated float64 fallback inside a graph, silence and scale, inference within measured bars, argument checks."""
import os

import numpy as np
import pytest

from gcc_nmf_b200 import lowlatency as ll

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SR = 16000


def _setup(N=256, m=32, hop=32, D=16, K=64, micSep=0.1, seed=0):
    from gcc_nmf_b200 import gccNMFFunctions as fn
    from gcc_nmf_b200.online import getAsymmetricAnalysisWindow, getAsymmetricSynthesisWindow
    F = N // 2 + 1
    rng = np.random.RandomState(seed)
    W = (rng.random_sample((F, K)) + 0.01).astype(np.float32)
    E = fn.getExpJOmegaTau(fn.getFrequenciesInHz(SR, F), fn.getTDOAsInSeconds(micSep, D))
    return dict(N=N, m=m, hop=hop, D=D, K=K, W=W, E=E, micSep=micSep,
                win=getAsymmetricAnalysisWindow(N, m, 0), syn=getAsymmetricSynthesisWindow(N, m, 0))


def _stereo(n, seed=1, delay=3):
    rng = np.random.RandomState(seed)
    s = rng.standard_normal(n + delay).astype(np.float32)
    return np.stack([s[delay:], s[:n] + 0.1 * rng.standard_normal(n).astype(np.float32)]).astype(np.float32)


def _engine(p, S=1, C=1, synthesis='lowlatency', eps=None, **kw):
    return ll.LowLatencyEngine(p['W'], p['E'], p['win'], p['syn'], p['hop'], numStreams=S, hopsPerCall=C, synthesis=synthesis,
                            targetTDOAEpsilon=0.05 * p['D'] if eps is None else eps, **kw)


def _items():
    return {'X': ll.EXPORT_X, 'ang': ll.EXPORT_ANGULAR, 'acc': ll.EXPORT_ACC_MAX, 'targets': ll.EXPORT_TARGETS, 'masks': ll.EXPORT_MASKS,
            'wiener': ll.EXPORT_WIENER, 'Y': ll.EXPORT_Y, 'argmax': ll.EXPORT_ARGMAX}


def _run(eng, x, schedule, use_graph=True, frames=True):
    """x (S, 2, n) through the engine with calls of schedule[i % len] hops -> (y (S, 2, n), per-stream dict of per-frame arrays)."""
    S, _, n = x.shape
    hop = eng.hop
    ys, per = [], [dict() for _ in range(S)]
    p, i = 0, 0
    items = _items()
    while p < n:
        c = min(schedule[i % len(schedule)], (n - p) // hop)
        ys.append(eng.process(x[:, :, p:p + c * hop], use_graph=use_graph))
        if frames:
            valid = eng.export(ll.EXPORT_VALID)
            got = {k: eng.export(v) for k, v in items.items()}
            for s in range(S):
                cols = [s * c + j for j in range(c) if valid[s * c + j]]
                for k, a in got.items():
                    per[s].setdefault(k, []).append(a[..., cols])
        p += c * hop
        i += 1
    y = np.concatenate(ys, axis=2)
    per = [{k: np.concatenate(v, axis=-1) for k, v in d.items()} for d in per] if frames else None
    return y, per


def _batch(p, x, synthesis, eps=None, **kw):
    from gcc_nmf_b200.online import performOnlineSpeechEnhancement
    return performOnlineSpeechEnhancement(x, SR, p['W'], p['win'], p['syn'], p['hop'], p['D'], p['micSep'],
                                          0.05 * p['D'] if eps is None else eps, **ll.batchArguments(synthesis), **kw)


def _running_max(ang):
    acc = np.empty_like(ang)
    m = np.full(ang.shape[0], -np.inf)
    for t in range(ang.shape[1]):
        v = ang[:, t]
        m = np.where((v > m) | np.isnan(v), v, m)
        acc[:, t] = m
    return acc


def _assert_stream_equals_batch(p, eng, y, fr, x, synthesis, out_slice=True, **kw):
    X, Y, out, accLast, targets, ang, masks, wf = _batch(p, x, synthesis, **kw)
    T = X.shape[2]
    assert fr['X'].shape[-1] >= T
    assert np.array_equal(fr['X'][..., :T], X, equal_nan=True)
    assert np.array_equal(fr['ang'][..., :T], ang, equal_nan=True)
    assert np.array_equal(fr['acc'][..., :T], _running_max(ang), equal_nan=True)
    assert np.array_equal(fr['acc'][:, T - 1], accLast, equal_nan=True)
    assert np.array_equal(fr['targets'][:T], targets.astype(np.int32))
    assert np.array_equal(fr['masks'][..., :T], masks.astype(np.float32))
    w = fr['wiener'][..., :T]
    assert np.array_equal(w if w.ndim == 3 else np.stack([w, w]), wf.astype(np.float32), equal_nan=True)
    assert np.array_equal(fr['Y'][..., :T], Y, equal_nan=True)
    if out_slice:
        L, z = eng.latency, p['N'] - p['hop'] - eng.latency
        done = T * p['hop'] + z
        assert np.array_equal(y[:, L:L + done], out[:, :done], equal_nan=True)
        assert not np.any(y[:, :L])
    return T


@pytest.mark.parametrize('synthesis', ['online', 'lowlatency', 'windowed'])
def test_stream_equals_batch_synthetic(synthesis):
    p = _setup()
    x = _stereo(96 * p['hop'])
    eng = _engine(p, synthesis=synthesis)
    y, fr = _run(eng, x[None], [1])
    T = _assert_stream_equals_batch(p, eng, y[0], fr[0], x, synthesis)
    assert T > 80
    assert eng.latency == {'online': 224, 'lowlatency': 224, 'windowed': 2 * p['m'] - p['hop'] - 1}[synthesis]


@pytest.mark.parametrize('synthesis', ['online', 'lowlatency', 'windowed'])
def test_stream_equals_batch_recording(synthesis):
    from scipy.io import wavfile
    from gcc_nmf_b200 import gccNMFFunctions as fn
    sr, data = wavfile.read(os.path.join(ROOT, 'tests', 'golden', 'dev1_female3_liverec_130ms_1m_mix.wav'))
    x = data.T.astype(np.float32)
    if data.dtype == np.int16:
        x = x / 32768.0
    p = _setup(N=1024, m=64, hop=64, D=32, K=64)
    p['E'] = fn.getExpJOmegaTau(fn.getFrequenciesInHz(sr, p['N'] // 2 + 1), fn.getTDOAsInSeconds(p['micSep'], p['D']))
    assert sr == SR
    x = np.ascontiguousarray(x[:, :3 * sr // p['hop'] * p['hop']])
    eng = _engine(p, C=8, synthesis=synthesis)
    y, fr = _run(eng, x[None], [8])
    _assert_stream_equals_batch(p, eng, y[0], fr[0], x, synthesis)


def test_chunking_does_not_matter():
    p = _setup()
    x = np.stack([_stereo(72 * p['hop'], seed=s) for s in range(3)])
    ref = None
    for C, sched in ((1, [1]), (3, [3]), (8, [8]), (8, [1, 5, 8, 2, 3, 7])):
        for synthesis in ('windowed',):
            y, fr = _run(_engine(p, S=3, C=C, synthesis=synthesis), x, sched)
            got = (y, [{k: v.tobytes() for k, v in d.items()} for d in fr])
            if ref is None:
                ref = got
            assert got[0].tobytes() == ref[0].tobytes(), (C, sched)
            assert got[1] == ref[1], (C, sched)


def test_streams_are_independent():
    p = _setup()
    S = 5
    eps = [0.5, 16.5, 1.5, 15.5, 2.5]               # neighbours differ by the ~10 TDOAs between the two sources
    x = np.stack([_two_sources(p, 64 * p['hop'], seed=10 + s)[0] for s in range(S)])
    p = _two_sources(p, 64)[1]
    eng = _engine(p, S=S, C=3)
    eng.set_params(range(S), targetTDOAEpsilon=eps)
    y, fr = _run(eng, x, [3])
    for s in range(S - 1):
        # the next stream's epsilon would give other masks on this stream's decisions, so a mixed-up epsilon cannot pass unseen
        dist = np.abs(fr[s]['argmax'].astype(np.float32) - fr[s]['targets'].astype(np.float32)[None, :])
        assert not np.array_equal((dist < np.float32(eps[s + 1])).astype(np.float32), fr[s]['masks']), s
    for s in range(S):
        y1, fr1 = _run(_engine(p, S=1, C=1, eps=eps[s]), x[s:s + 1], [1])
        assert np.array_equal(y[s], y1[0])
        for k in fr1[0]:
            assert fr[s][k].tobytes() == fr1[0][k].tobytes(), (s, k)


def test_many_streams_fill_the_card():
    p = _setup()
    S = 1056                     # 8 CTAs of every per-stream kernel per SM of an H100
    base = np.stack([_stereo(40 * p['hop'], seed=s) for s in range(4)])
    x = base[np.arange(S) % 4] * (1.0 + (np.arange(S) // 4)[:, None, None].astype(np.float32) / 256)
    y, _ = _run(_engine(p, S=S, C=2), x, [2], frames=False)
    for s in (0, 1, 517, S - 1):
        y1, _ = _run(_engine(p, S=1, C=2), x[s:s + 1], [2], frames=False)
        assert np.array_equal(y[s], y1[0]), s


def test_reset_inactive_and_graph():
    p = _setup()
    x = np.stack([_stereo(64 * p['hop'], seed=s) for s in range(3)])
    eng = _engine(p, S=3, C=2, synthesis='windowed')
    half = 32 * p['hop']
    ya, _ = _run(eng, x[:, :, :half], [2], frames=False)
    eng.reset(1)
    eng.set_active(2, False)
    carry = eng.export(ll.EXPORT_CARRY)[2].copy()
    yb, _ = _run(eng, x[:, :, half:], [2], frames=False)
    assert not np.any(yb[2])
    assert np.array_equal(eng.export(ll.EXPORT_CARRY)[2], carry, equal_nan=True)
    fresh, _ = _run(_engine(p, S=1, C=2, synthesis='windowed'), x[1:2, :, half:], [2], frames=False)
    assert np.array_equal(yb[1], fresh[0])
    full, _ = _run(_engine(p, S=1, C=2, synthesis='windowed'), x[0:1], [2], frames=False)
    assert np.array_equal(np.concatenate([ya[0], yb[0]], axis=1), full[0])
    # the inactive stream resumes where it stopped: its next samples continue the first half
    eng.set_active(2, True)
    yc, _ = _run(eng, x[:, :, half:], [2], frames=False)
    cont, _ = _run(_engine(p, S=1, C=2, synthesis='windowed'), x[2:3], [2], frames=False)
    assert np.array_equal(np.concatenate([ya[2], yc[2]], axis=1), cont[0])
    # graph launches against kernel-by-kernel calls
    g, gf = _run(_engine(p, S=3, C=2), x, [2], use_graph=True)
    k, kf = _run(_engine(p, S=3, C=2), x, [2], use_graph=False)
    assert g.tobytes() == k.tobytes()
    for s in range(3):
        for key in gf[s]:
            assert gf[s][key].tobytes() == kf[s][key].tobytes()


def test_fallback_fires_inside_graph():
    """Mono input: the two central TDOAs of the symmetric grid tie in every decision, so the refinement list overflows."""
    p = _setup(D=16, K=64)
    S, C = 256, 8
    rng = np.random.RandomState(3)
    mono = rng.standard_normal((S, 1, (C + 8) * p['hop'])).astype(np.float32)
    x = np.repeat(mono, 2, axis=1)
    eng = _engine(p, S=S, C=C)
    eng.process(x[:, :, :8 * p['hop']])
    eng.process(x[:, :, 8 * p['hop']:])                 # graph launch; every frame of this call is whole
    refined = int(eng.export(ll.EXPORT_REFINED)[0])
    cap = eng.h.lib.gccnmf_tdoa_argmax_refine_capacity(p['K'], S * C)
    assert refined > cap, (refined, cap)
    assert int(eng.export(ll.EXPORT_STATUS)[0]) == 1
    h = eng.h
    coh = h.to_device(eng.export(ll.EXPORT_COHERENCE))
    _, ref = h.tdoa_gccnmf(coh, h.to_device(np.ascontiguousarray(p['E'])), h.to_device(p['W']))
    assert np.array_equal(eng.export(ll.EXPORT_ARGMAX), ref.cpu().numpy())


@pytest.mark.parametrize('where', ['start', 'middle', 'channel'])
def test_silence_gives_the_batch_nan_patterns(where):
    p = _setup()
    x = _stereo(64 * p['hop'])
    if where == 'start':
        x[:, :20 * p['hop']] = 0
    elif where == 'middle':
        x[:, 24 * p['hop']:40 * p['hop']] = 0
    else:
        x[1] = 0
    for synthesis in ('online', 'lowlatency', 'windowed'):
        eng = _engine(p, synthesis=synthesis)
        y, fr = _run(eng, x[None], [1])
        _assert_stream_equals_batch(p, eng, y[0], fr[0], x, synthesis)
        assert np.isnan(fr[0]['ang']).any()                           # the silent frames' coherence is 0 / 0
        assert np.isfinite(y).all()                                    # masks, filters and Y = filter x 0 stay finite


def test_scaled_inputs_give_identical_decisions():
    p = _setup()
    x = _stereo(48 * p['hop'])
    ref = None
    for scale in (1.0, 2.0 ** 20, 2.0 ** -20):
        _, fr = _run(_engine(p, C=4), (x * np.float32(scale))[None], [4])
        got = (fr[0]['targets'], fr[0]['argmax'], fr[0]['masks'])
        if ref is None:
            ref = got
        for a, b in zip(got, ref):
            assert np.array_equal(a, b), scale


# Inference bars: 4 x the worst relative error measured on an H100 80GB HBM3 (700 W) over both shapes and both alphas below
# (DESIGN.md section 4.6): H 1.43e-6 (against the float64 model), Wiener filters 1.20e-6 and output 8.97e-7 (against the batch).
INFER_BAR_H = 4 * 1.43e-6
INFER_BAR_WIENER = 4 * 1.20e-6
INFER_BAR_OUT = 4 * 8.97e-7


def _relerr(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.linalg.norm((a - b).ravel()) / max(np.linalg.norm(b.ravel()), 1e-300)


def _two_sources(p, n, seed=5):
    """A low-band source at one TDOA and a high-band source at another, and a dictionary of banded atoms: atoms in the low band
    localise on the first source, atoms in the high band on the second, so the atom masks of a frame are mixed."""
    rng = np.random.RandomState(seed)
    F, K = p['N'] // 2 + 1, p['K']
    f = np.fft.rfftfreq(n + 16)

    def band(lo, hi, delay):
        spec = (rng.standard_normal(len(f)) + 1j * rng.standard_normal(len(f))) * ((f >= lo) & (f < hi))
        s = np.fft.irfft(spec, n + 16)
        return np.stack([s[8:8 + n], s[8 - delay:8 - delay + n]])

    x = band(0.01, 0.2, 3) + band(0.25, 0.49, -3)
    x = (x / np.abs(x).max()).astype(np.float32)
    centres = np.linspace(0, F - 1, K)
    W = np.exp(-0.5 * ((np.arange(F)[:, None] - centres[None, :]) / (F / K * 1.5)) ** 2) + 1e-3
    return x, dict(p, W=W.astype(np.float32))


def _h_model(X, W, H0, iterations, alpha, eps):
    """Float64 H-only KL updates (gccNMFFunctions.py:76) of every (frame, channel) column from H0, V = |X| as the STFT writes it."""
    V = np.abs(X.astype(np.complex128)).astype(np.float32).astype(np.float64)      # (2, F, T)
    W = W.astype(np.float64)
    T = X.shape[2]
    H = np.concatenate([np.repeat(H0[:, c:c + 1].astype(np.float64), T, axis=1) for c in range(2)], axis=1)   # (K, 2T)
    Vc = np.concatenate([V[0], V[1]], axis=1)
    denom = (W.sum(axis=0) + alpha + eps)[:, None]
    for _ in range(iterations):
        H = H * (W.T @ (Vc / (W @ H))) / denom
    return H


@pytest.mark.parametrize('alpha', [0.0, 0.5])
@pytest.mark.parametrize('shape', ['small', 'configs4'])
def test_inference_decisions_exact_filters_bounded(shape, alpha):
    # small: the batch's H-only updates run on the float32 SIMT kernels; configs4 (2T >= 128 columns, K = 256): on the tensor cores
    p = _setup() if shape == 'small' else _setup(N=1024, m=64, hop=64, D=32, K=256)
    x, p = _two_sources(p, (64 if shape == 'small' else 96) * p['hop'] + (0 if shape == 'small' else p['N']))
    n, eps16 = 5, 1e-16
    eng = _engine(p, C=4, synthesis='online', numInferenceIterations=n, sparsityAlpha=alpha)
    y, fr = _run(eng, x[None], [4])
    X, Y, out, accLast, targets, ang, masks, wf = _batch(p, x, 'online', numInferenceIterations=n, sparsityAlpha=alpha)
    T = X.shape[2]
    assert np.array_equal(fr[0]['X'][..., :T], X)
    assert np.array_equal(fr[0]['targets'][:T], targets.astype(np.int32))
    assert np.array_equal(fr[0]['masks'][..., :T], masks.astype(np.float32))
    share = masks.mean(axis=0)
    assert np.mean((share > 0) & (share < 1)) > 0.8, share          # mixed masks: the filter depends on H
    ew = _relerr(fr[0]['wiener'][..., :T], wf)
    L, z = eng.latency, p['N'] - p['hop'] - eng.latency
    done = T * p['hop'] + z
    eo = _relerr(y[0][:, L:L + done], out[:, :done])
    # H of the last call's frames against the float64 model
    np.random.seed(0)
    H0 = (np.random.random((p['K'], 2)).astype(np.float32) + eps16).astype(np.float32)
    Hd = eng.export(ll.EXPORT_H)
    Xl = eng.export(ll.EXPORT_X)
    eh = _relerr(Hd, _h_model(Xl, p['W'], H0, n, alpha, eps16))
    print('inference %s alpha %g: H relerr %.3g, wiener relerr %.3g, output relerr %.3g' % (shape, alpha, eh, ew, eo))
    assert eh < INFER_BAR_H and ew < INFER_BAR_WIENER and eo < INFER_BAR_OUT
    # chunk invariance stays bit-exact
    y1, fr1 = _run(_engine(p, C=1, synthesis='online', numInferenceIterations=n, sparsityAlpha=alpha), x[None], [1])
    assert y1.tobytes() == y.tobytes()
    assert fr1[0]['wiener'].tobytes() == fr[0]['wiener'].tobytes()


def test_argument_checks():
    from gcc_nmf_b200._lib import ParameterError
    p = _setup()
    eng = _engine(p, S=2, C=2)
    with pytest.raises(ValueError):
        eng.process(np.zeros((2, 2, 3 * p['hop']), np.float32))        # more hops than hopsPerCall
    with pytest.raises(ValueError):
        eng.process(np.zeros((1, 2, p['hop']), np.float32))
    with pytest.raises(ValueError):
        eng.set_params(0, targetOverride=p['D'])
    with pytest.raises(ValueError):
        eng.reset(5)
    with pytest.raises(ValueError):
        _engine(p, S=0)
    with pytest.raises(ValueError):
        _engine(p, C=65)                                                  # at most 64 hops per call
    # the C entry points check before enqueueing
    import ctypes
    lib = eng.h.lib
    st = lib.gccnmf_ll_process(eng.h.h, ctypes.byref(eng.cfg), eng.state.data_ptr(), eng.state_bytes, 3, eng.state.data_ptr(),
                               eng.state.data_ptr(), eng.stream.cuda_stream)
    assert st == -1
    st = lib.gccnmf_ll_process(eng.h.h, ctypes.byref(eng.cfg), eng.state.data_ptr(), eng.state_bytes - 256, 1, eng.state.data_ptr(),
                               eng.state.data_ptr(), eng.stream.cuda_stream)
    assert st == -3
    st = lib.gccnmf_ll_export(eng.h.h, ctypes.byref(eng.cfg), eng.state.data_ptr(), eng.state_bytes, 1, 99, eng.state.data_ptr(),
                              eng.stream.cuda_stream)
    assert st == -1
    # synthesis weights whose support is shorter than a hop cannot emit a hop per call
    bad = np.zeros(p['N'])
    bad[-p['hop'] // 2:] = 1
    h = eng.h
    st = h.lib.gccnmf_ll_init(h.h, ctypes.byref(eng.cfg), eng._const[0].data_ptr(), eng._const[1].data_ptr(), eng._const[2].data_ptr(),
                              h.to_device(bad).data_ptr(), 1.0, None, eng.state.data_ptr(), eng.state_bytes, eng.stream.cuda_stream)
    with pytest.raises(ParameterError):
        h.check(st)
