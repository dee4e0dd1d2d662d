"""GPU: the low-latency engine with several sources per stream (LowLatencyEngine(numSources=P), gccnmf_llsep_*).  Decisions bit for
bit against the host model (oracle/ll_sources.py) fed the device's angular spectrum; values and masks bit for bit against the
all-TDOA contraction and coeff_mask; every source bit for bit against performOnlineSpeechEnhancement fed its masks; inference;
the sum of the sources; independence of streams, call sizes and graphs; silence, scale and argument checks."""
import ctypes

import numpy as np
import pytest

from gcc_nmf_b200 import lowlatency as ll
from oracle import ll_sources as model

pytestmark = pytest.mark.gpu

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


def _moving(n, seed=1, delays=(-3, 0, 3)):
    """Delayed sources entering one after the other: source i (delay delays[i] between the channels) starts at i n / len(delays),
    so the peaks of the running maximum move while the stream runs."""
    rng = np.random.RandomState(seed)
    x = np.zeros((2, n))
    for i, d in enumerate(delays):
        s = rng.standard_normal(n + 16)
        start = i * n // len(delays)
        part = np.stack([s[8:8 + n], s[8 - d:8 - d + n]])
        part[:, :start] = 0
        x += part
    return (x / np.abs(x).max()).astype(np.float32)


def _engine(p, S=1, C=1, P=3, synthesis='lowlatency', **kw):
    return ll.LowLatencyEngine(p['W'], p['E'], p['win'], p['syn'], p['hop'], numStreams=S, hopsPerCall=C, synthesis=synthesis,
                               numSources=P, **kw)


ITEMS = {'X': ll.EXPORT_X, 'ang': ll.EXPORT_ANGULAR, 'acc': ll.EXPORT_ACC_MAX, 'targets': ll.EXPORT_SOURCE_TARGETS,
         'values': ll.EXPORT_SOURCE_VALUES, 'masks': ll.EXPORT_SOURCE_MASKS, 'wiener': ll.EXPORT_SOURCE_WIENER, 'Y': ll.EXPORT_SOURCE_Y}


def _run(eng, x, schedule, use_graph=True, frames=True, check_values=None):
    """x (S, 2, n) through the engine with calls of schedule[i % len] hops -> (y (S, P, 2, n), per-stream dict of per-valid-frame
    arrays with the frame last, call status words).  check_values = (W, E): every call's values and masks are checked bit for bit
    against the all-TDOA contraction of its exported coherence, gathered at its column targets, and coeff_mask of those."""
    S, _, n = x.shape
    hop = eng.hop
    ys, per, calls = [], [dict() for _ in range(S)], []
    p, i = 0, 0
    while p < n:
        c = min(schedule[i % len(schedule)], (n - p) // hop)
        ys.append(eng.process(x[:, :, p:p + c * hop], use_graph=use_graph))
        calls.append(int(eng.export(ll.EXPORT_CALL_STATUS)[0]))
        if frames:
            valid = eng.export(ll.EXPORT_VALID)
            got = {k: eng.export(v) for k, v in ITEMS.items()}
            got['targets'] = np.ascontiguousarray(got['targets'].T)                    # (P, T)
            if check_values is not None:
                _check_values(eng, got, calls[-1], *check_values)
            for s in range(S):
                cols = [s * c + j for j in range(c) if valid[s * c + j]]
                for k, a in got.items():
                    per[s].setdefault(k, []).append(a[..., cols])
        p += c * hop
        i += 1
    y = np.concatenate(ys, axis=-1)
    per = [{k: np.concatenate(v, axis=-1) for k, v in d.items()} for d in per] if frames else None
    return y, per, calls


def _check_values(eng, got, call_status, W, E):
    h = eng.h
    coh = h.to_device(eng.export(ll.EXPORT_COHERENCE))
    every, _ = h.tdoa_gccnmf(coh, h.to_device(np.ascontiguousarray(E)), h.to_device(W), want_values=True, want_argmax=False)
    every = every.cpu().numpy()                                                            # (D, K, T)
    tg = got['targets']                                                                    # (P, T)
    T = tg.shape[1]
    ref = np.stack([every[tg[q], :, np.arange(T)].T for q in range(tg.shape[0])])           # (P, K, T)
    assert ref.tobytes() == got['values'].tobytes()
    masks, flag = h.coeff_mask(h.to_device(ref))
    assert np.array_equal(masks.cpu().numpy(), got['masks'])
    assert call_status == (ll.STATUS_ALL_NAN if int(flag.cpu().numpy()[0]) else 0)


def _check_decisions(eng, fr, D, P, stream=0, override=None, status=None):
    """The running maximum and column targets of every valid frame, the carried targets and the status against the model."""
    m = model.SourceTargets(D, P)
    if override is not None:
        m.set_override(override)
    for j in range(fr['ang'].shape[1]):
        acc, t = m.frame(fr['ang'][:, j])
        assert np.array_equal(fr['acc'][:, j], acc, equal_nan=True), j
        assert fr['targets'][:, j].tolist() == t.tolist(), j
    assert eng.export(ll.EXPORT_CARRIED_TARGETS)[stream].tolist() == m.targets.tolist()
    assert int(eng.export(ll.EXPORT_STREAM_STATUS)[stream]) == m.status
    if status is not None:
        assert m.status == status
    return m


def _batch(p, x, synthesis, mask, **kw):
    from gcc_nmf_b200.online import performOnlineSpeechEnhancement
    return performOnlineSpeechEnhancement(x, SR, p['W'], p['win'], p['syn'], p['hop'], p['D'], p['micSep'], 1.0,
                                          _forcedAtomMasks=mask, **ll.batchArguments(synthesis), **kw)


def _assert_sources_equal_batch(p, eng, y, fr, x, synthesis):
    """Source q's samples == the batch function fed the exported masks of source q, shifted by the latency."""
    T = (x.shape[1] - p['N']) // p['hop']
    L, z = eng.latency, p['N'] - p['hop'] - eng.latency
    done = T * p['hop'] + z
    for q in range(eng.P):
        X, Y, out, _, _, _, masks, wf = _batch(p, x, synthesis, fr['masks'][q][:, :T])
        assert np.array_equal(fr['X'][..., :T], X)
        assert np.array_equal(fr['Y'][q][..., :T], Y, equal_nan=True), q
        assert np.array_equal(fr['wiener'][q][..., :T], wf[0].astype(np.float32), equal_nan=True), q
        assert np.array_equal(y[q][:, L:L + done], out[:, :done]), q
        assert not np.any(y[q][:, :L])
    return T


CASES = [(2, 16, 'online', 1), (2, 128, 'windowed', 3), (3, 16, 'lowlatency', 8), (3, 128, 'online', 3), (8, 16, 'windowed', 1),
         (8, 128, 'lowlatency', 8)]


@pytest.mark.parametrize('P,D,synthesis,C', CASES)
def test_decisions_values_masks_and_sources_exact(P, D, synthesis, C):
    p = _setup(D=D)
    x = _moving(96 * p['hop'])
    eng = _engine(p, C=C, P=P, synthesis=synthesis)
    y, fr, calls = _run(eng, x[None], [C], check_values=(p['W'], p['E']))
    m = _check_decisions(eng, fr[0], D, P)
    print('P %d D %d: %d distinct target sets over %d frames, status %d' % (P, D, len({tuple(t) for t in fr[0]['targets'].T}),
                                                                          fr[0]['targets'].shape[1], m.status))
    assert np.array_equal(fr[0]['masks'].sum(axis=0), np.ones(fr[0]['masks'].shape[1:]))     # no NaN here: a partition
    assert not any(calls)
    _assert_sources_equal_batch(p, eng, y[0], fr[0], x, synthesis)


def _sum_bar(y_sum, y_all):
    return np.abs(y_sum.astype(np.float64) - y_all).max() <= 1e-6 * np.abs(y_all).max()


@pytest.mark.parametrize('iterations', [0, 5])
def test_sources_sum_to_the_all_atoms_output(iterations):
    p = _setup(D=32)
    x = _moving(64 * p['hop'])
    y, _, _ = _run(_engine(p, C=4, P=3, synthesis='windowed', numInferenceIterations=iterations), x[None], [4], frames=False)
    single = ll.LowLatencyEngine(p['W'], p['E'], p['win'], p['syn'], p['hop'], hopsPerCall=4, synthesis='windowed',
                                 targetTDOAEpsilon=p['D'] + 1.0, numInferenceIterations=iterations)
    ys = np.concatenate([single.process(x[None, :, i:i + 4 * p['hop']]) for i in range(0, x.shape[1], 4 * p['hop'])], axis=-1)
    assert np.abs(ys).max() > 0
    assert _sum_bar(y[0].sum(axis=0), ys[0])


# Inference bars of DESIGN.md section 4.6 (tests/test_gpu_lowlatency.py): Wiener filters and output against the batch.
INFER_BAR_WIENER = 4 * 1.20e-6
INFER_BAR_OUT = 4 * 8.97e-7


def _relerr(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.linalg.norm((a - b).ravel()) / max(np.linalg.norm(b.ravel()), 1e-300)


@pytest.mark.parametrize('alpha', [0.0, 0.5])
def test_inference_shares_h_and_filters_are_exact(alpha):
    p = _setup(D=32)
    x = _moving(64 * p['hop'])
    n, P, C = 5, 3, 4
    eng = _engine(p, C=C, P=P, synthesis='online', numInferenceIterations=n, sparsityAlpha=alpha)
    single = ll.LowLatencyEngine(p['W'], p['E'], p['win'], p['syn'], p['hop'], hopsPerCall=C, synthesis='online',
                                 numInferenceIterations=n, sparsityAlpha=alpha)
    h = eng.h
    ys, masks = [], []
    for i in range(0, x.shape[1], C * p['hop']):
        chunk = x[None, :, i:i + C * p['hop']]
        ys.append(eng.process(chunk))
        single.process(chunk)
        H = eng.export(ll.EXPORT_H)
        assert H.tobytes() == single.export(ll.EXPORT_H).tobytes()
        mk, X, wf = eng.export(ll.EXPORT_SOURCE_MASKS), eng.export(ll.EXPORT_X), eng.export(ll.EXPORT_SOURCE_WIENER)
        for q in range(P):
            _, ref = h.wiener_apply_h(h.to_device(mk[q]), h.to_device(p['W']), h.to_device(H), h.to_device(X), want_filter=True)
            assert ref.cpu().numpy().tobytes() == wf[q].tobytes(), q
        valid = eng.export(ll.EXPORT_VALID)
        masks.append(mk[..., valid.astype(bool)])
    y = np.concatenate(ys, axis=-1)[0]
    masks = np.concatenate(masks, axis=-1)
    T = (x.shape[1] - p['N']) // p['hop']
    L, z = eng.latency, p['N'] - p['hop'] - eng.latency
    done = T * p['hop'] + z
    for q in range(P):
        _, _, out, _, _, _, _, _ = _batch(p, x, 'online', masks[q][:, :T], numInferenceIterations=n, sparsityAlpha=alpha)
        eo = _relerr(y[q][:, L:L + done], out[:, :done])
        print('inference alpha %g source %d: output relerr %.3g' % (alpha, q, eo))
        assert eo < INFER_BAR_OUT


def test_call_schedules_do_not_matter():
    p = _setup(D=32)
    x = np.stack([_moving(72 * p['hop'], seed=s) for s in range(3)])
    ref = None
    for C, sched in ((1, [1]), (3, [3]), (8, [8]), (8, [1, 5, 8, 2, 3, 7])):
        y, fr, _ = _run(_engine(p, S=3, C=C, P=3, synthesis='windowed'), x, sched)
        got = (y.tobytes(), [{k: v.tobytes() for k, v in d.items()} for d in fr])
        if ref is None:
            ref = got
        assert got[0] == ref[0], (C, sched)
        assert got[1] == ref[1], (C, sched)


def test_heterogeneous_streams_equal_one_stream_engines():
    """S = 5: defaults, a partial override, a full override, an inactive stream and one reset half way; each equals a one-stream
    engine with the same settings, and the graph equals kernel-by-kernel calls."""
    p = _setup(D=32)
    S, P, C = 5, 3, 2
    x = np.stack([_moving(64 * p['hop'], seed=20 + s) for s in range(S)])
    over = {1: [-1, 9, -1], 2: [3, 16, 28]}
    half = 32 * p['hop']

    def configure(e, s_of):
        for s, t in over.items():
            if s in s_of:
                e.set_targets(s_of.index(s), t)
        if 3 in s_of:
            e.set_active(s_of.index(3), False)

    for use_graph in (True, False):
        eng = _engine(p, S=S, C=C, P=P)
        configure(eng, list(range(S)))
        ya, fa, _ = _run(eng, x[:, :, :half], [C], use_graph=use_graph)
        eng.reset(4)
        yb, fb, _ = _run(eng, x[:, :, half:], [C], use_graph=use_graph)
        assert not np.any(ya[3]) and not np.any(yb[3])
        for s in range(S):
            one = _engine(p, S=1, C=C, P=P)
            configure(one, [s])
            if s == 4:
                y1a, _, _ = _run(one, x[s:s + 1, :, :half], [C], frames=False)
                one.reset()
                y1b, f1b, _ = _run(one, x[s:s + 1, :, half:], [C])
                assert np.array_equal(ya[s], y1a[0]) and np.array_equal(yb[s], y1b[0])
                for k in f1b[0]:
                    assert fb[s][k].tobytes() == f1b[0][k].tobytes(), (s, k)
                continue
            y1, f1, _ = _run(one, x[s:s + 1], [C])
            assert np.array_equal(np.concatenate([ya[s], yb[s]], axis=-1), y1[0]), s
            for k in f1[0]:
                assert np.concatenate([fa[s][k], fb[s][k]], axis=-1).tobytes() == f1[0][k].tobytes(), (s, k)
        if use_graph:
            ref = (ya.tobytes(), yb.tobytes())
        else:
            assert (ya.tobytes(), yb.tobytes()) == ref
    # the overrides replace their sources' targets and leave the others to the localisation
    _check_decisions(eng, {k: np.concatenate([fa[1][k], fb[1][k]], axis=-1) for k in fa[1]}, p['D'], P, stream=1, override=over[1])


def test_many_streams_fill_the_card():
    p = _setup(D=32)
    S, C, P = 1056, 2, 3
    base = np.stack([_moving(40 * p['hop'], seed=s) for s in range(4)])
    x = base[np.arange(S) % 4] * (1.0 + (np.arange(S) // 4)[:, None, None].astype(np.float32) / 256)
    y, _, _ = _run(_engine(p, S=S, C=C, P=P), x, [C], frames=False)
    for s in (0, 1, 517, S - 1):
        y1, _, _ = _run(_engine(p, S=1, C=C, P=P), x[s:s + 1], [C], frames=False)
        assert np.array_equal(y[s], y1[0]), s


@pytest.mark.parametrize('where', ['start', 'middle', 'channel'])
def test_silence(where):
    p = _setup(D=32)
    x = _moving(64 * p['hop'])
    if where == 'start':
        x[:, :20 * p['hop']] = 0
    elif where == 'middle':
        x[:, 24 * p['hop']:40 * p['hop']] = 0
    else:
        x[1] = 0
    for synthesis in ('online', 'lowlatency', 'windowed'):
        eng = _engine(p, C=3, P=3, synthesis=synthesis)
        y, fr, calls = _run(eng, x[None], [3], check_values=(p['W'], p['E']))
        m = _check_decisions(eng, fr[0], p['D'], 3)
        assert np.isnan(fr[0]['ang']).any()
        # a silent frame's angular spectrum is NaN everywhere: it sticks in the running maximum, which then has no peak
        assert m.status == model.STATUS_FEW_PEAKS
        assert any(c == ll.STATUS_ALL_NAN for c in calls)
        dead = np.isnan(fr[0]['values']).all(axis=0)
        assert dead.any() and not fr[0]['masks'][:, dead].any()                     # an all-NaN (k, t) goes to no source
        _assert_sources_equal_batch(p, eng, y[0], fr[0], x, synthesis)
        assert np.isfinite(y).all()


def test_scaled_inputs_give_identical_decisions():
    p = _setup(D=32)
    x = _moving(48 * p['hop'])
    ref = None
    for scale in (1.0, 2.0 ** 20, 2.0 ** -20):
        _, fr, _ = _run(_engine(p, C=4, P=3), (x * np.float32(scale))[None], [4])
        got = (fr[0]['targets'], fr[0]['masks'])
        if ref is None:
            ref = got
        for a, b in zip(got, ref):
            assert np.array_equal(a, b), scale


def test_refusals_launch_nothing():
    from gcc_nmf_b200._lib import ParameterError
    p = _setup()
    P = 3
    eng = _engine(p, S=2, C=2, P=P)
    eng.process(np.zeros((2, 2, p['hop']), np.float32))
    h, lib = eng.h, eng.h.lib
    with pytest.raises(ValueError):
        _engine(p, P=1)
    with pytest.raises(ValueError):
        _engine(p, P=9)
    with pytest.raises(ValueError):
        eng.set_targets(0, [0, 1, p['D']])
    with pytest.raises(ValueError):
        eng.set_targets(0, [0, -2, 1])
    with pytest.raises(ValueError):
        ll.LowLatencyEngine(p['W'], p['E'], p['win'], p['syn'], p['hop']).set_targets(0, [1, 2])
    before = h.launches
    cfg, st, nb, cs = ctypes.byref(eng.cfg), eng.state.data_ptr(), eng.state_bytes, eng.stream.cuda_stream
    bad = (np.array([[0, 1, p['D']], [0, 1, 2]], np.int32), np.array([[0, -3, 1], [0, 1, 2]], np.int32))
    for t in bad:
        assert lib.gccnmf_llsep_set_targets(h.h, cfg, P, st, nb, 0, 2, t.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), cs) == -1
    for q in (0, 1, 9):
        assert lib.gccnmf_llsep_process(h.h, cfg, q, st, nb, 1, st, st, cs) == -1, q
    assert lib.gccnmf_llsep_process(h.h, cfg, P, st, nb, 3, st, st, cs) == -1                 # more hops than hops_per_call
    assert lib.gccnmf_llsep_process(h.h, cfg, P, st, nb - 256, 1, st, st, cs) == -3
    assert lib.gccnmf_llsep_process(h.h, cfg, P + 1, st, nb, 1, st, st, cs) == -3               # a state carved for fewer sources
    for what in range(4, 11):
        assert lib.gccnmf_llsep_export(h.h, cfg, P, st, nb, 1, what, st, cs) == -1, what     # not computed with sources
    assert lib.gccnmf_llsep_export(h.h, cfg, P, st, nb, 1, 22, st, cs) == -1
    big = ll.LLConfig(p['N'], p['hop'], 2, 60000, p['D'], 4096, 0, 0.0, 1e-16)
    assert lib.gccnmf_llsep_process(h.h, ctypes.byref(big), 8, st, nb, 1, st, st, cs) == -1    # P K T overflows int32
    assert h.launches == before
    # the single-target entries do not know the source items
    one = ll.LowLatencyEngine(p['W'], p['E'], p['win'], p['syn'], p['hop'])
    one.process(np.zeros((1, 2, p['hop']), np.float32))
    with pytest.raises(Exception):
        one.export(ll.EXPORT_SOURCE_MASKS)
    with pytest.raises(ParameterError):
        h.check(lib.gccnmf_ll_export(one.h.h, ctypes.byref(one.cfg), one.state.data_ptr(), one.state_bytes, 1, ll.EXPORT_SOURCE_VALUES,
                                     one.state.data_ptr(), one.stream.cuda_stream))


def test_stream_signals_returns_one_array_per_source():
    p = _setup(D=32)
    sig = [_moving(40 * p['hop'], seed=3), _moving(33 * p['hop'] + 5, seed=4)]
    outs = ll.streamSignals(sig, p['W'], p['E'], p['win'], p['syn'], p['hop'], hopsPerCall=4, numSources=3)
    assert [o.shape for o in outs] == [(3, 2, s.shape[1]) for s in sig]
    single = ll.streamSignals(sig, p['W'], p['E'], p['win'], p['syn'], p['hop'], hopsPerCall=4, targetTDOAEpsilon=p['D'] + 1.0)
    for o, s in zip(outs, single):
        assert _sum_bar(o.sum(axis=0), s)
