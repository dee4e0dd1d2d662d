"""GPU: localisation over a sliding window of each stream's recent frames (LowLatencyEngine(historyLength=Lh), set_localization,
gccnmf_llhist_*).  Bit for bit, NaN-equal:
  - window 0 of an Lh > 0 engine, and the whole Lh = 0 family, are the plain engines;
  - the ring, its index, the window means and the decisions equal the host model (oracle/ll_window.py) fed the device's angular
    spectrum, and the outputs equal a plain engine driven by the model's targets as overrides;
  - a talker who moves and a stream that opens with digital silence: the running maximum stays, the window follows;
  - streams, schedules, graphs and input scale do not change a stream's bytes; records move a stream with its ring;
  - refusals launch nothing."""
import ctypes

import numpy as np
import pytest

from gcc_nmf_b200 import _lib
from gcc_nmf_b200 import lowlatency as ll
from oracle import ll_window as lw

pytestmark = pytest.mark.gpu

SR = 16000


def _setup(N=256, m=32, hop=32, D=16, K=64, micSep=0.1, seed=0):
    from gcc_nmf_b200 import gccNMFFunctions as fn
    from gcc_nmf_b200.online import getAsymmetricAnalysisWindow, getAsymmetricSynthesisWindow
    F = N // 2 + 1
    rng = np.random.RandomState(seed)
    W = (rng.random_sample((F, K)) + 0.01).astype(np.float32)
    E = fn.getExpJOmegaTau(fn.getFrequenciesInHz(SR, F), fn.getTDOAsInSeconds(micSep, D))
    return dict(N=N, hop=hop, D=D, K=K, W=W, E=E, win=getAsymmetricAnalysisWindow(N, m, 0), syn=getAsymmetricSynthesisWindow(N, m, 0))


def _audio(S, hops, hop, seed=1, silence=True):
    """S different stereo streams: a delayed source per stream plus a second one entering half way; with `silence`, stream s is
    digitally silent over hops [10 + 3 s, 10 + 3 s + 12) (NaN angular spectra, which the window must get over)."""
    rng = np.random.RandomState(seed)
    n = hops * hop
    x = np.zeros((S, 2, n))
    for s in range(S):
        for i, d in enumerate((s % 7 - 3, 3 - s % 5)):
            v = rng.standard_normal(n + 16)
            part = np.stack([v[8:8 + n], v[8 - d:8 - d + n]])
            part[:, :i * n // 2] = 0
            x[s] += part
        if silence:
            a = (10 + 3 * (s % 11)) * hop
            x[s, :, a:a + 12 * hop] = 0
    return (x / np.abs(x).max()).astype(np.float32)


def _engine(p, S, C=1, P=0, synthesis='lowlatency', inference=0, Lh=0, cls=ll.LowLatencyEngine):
    return cls(p['W'], p['E'], p['win'], p['syn'], p['hop'], numStreams=S, hopsPerCall=C, synthesis=synthesis, numSources=P,
               numInferenceIterations=inference, targetTDOAEpsilon=2.5, historyLength=Lh)


class _HistZero(ll.LowLatencyEngine):
    """An engine on the gccnmf_llhist_* entries with history_length 0."""
    @property
    def _p(self):
        return (self.P, 0)

    def _fn(self, name):
        return getattr(self.h.lib, 'gccnmf_llhist_' + name)

    def _rec(self, name):
        fn = getattr(self.h.lib, 'gccnmf_llhist_' + name)
        if name.endswith('_bytes'):
            return lambda *a: fn(ctypes.byref(self.cfg), self.P, 0, *a)
        return lambda *a: fn(self.h.h, ctypes.byref(self.cfg), self.P, 0, *a)


def _calls(eng, x, h0, h1, use_graph=True, schedule=None, each=None):
    """Hops [h0, h1) of x through eng, in calls of eng.C hops (or the sizes of `schedule`, cycled); each(eng, h, c) after a call."""
    out, h, k = [], h0, 0
    while h < h1:
        c = min(schedule[k % len(schedule)] if schedule else eng.C, h1 - h)
        out.append(eng.process(x[:, :, h * eng.hop:(h + c) * eng.hop], use_graph=use_graph))
        if each:
            each(eng, h, c)
        h += c
        k += 1
    return np.concatenate(out, axis=-1) if out else None


def _eq(a, b):
    return np.array_equal(a, b, equal_nan=True)


def _decisions(eng):
    if eng.P:
        return [eng.export(ll.EXPORT_SOURCE_TARGETS), eng.export(ll.EXPORT_CARRIED_TARGETS), eng.export(ll.EXPORT_STREAM_STATUS),
                eng.export(ll.EXPORT_CALL_STATUS), eng.export(ll.EXPORT_CARRY)]
    return [eng.export(ll.EXPORT_TARGETS), eng.export(ll.EXPORT_CARRY), eng.export(ll.EXPORT_STATUS)]


# ---------------------------------------------------------------------------------------------- 1. nothing changes at w = 0
ZERO = [('lowlatency', 0, 0), ('online', 0, 5), ('windowed', 0, 0), ('windowed', 2, 0), ('lowlatency', 2, 5), ('online', 2, 0),
        ('online', 8, 0), ('windowed', 8, 5), ('lowlatency', 8, 0)]


@pytest.mark.parametrize('synthesis,P,inference', ZERO, ids=['-'.join(map(str, c)) for c in ZERO])
def test_window_zero_is_the_plain_engine(synthesis, P, inference):
    p = _setup()
    S, hops = 3, 60
    x = _audio(S, hops, p['hop'])
    engines = [_engine(p, S, 3, P, synthesis, inference), _engine(p, S, 3, P, synthesis, inference, Lh=64),
               _engine(p, S, 3, P, synthesis, inference, cls=_HistZero)]
    assert engines[2].state_bytes == engines[0].state_bytes
    for e in engines:
        if P:
            e.set_targets([2], [[-1] * (P - 1) + [5]])
        else:
            e.set_params([2], targetOverride=4)
    engines[1].set_localization([0], 6)        # a neighbour on a window changes nothing for the others
    engines[1].set_localization([0], 0)
    got = [[], [], []]
    for h in range(0, hops, 3):
        for i, e in enumerate(engines):
            before = e.h.launches
            got[i].append([e.process(x[:, :, h * p['hop']:(h + 3) * p['hop']], use_graph=(h // 3) % 2 == 0)] + _decisions(e))
            got[i][-1].append(e.h.launches - before)
    for i in (1, 2):
        for a, b in zip(got[0], got[i]):
            assert all(_eq(u, v) for u, v in zip(a[:-1], b[:-1]))
    # the Lh = 0 family enqueues exactly the plain launches; Lh > 0 the same number (its targets kernel replaces the plain one)
    assert [g[-1] for g in got[2]] == [g[-1] for g in got[0]] == [g[-1] for g in got[1]]


# ---------------------------------------------------------------------------------------------- 2. the window rule against the model
RULE = [(5, 0, (1, 5, 0, 3)), (64, 0, (1, 6, 64, 0)), (1024, 0, (1, 6, 64, 1024)), (5, 2, (1, 5, 0, 2)), (64, 2, (1, 6, 64, 0)),
        (1024, 2, (6, 64, 1024, 1)), (64, 8, (1, 6, 64, 0)), (1024, 8, (1, 64, 1024, 6))]


@pytest.mark.parametrize('Lh,P,windows', RULE, ids=['%d-%d' % c[:2] for c in RULE])
def test_window_rule_equals_model(Lh, P, windows):
    """The ring wraps many times (hops > 2 Lh + 200); every call's means and decisions, and the ring and index, equal the model."""
    p = _setup(D=32 if P == 8 else 16)
    S, C = len(windows), 8
    hops = 2 * Lh + 240
    x = _audio(S, hops, p['hop'], seed=Lh + P)
    eng = _engine(p, S, C, P, Lh=Lh)
    eng.set_localization(range(S), list(windows))
    if not P:
        eng.set_params([S - 1], targetOverride=2)
    models = [lw.WindowTargets(eng.D, Lh, P) for _ in range(S)]
    for s, m in enumerate(models):
        m.window = windows[s]
    models[S - 1].override = 2 if not P else models[S - 1].override
    nan_frames = []

    def check(e, h, c):
        ang, valid, means = e.export(ll.EXPORT_ANGULAR), e.export(ll.EXPORT_VALID), e.export(ll.EXPORT_WINDOW_MEANS)
        nan_frames.append(int(np.isnan(ang[0, valid.astype(bool)]).sum()))
        tg = e.export(ll.EXPORT_SOURCE_TARGETS if P else ll.EXPORT_TARGETS)
        for s, m in enumerate(models):
            for i in range(c):
                t = s * c + i
                mean, want = m.frame(ang[:, t], bool(valid[t]))
                assert _eq(means[:, t], mean), (h, s, i)
                assert np.array_equal(tg[t], want), (h, s, i, tg[t], want)
        if P:
            assert np.array_equal(e.export(ll.EXPORT_CARRIED_TARGETS), np.stack([m.targets for m in models]))
            assert np.array_equal(e.export(ll.EXPORT_STREAM_STATUS), [m.status for m in models])
    _calls(eng, x, 0, hops, each=check)
    assert _eq(eng.export(ll.EXPORT_HISTORY), np.stack([m.ring for m in models]))
    assert np.array_equal(eng.export(ll.EXPORT_HISTORY_INDEX), [m.index for m in models])
    assert np.array_equal(eng.export(ll.EXPORT_WINDOWS), list(windows))
    assert _eq(eng.export(ll.EXPORT_CARRY), np.stack([m.carry for m in models]))
    assert sum(nan_frames) > 0                                              # silent frames took part


# ---------------------------------------------------------------------------------------------- 3. outputs are the teacher-forced plain engine
@pytest.mark.parametrize('P,synthesis,inference', [(0, 'windowed', 0), (0, 'online', 5), (2, 'lowlatency', 0), (8, 'windowed', 5)])
def test_outputs_equal_teacher_forced_plain_engine(P, synthesis, inference):
    p = _setup(D=32 if P == 8 else 16)
    S, Lh, hops = 2, 64, 140
    x = _audio(S, hops, p['hop'], seed=7)
    win = _engine(p, S, 1, P, synthesis, inference, Lh=Lh)
    win.set_localization(range(S), [6, 64])
    plain = _engine(p, S, 1, P, synthesis, inference)
    models = [lw.WindowTargets(win.D, Lh, P) for _ in range(S)]
    models[0].window, models[1].window = 6, 64
    for h in range(hops):
        xs = x[:, :, h * p['hop']:(h + 1) * p['hop']]
        y = win.process(xs)
        ang, valid = win.export(ll.EXPORT_ANGULAR), win.export(ll.EXPORT_VALID)
        want = [m.frame(ang[:, s], bool(valid[s]))[1] for s, m in enumerate(models)]
        if P:
            plain.set_targets(range(S), np.stack(want))
        else:
            plain.set_params(range(S), targetOverride=[int(t) for t in want])
        assert _eq(plain.process(xs), y), h


# ---------------------------------------------------------------------------------------------- 4. the two failures this fixes
def _moving_and_silent(hop, half=250, delays=(-3, 2), seed=5):
    """Stream 0: a source whose inter-channel delay jumps from delays[0] to delays[1] after `half` hops, plus independent noise on
    each channel in the second half.  Stream 1: 0.5 s (`half` hops) of digital silence, then the source at delays[0]."""
    rng = np.random.RandomState(seed)
    n = 2 * half * hop
    v = rng.standard_normal(n + 16)
    x = np.zeros((2, 2, n))
    a, b = delays
    x[0, 0] = v[8:8 + n]
    x[0, 1, :half * hop] = v[8 - a:8 - a + half * hop]
    x[0, 1, half * hop:] = v[8 - b + half * hop:8 - b + n]
    x[0, :, half * hop:] += 0.5 * rng.standard_normal((2, n - half * hop))
    x[1, 0, half * hop:] = v[8 + half * hop:8 + n]
    x[1, 1, half * hop:] = v[8 - a + half * hop:8 - a + n]
    return (x / np.abs(x).max()).astype(np.float32)


def test_window_follows_a_moving_talker_and_recovers_from_silence():
    p = _setup()
    half, hop = 250, p['hop']
    x2 = _moving_and_silent(hop, half)
    x = np.concatenate([x2, x2])                     # streams 0, 1 on the running maximum; 2, 3 on a 64-frame window
    eng = _engine(p, 4, 8, Lh=64)
    eng.set_localization([2, 3], 64)
    targets = []
    _calls(eng, x, 0, 2 * half, each=lambda e, h, c: targets.append(e.export(ll.EXPORT_TARGETS).reshape(4, c)))
    tg = np.concatenate(targets, axis=1)             # (4, hops): target of each stream's frame ending in hop h
    # the direction of each half on its own, from a running maximum started fresh there
    ref = _engine(p, 2, 8)
    seg = np.stack([x2[0, :, :half * hop], x2[0, :, half * hop:]])
    r = []
    _calls(ref, seg, 0, half, each=lambda e, h, c: r.append(e.export(ll.EXPORT_TARGETS).reshape(2, c)))
    tau_a, tau_b = [int(t) for t in np.concatenate(r, axis=1)[:, -1]]
    assert tau_a != tau_b and tau_a != 0
    # the running maximum never forgets: it stays on tau_a; after the silence it stays on TDOA 0
    assert (tg[0, half:] == tau_a).all()
    assert (tg[1, half:] == 0).all()
    # the window reaches tau_b within 64 frames of the jump, and leaves TDOA 0 within 64 frames of the first sound
    assert (tg[2, half:half + 64] == tau_b).any() and tg[2, -1] == tau_b
    assert (tg[3, half:half + 64] != 0).any() and tg[3, -1] == tau_a


# ---------------------------------------------------------------------------------------------- 5. streams and schedules
def test_heterogeneous_streams_equal_one_stream_engines():
    p = _setup()
    Lh, hops, windows = 100, 220, [0, 1, 6, 64, 100]
    x = _audio(5, hops, p['hop'], seed=11)
    big = _engine(p, 5, 3, Lh=Lh)
    big.set_localization(range(5), windows)
    singles = [_engine(p, 1, 1, Lh=Lh) for _ in range(5)]
    for s, e in enumerate(singles):
        e.set_localization([0], windows[s])
    # hop -> (stream, what happens to it); reset sets the window back to 0, so stream 2 is put on its window again
    events = {60: (1, lambda e, i: e.set_active([i], False)), 90: (1, lambda e, i: e.set_active([i], True)),
              111: (2, lambda e, i: (e.reset([i]), e.set_localization([i], 6))), 120: (0, lambda e, i: e.set_localization([i], 64)),
              180: (0, lambda e, i: e.set_localization([i], 0))}
    got, want = [], [[] for _ in range(5)]
    for h in range(0, hops, 3):
        if h in events:
            s, ev = events[h]
            ev(big, s)
            ev(singles[s], 0)
        xs = x[:, :, h * p['hop']:(h + 3) * p['hop']]
        got.append(big.process(xs))
        for s in range(5):
            want[s].append(_calls(singles[s], xs[s:s + 1], 0, xs.shape[2] // p['hop'], use_graph=False))
    y = np.concatenate(got, axis=-1)
    for s in range(5):
        assert _eq(y[s], np.concatenate(want[s], axis=-1)[0]), s
        assert _eq(big.export(ll.EXPORT_HISTORY)[s], singles[s].export(ll.EXPORT_HISTORY)[0]), s


def test_stream_of_a_1056_stream_engine():
    p = _setup()
    S, Lh, hops = 1056, 64, 100
    x = _audio(S, hops, p['hop'], seed=13)
    big = _engine(p, S, 4, Lh=Lh)
    big.set_localization(range(S), [(0, 1, 6, 64)[s % 4] for s in range(S)])
    y = _calls(big, x, 0, hops)
    for s in (0, 517, 1055):
        one = _engine(p, 1, 4, Lh=Lh)
        one.set_localization([0], (0, 1, 6, 64)[s % 4])
        assert np.array_equal(_calls(one, x[s:s + 1], 0, hops), y[s:s + 1]), s


@pytest.mark.parametrize('P', [0, 2])
def test_schedules_graphs_and_scale(P):
    p = _setup()
    S, Lh, hops = 3, 64, 168
    x = _audio(S, hops, p['hop'], seed=17)
    runs = {}
    for key, C, schedule, use_graph, scale in [('c1', 1, None, True, 1.0), ('c3', 3, None, False, 1.0), ('c8', 8, None, True, 1.0),
                                               ('mix', 8, [1, 8, 3, 5, 2], True, 1.0), ('kernels', 8, None, False, 1.0),
                                               ('up', 8, None, True, 2.0 ** 20), ('down', 8, None, True, 2.0 ** -20)]:
        eng = _engine(p, S, C, P, Lh=Lh)
        eng.set_localization(range(S), [6, 64, 1])
        tg = []
        k = ll.EXPORT_SOURCE_TARGETS if P else ll.EXPORT_TARGETS
        y = _calls(eng, (x * scale).astype(np.float32), 0, hops, use_graph, schedule,
                   each=lambda e, h, c: tg.append(e.export(k).reshape((S, c) + ((P,) if P else ()))))
        runs[key] = (y, np.concatenate(tg, axis=1), eng.export(ll.EXPORT_HISTORY))
    for key in ('c3', 'c8', 'mix', 'kernels'):
        assert all(_eq(a, b) for a, b in zip(runs['c1'], runs[key])), key
    for key in ('up', 'down'):
        assert np.array_equal(runs[key][1], runs['c1'][1]), key


# ---------------------------------------------------------------------------------------------- 6. records
@pytest.mark.parametrize('P', [0, 2])
@pytest.mark.parametrize('at', [0, 1, 63, 64, 71])
def test_record_round_trip_equals_unmoved(P, at):
    """Saved from stream 5 of an 8-stream engine (graph, 3 hops per call), loaded into stream 0 of a 3-stream engine (kernel by
    kernel, 1 hop per call), run there, then saved back into stream 5: both stretches and the ring equal an unmoved engine."""
    p = _setup()
    Lh = 64
    mid = at + Lh + 7
    h1 = mid + Lh + 9
    x = _audio(8, h1, p['hop'], seed=23)
    wins = [64, 6, 0, 1, 64, 64, 6, 0]
    ref = _engine(p, 8, 1, P, 'windowed', Lh=Lh)
    ref.set_localization(range(8), wins)
    want = [_calls(ref, x, 0, mid)]
    mid_state = [ref.export(k)[5] for k in (ll.EXPORT_HISTORY, ll.EXPORT_HISTORY_INDEX, ll.EXPORT_WINDOWS)]
    want = np.concatenate(want + [_calls(ref, x, mid, h1)], axis=-1)
    want_ring = ref.export(ll.EXPORT_HISTORY)[5]
    big, small = _engine(p, 8, 3, P, 'windowed', Lh=Lh), _engine(p, 3, 1, P, 'windowed', Lh=Lh)
    big.set_localization(range(8), wins)
    small.set_localization(range(3), [0, 6, 1])               # slot 0 runs on the running maximum until the load
    y0 = _calls(big, x, 0, at, True)
    small.load_streams([0], big.save_streams([5]))
    y1 = _calls(small, x[[5, 6, 7]], at, mid, False)
    got_state = [small.export(k)[0] for k in (ll.EXPORT_HISTORY, ll.EXPORT_HISTORY_INDEX, ll.EXPORT_WINDOWS)]
    assert all(_eq(a, b) for a, b in zip(got_state, mid_state)) and got_state[2] == 64
    big.load_streams([5], small.save_streams([0]))
    y2 = _calls(big, x, mid, h1, True)
    hop = p['hop']
    if y0 is not None:
        assert np.array_equal(y0[5], want[5, ..., :at * hop])
    assert np.array_equal(y1[0], want[5, ..., at * hop:mid * hop])
    assert np.array_equal(y2[5], want[5, ..., mid * hop:])
    assert _eq(big.export(ll.EXPORT_HISTORY)[5], want_ring)
    assert big._window[5] == 64


@pytest.mark.parametrize('P', [0, 2, 8])
def test_history_zero_records_are_llrec_records(P):
    p = _setup(D=32 if P == 8 else 16)
    x = _audio(3, 30, p['hop'], seed=29)
    plain, zero = _engine(p, 3, 3, P), _engine(p, 3, 3, P, cls=_HistZero)
    _calls(plain, x, 0, 30)
    _calls(zero, x, 0, 30)
    for e in (plain, zero):        # the staging's gaps between 16-aligned regions are not written by the library: start them equal
        e._staging = e.torch.zeros(1 << 20, dtype=e.torch.uint8, device=e.h.device)
    a, b = plain.save_streams(), zero.save_streams()
    assert np.array_equal(a.data.numpy(), b.data.numpy())
    plain.load_streams([2, 0, 1], b)
    zero.load_streams([2, 0, 1], a)
    assert np.array_equal(plain.process(x[:, :, :3 * p['hop']]), zero.process(x[:, :, :3 * p['hop']]))


def test_refused_loads_launch_nothing():
    p = _setup()
    x = _audio(2, 20, p['hop'], seed=31)
    src = _engine(p, 2, 2, Lh=64)
    _calls(src, x, 0, 20)
    rec = src.save_streams([1])
    others = [_engine(p, 2, 2, Lh=32), _engine(p, 2, 2, 2, Lh=64), _engine(p, 2, 2, Lh=64, inference=5), _engine(p, 2, 2)]
    for dst in others:
        n = dst.h.launches
        with pytest.raises(_lib.ParameterError):
            dst.load_streams([0], rec)
        assert dst.h.launches == n
    dst = _engine(p, 2, 2, Lh=64)
    bad = src.save_streams([1])
    bad.data[0, 0] ^= 1                                        # magic
    n = dst.h.launches
    with pytest.raises(_lib.ParameterError):
        dst.load_streams([0], bad)
    assert dst.h.launches == n
    # through the C entry: a record of another history length is refused before anything is enqueued
    lib, other = dst.h.lib, others[0]
    ws = dst.torch.empty(1 << 20, dtype=dst.torch.uint8, device=dst.h.device)
    n = other.h.launches
    st = lib.gccnmf_llhist_load_streams(other.h.h, ctypes.byref(other.cfg), 0, 32, other.state.data_ptr(), other.state_bytes, 0, 1,
                                        rec.data[0].data_ptr(), other.record_bytes, ws.data_ptr(), ws.numel(), other.stream.cuda_stream)
    assert st != 0 and other.h.launches == n


# ---------------------------------------------------------------------------------------------- 7. refusals
def test_refusals_launch_nothing():
    p = _setup()
    eng = _engine(p, 3, 2, Lh=16)
    eng.process(_audio(3, 2, p['hop']))
    lib, cfg = eng.h.lib, ctypes.byref(eng.cfg)
    args = (eng.state.data_ptr(), eng.state_bytes)
    buf = eng.torch.zeros(1 << 16, dtype=eng.torch.uint8).pin_memory()
    zero = _HistZero(p['W'], p['E'], p['win'], p['syn'], p['hop'], numStreams=3, hopsPerCall=2)
    zero.process(_audio(3, 2, p['hop']))
    n = eng.h.launches
    w = (ctypes.c_int32 * 3)(0, 17, 1)
    assert lib.gccnmf_llhist_set_window(eng.h.h, cfg, 0, 16, *args, 0, 3, w, eng.stream.cuda_stream) != 0
    w = (ctypes.c_int32 * 1)(-1)
    assert lib.gccnmf_llhist_set_window(eng.h.h, cfg, 0, 16, *args, 0, 1, w, eng.stream.cuda_stream) != 0
    assert lib.gccnmf_llhist_set_window(eng.h.h, cfg, 0, 16, *args, 2, 2, w, eng.stream.cuda_stream) != 0
    for Lh in (-1, 1025):
        assert lib.gccnmf_llhist_process(eng.h.h, cfg, 0, Lh, *args, 1, None, None, eng.stream.cuda_stream) != 0
        assert lib.gccnmf_llhist_reset_streams(eng.h.h, cfg, 0, Lh, *args, 0, 1, eng.stream.cuda_stream) != 0
    for item in range(22, 26):
        assert lib.gccnmf_llhist_export(zero.h.h, ctypes.byref(zero.cfg), 0, 0, zero.state.data_ptr(), zero.state_bytes, 2, item,
                                        buf.data_ptr(), zero.stream.cuda_stream) != 0
    assert lib.gccnmf_llhist_set_window(zero.h.h, ctypes.byref(zero.cfg), 0, 0, zero.state.data_ptr(), zero.state_bytes, 0, 1,
                                        (ctypes.c_int32 * 1)(0), zero.stream.cuda_stream) != 0
    assert lib.gccnmf_llhist_set_targets(eng.h.h, cfg, 0, 16, *args, 0, 1, (ctypes.c_int32 * 2)(1, 2), eng.stream.cuda_stream) != 0
    with pytest.raises(ValueError):
        eng.set_localization([0], 17)
    assert eng.h.launches == n
