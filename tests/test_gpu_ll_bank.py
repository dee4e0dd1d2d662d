"""GPU: a bank of steering tables in the low-latency engine (LowLatencyEngine(expJOmegaTau=[...]), gccnmf_llbank_*).  Bit for bit,
NaN-equal, a stream on table j against a plain engine built with that table alone:
  - a one-entry bank against ll, llsep and llhist, across synthesis modes, inference, P and Lh;
  - 8 spacings spread unsorted over 37 streams, hops per call 1 and 3, mixed schedules, graphs and kernel-by-kernel;
  - 1056 streams over 64 entries;
  - assign and load_steering between graph launches, against a plain stream moved by an llhist record onto the new table;
  - the gated float64 fallback on mono input;
  - records between banks (permuted and duplicated entries, another S, the lowest matching entry, refusals, a file)."""
import numpy as np
import pytest

from gcc_nmf_b200 import lowlatency as ll
from gcc_nmf_b200 import records

pytestmark = pytest.mark.gpu

SR = 16000
SPACINGS = [0.05, 0.1, 0.2, 0.3, 0.45, 0.6, 0.8, 1.0]


def _setup(N=256, m=32, hop=32, D=16, K=64, seed=0):
    from gcc_nmf_b200 import gccNMFFunctions as fn
    from gcc_nmf_b200.online import getAsymmetricAnalysisWindow, getAsymmetricSynthesisWindow
    F = N // 2 + 1
    rng = np.random.RandomState(seed)
    W = (rng.random_sample((F, K)) + 0.01).astype(np.float32)
    E = [fn.getExpJOmegaTau(fn.getFrequenciesInHz(SR, F), fn.getTDOAsInSeconds(d, D)) for d in SPACINGS]
    return dict(N=N, hop=hop, D=D, K=K, W=W, E=E, win=getAsymmetricAnalysisWindow(N, m, 0), syn=getAsymmetricSynthesisWindow(N, m, 0))


def _audio(S, hops, hop, seed=1, mono=False):
    """S different stereo streams: two delayed sources per stream, the second entering half way (mono: both channels equal)."""
    rng = np.random.RandomState(seed)
    n = hops * hop
    x = np.zeros((S, 2, n))
    for s in range(S):
        for i, d in enumerate((s % 7 - 3, 3 - s % 5)):
            v = rng.standard_normal(n + 16)
            part = np.stack([v[8:8 + n], v[8 - d:8 - d + n]])
            part[:, :i * n // 2] = 0
            x[s] += part
    if mono:
        x[:, 1] = x[:, 0]
    return (x / np.abs(x).max()).astype(np.float32)


def _engine(p, S, E, C=1, P=0, synthesis='lowlatency', inference=0, Lh=0):
    return ll.LowLatencyEngine(p['W'], E, p['win'], p['syn'], p['hop'], numStreams=S, hopsPerCall=C, synthesis=synthesis, numSources=P,
                               numInferenceIterations=inference, targetTDOAEpsilon=2.5, historyLength=Lh)


def _calls(eng, x, h0, h1, use_graph=True, schedule=None):
    out, h, k = [], h0, 0
    while h < h1:
        c = min(schedule[k % len(schedule)] if schedule else eng.C, h1 - h)
        out.append(eng.process(x[:, :, h * eng.hop:(h + c) * eng.hop], use_graph=use_graph))
        h += c
        k += 1
    return np.concatenate(out, axis=-1)


def _eq(a, b):
    return np.array_equal(a, b, equal_nan=True)


def _column_items(eng):
    """Per-column export items of the last call: (name, array with the column last)."""
    items = [('X', eng.export(ll.EXPORT_X)), ('coherence', eng.export(ll.EXPORT_COHERENCE)), ('angular', eng.export(ll.EXPORT_ANGULAR)),
             ('accmax', eng.export(ll.EXPORT_ACC_MAX)), ('valid', eng.export(ll.EXPORT_VALID))]
    if eng.P:
        items += [('targets', eng.export(ll.EXPORT_SOURCE_TARGETS).T), ('values', eng.export(ll.EXPORT_SOURCE_VALUES)),
                  ('masks', eng.export(ll.EXPORT_SOURCE_MASKS)), ('wiener', eng.export(ll.EXPORT_SOURCE_WIENER)),
                  ('Y', eng.export(ll.EXPORT_SOURCE_Y))]
    else:
        items += [('targets', eng.export(ll.EXPORT_TARGETS)), ('argmax', eng.export(ll.EXPORT_ARGMAX)), ('masks', eng.export(ll.EXPORT_MASKS)),
                  ('wiener', eng.export(ll.EXPORT_WIENER)), ('Y', eng.export(ll.EXPORT_Y))]
    if eng.inference:
        H = eng.export(ll.EXPORT_H)
        T = H.shape[1] // 2
        items.append(('H', np.stack([H[:, :T], H[:, T:]])))
    if eng.Lh:
        items.append(('means', eng.export(ll.EXPORT_WINDOW_MEANS)))
    return items


def _stream_items(eng):
    items = [('carry', eng.export(ll.EXPORT_CARRY))]
    if eng.P:
        items += [('carried', eng.export(ll.EXPORT_CARRIED_TARGETS)), ('status', eng.export(ll.EXPORT_STREAM_STATUS))]
    if eng.Lh:
        items += [('ring', eng.export(ll.EXPORT_HISTORY)), ('index', eng.export(ll.EXPORT_HISTORY_INDEX))]
    return items


def _check_streams(bank, plain, streams, hops):
    """Streams `streams` of `bank` against streams 0 .. len - 1 of `plain`, over the last call of `hops` hops each."""
    cols_b = np.concatenate([np.arange(s * hops, (s + 1) * hops) for s in streams])
    cols_p = np.arange(len(streams) * hops)
    for (name, a), (_, b) in zip(_column_items(bank), _column_items(plain)):
        assert _eq(a[..., cols_b], b[..., cols_p]), name
    for (name, a), (_, b) in zip(_stream_items(bank), _stream_items(plain)):
        assert _eq(a[streams], b), name


# ---------------------------------------------------------------------------------------------- 1. one entry is the plain engine
ONE = [('lowlatency', 0, 0, 0), ('online', 5, 0, 64), ('windowed', 0, 2, 0), ('lowlatency', 5, 2, 64), ('online', 0, 4, 64),
       ('windowed', 5, 4, 0), ('windowed', 0, 0, 64), ('online', 5, 4, 0)]


@pytest.mark.parametrize('synthesis,inference,P,Lh', ONE, ids=['-'.join(map(str, c)) for c in ONE])
def test_one_entry_is_the_plain_engine(synthesis, inference, P, Lh):
    p = _setup()
    S, hops = 5, 48
    x = _audio(S, hops, p['hop'])
    bank = _engine(p, S, [p['E'][2]], 3, P, synthesis, inference, Lh)
    plain = _engine(p, S, p['E'][2], 3, P, synthesis, inference, Lh)
    for e in (bank, plain):
        if Lh:
            e.set_localization(None, [0, 1, 7, 64, 20])
    assert _eq(_calls(bank, x, 0, hops), _calls(plain, x, 0, hops))
    for (name, a), (_, b) in zip(_column_items(bank) + _stream_items(bank), _column_items(plain) + _stream_items(plain)):
        assert _eq(a, b), name
    assert _eq(bank.export(ll.EXPORT_ASSIGNMENT), np.zeros(S, np.int32))
    if not P:
        assert _eq(bank.export(ll.EXPORT_REFINED), plain.export(ll.EXPORT_REFINED))


# ---------------------------------------------------------------------------------------------- 2. spread spacings
# D 32 and 128: the tensor-core argmax over bank-built planes and its refinement over each column's table
SPREAD = [(1, True, None, 0, 0, 16), (3, True, None, 0, 0, 16), (3, False, [1, 3, 2], 0, 0, 16), (1, False, None, 4, 0, 16),
          (3, True, [2, 1], 4, 64, 16), (1, True, None, 0, 64, 16), (3, True, [2, 1], 0, 0, 32), (1, False, None, 0, 0, 128)]


@pytest.mark.parametrize('C,graph,schedule,P,Lh,D', SPREAD, ids=['-'.join(map(str, c[:5])) + ('-D%d' % c[5] if c[5] != 16 else '') for c in SPREAD])
def test_spread_entries_equal_plain_engines(C, graph, schedule, P, Lh, D):
    p = _setup(D=D)
    S, hops = 37, 40
    x = _audio(S, hops, p['hop'])
    entries = np.random.RandomState(5).permutation(np.arange(S) % 8)
    bank = _engine(p, S, p['E'], C, P, Lh=Lh)
    bank.assign_steering(None, entries)
    if Lh:
        bank.set_localization(None, np.arange(S) % 9)
    out = _calls(bank, x, 0, hops, graph, schedule)
    assert _eq(bank.export(ll.EXPORT_ASSIGNMENT), entries)
    last = bank.last_hops
    for j in range(8):
        streams = np.flatnonzero(entries == j)
        plain = _engine(p, len(streams), p['E'][j], C, P, Lh=Lh)
        if Lh:
            plain.set_localization(None, streams % 9)
        ref = _calls(plain, x[streams], 0, hops, graph, schedule)
        assert _eq(out[streams], ref), j
        assert plain.last_hops == last
        _check_streams(bank, plain, streams, last)


def test_1056_streams_over_64_entries():
    from gcc_nmf_b200 import gccNMFFunctions as fn
    p = _setup()
    F = p['N'] // 2 + 1
    E = [fn.getExpJOmegaTau(fn.getFrequenciesInHz(SR, F), fn.getTDOAsInSeconds(0.03 + 0.015 * j, p['D'])) for j in range(64)]
    S, hops = 1056, 12
    x = _audio(S, hops, p['hop'])
    entries = np.random.RandomState(7).randint(0, 64, S)
    entries[:64] = np.arange(64)
    bank = _engine(p, S, E)
    bank.assign_steering(None, entries)
    out = _calls(bank, x, 0, hops)
    for j in (0, 17, 40, 63):
        streams = np.flatnonzero(entries == j)
        plain = _engine(p, len(streams), E[j])
        assert _eq(out[streams], _calls(plain, x[streams], 0, hops)), j
        _check_streams(bank, plain, streams, 1)


# ---------------------------------------------------------------------------------------------- 3. switching between launches
@pytest.mark.parametrize('switch', [0, 1, 8, 9])          # Q = ceil(256 / 32) = 8
@pytest.mark.parametrize('how', ['assign', 'load'])
@pytest.mark.parametrize('P,Lh', [(0, 0), (2, 16)])
def test_switching_between_graph_launches(switch, how, P, Lh):
    """Stream 1 moves from table a = 1 to table b = 6 after `switch` hops (by assign, or by loading E_b over its entry).  The
    reference: a plain stream on E_a up to the switch, moved by an llhist record (which names no table) onto a plain engine on E_b."""
    p = _setup()
    S, hops, a, b = 3, 30, 1, 6
    x = _audio(S, hops, p['hop'])
    bank = _engine(p, S, p['E'], 1, P, Lh=Lh)
    bank.assign_steering(None, [0, a, 3])
    if Lh:
        bank.set_localization(None, 5)
    first = _calls(bank, x, 0, switch) if switch else None
    if how == 'assign':
        bank.assign_steering(1, b)
    else:
        bank.load_steering(a, p['E'][b])
    rest = _calls(bank, x, switch, hops)
    got = np.concatenate([first, rest], axis=-1) if switch else rest
    ref_a = _engine(p, 1, p['E'][a], 1, P, Lh=max(Lh, 1))
    ref_b = _engine(p, 1, p['E'][b], 1, P, Lh=max(Lh, 1))
    for e in (ref_a, ref_b):
        e.set_localization(None, 5 if Lh else 0)
    r0 = _calls(ref_a, x[1:2], 0, switch) if switch else None
    ref_b.load_streams([0], ref_a.save_streams([0]))
    r1 = _calls(ref_b, x[1:2], switch, hops)
    want = np.concatenate([r0, r1], axis=-1) if switch else r1
    assert _eq(got[1:2], want)
    if not Lh:                       # the reference's ring was a window-0 ring of one frame: compare the rest of the column items
        _check_streams(bank, ref_b, [1], 1)


# ---------------------------------------------------------------------------------------------- 4. the gated float64 fallback
def test_mono_input_takes_the_float64_fallback():
    """K T = 512 x 256 decisions, more than half of them near-ties: past the refinement list's 65536 entries."""
    p = _setup(K=512)
    S, hops = 256, 3
    x = _audio(S, hops, p['hop'], mono=True)
    entries = np.arange(S) % 8
    bank = _engine(p, S, p['E'])
    bank.assign_steering(None, entries)
    out = _calls(bank, x, 0, hops)
    assert bank.export(ll.EXPORT_STATUS)[0] == 1
    assert bank.export(ll.EXPORT_REFINED)[0] > int(bank.h.lib.gccnmf_tdoa_argmax_refine_capacity(p['K'], S))
    for j in range(8):
        streams = np.flatnonzero(entries == j)
        plain = _engine(p, len(streams), p['E'][j])
        assert _eq(out[streams], _calls(plain, x[streams], 0, hops)), j
        assert _eq(bank.export(ll.EXPORT_ARGMAX)[:, streams], plain.export(ll.EXPORT_ARGMAX)), j


# ---------------------------------------------------------------------------------------------- 5. records
def test_records_between_banks(tmp_path):
    p = _setup()
    S, hops, cut = 6, 30, 17
    x = _audio(S, hops, p['hop'])
    src = _engine(p, S, p['E'][:4], 1, 2, Lh=8)
    src.assign_steering(None, [0, 1, 2, 3, 1, 2])
    src.set_localization(None, 3)
    ref = _calls(src, x, 0, hops)
    # destination: another S, the tables permuted with entry 1 twice (entries 0 and 4 hold E_1)
    src2 = _engine(p, S, p['E'][:4], 1, 2, Lh=8)
    src2.assign_steering(None, [0, 1, 2, 3, 1, 2])
    src2.set_localization(None, 3)
    _calls(src2, x, 0, cut)
    rec = src2.save_streams([1, 2, 3, 0])
    assert [rec.header(i).steering_digest for i in range(4)] == [records.content_digest(p['E'][j]) for j in (1, 2, 3, 0)]
    dst = _engine(p, 9, [p['E'][1], p['E'][3], p['E'][0], p['E'][2], p['E'][1]], 1, 2, Lh=8)
    dst.load_streams([5, 6, 7, 8], rec)
    assert _eq(dst._assign[5:], [0, 3, 1, 2])                                # E_1 -> the lowest of entries 0 and 4
    out = []
    for h in range(cut, hops):
        xi = np.zeros((9, 2, p['hop']), np.float32)
        xi[5:] = x[[1, 2, 3, 0], :, h * p['hop']:(h + 1) * p['hop']]
        out.append(dst.process(xi))
    y = np.concatenate(out, axis=-1)
    assert _eq(dst.export(ll.EXPORT_ASSIGNMENT)[5:], [0, 3, 1, 2])
    assert _eq(y[5:], ref[[1, 2, 3, 0], ..., cut * p['hop']:])
    # a file onto a second engine
    rec.save(str(tmp_path / 'r.npz'))
    dst2 = _engine(p, 4, [p['E'][3], p['E'][2], p['E'][1], p['E'][0]], 1, 2, Lh=8)
    dst2.load_streams([0, 1, 2, 3], records.load(str(tmp_path / 'r.npz')))
    y2 = _calls(dst2, x[[1, 2, 3, 0]], cut, hops)
    assert _eq(dst2.export(ll.EXPORT_ASSIGNMENT), [2, 1, 0, 3])
    assert _eq(y2, ref[[1, 2, 3, 0], ..., cut * p['hop']:])


def test_refused_bank_records_change_nothing():
    p = _setup()
    S = 4
    x = _audio(S, 12, p['hop'])
    src = _engine(p, S, p['E'][:3])
    src.assign_steering(None, [0, 1, 2, 1])
    _calls(src, x, 0, 12)
    rec = src.save_streams([0, 1, 2, 3])
    dst = _engine(p, S, [p['E'][0], p['E'][1]])                      # no entry holds E_2
    _calls(dst, x, 0, 5)
    before = dst.state.cpu().numpy().copy()
    launches = dst.h.launches
    with pytest.raises(Exception, match='steering entry'):
        dst.load_streams([0, 1, 2, 3], rec)
    assert dst.h.launches == launches
    assert np.array_equal(dst.state.cpu().numpy(), before)
    W2 = p['W'].copy()
    W2[3, 5] *= 2
    dw = ll.LowLatencyEngine(W2, p['E'][:3], p['win'], p['syn'], p['hop'], numStreams=S, targetTDOAEpsilon=2.5)
    before = dw.state.cpu().numpy().copy()
    launches = dw.h.launches
    with pytest.raises(Exception, match='dictionary'):
        dw.load_streams([0, 1, 2, 3], rec)
    assert dw.h.launches == launches
    assert np.array_equal(dw.state.cpu().numpy(), before)
    # through the C entry, past the host checks: the device digests refuse and the state stays byte-identical
    dst._dict_digest = rec.header(0).dictionary_digest
    dst._steer_digests = [rec.header(2).steering_digest, rec.header(1).steering_digest]
    before = dst.state.cpu().numpy().copy()
    with pytest.raises(Exception):
        dst.load_streams([0, 1, 2, 3], rec)
    assert np.array_equal(dst.state.cpu().numpy(), before)
    # a bank record is not a plain one, and the other way round
    plain = _engine(p, S, p['E'][0])
    with pytest.raises(ValueError):
        plain.load_streams([0], src.save_streams([0]))
    with pytest.raises(ValueError):
        src.load_streams([0], plain.save_streams([0]))


def test_bank_refusals_launch_nothing():
    p = _setup()
    eng = _engine(p, 4, p['E'][:3])
    launches = eng.h.launches
    for bad in ([3], [-1]):
        with pytest.raises(ValueError):
            eng.assign_steering([0], bad)
    with pytest.raises(ValueError):
        eng.load_steering(3, p['E'][0])
    import ctypes
    e = (ctypes.c_int32 * 1)(3)
    assert eng.h.lib.gccnmf_llbank_assign(eng.h.h, ctypes.byref(eng.cfg), 0, 0, 3, eng.state.data_ptr(), eng.state_bytes, 0, 1, e,
                                          eng.stream.cuda_stream) != 0
    assert eng.h.lib.gccnmf_llbank_load_steering(eng.h.h, ctypes.byref(eng.cfg), 0, 0, 3, eng.state.data_ptr(), eng.state_bytes, 3,
                                                 eng._const[1].data_ptr(), eng.stream.cuda_stream) != 0
    assert eng.h.lib.gccnmf_llbank_state_bytes(ctypes.byref(eng.cfg), 0, 0, 65) == 0
    assert eng.h.launches == launches


def test_reset_puts_streams_on_entry_zero():
    p = _setup()
    S, hops = 5, 20
    x = _audio(S, hops, p['hop'])
    bank = _engine(p, S, p['E'][:5])
    bank.assign_steering(None, [4, 3, 2, 1, 0])
    _calls(bank, x, 0, 7)
    bank.reset([1, 3])
    assert _eq(bank._assign, [4, 0, 2, 0, 0])
    out = _calls(bank, x, 0, hops)
    assert _eq(bank.export(ll.EXPORT_ASSIGNMENT), [4, 0, 2, 0, 0])
    plain = _engine(p, 2, p['E'][0])
    assert _eq(out[[1, 3]], _calls(plain, x[[1, 3]], 0, hops))


def test_stream_signals_takes_steering_entries():
    p = _setup()
    sig = [_audio(1, 20, p['hop'], seed=s)[0] for s in range(3)]
    got = ll.streamSignals(sig, p['W'], p['E'][:3], p['win'], p['syn'], p['hop'], steeringEntries=[2, 0, 1])
    for s, j in zip(range(3), (2, 0, 1)):
        want = ll.streamSignals([sig[s]], p['W'], p['E'][j], p['win'], p['syn'], p['hop'])[0]
        assert _eq(got[s], want)
