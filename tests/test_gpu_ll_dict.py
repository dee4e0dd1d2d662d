"""GPU: a bank of dictionaries in the low-latency engine (LowLatencyEngine(W=[...]), gccnmf_lldict_*).  Bit for bit, NaN-equal, a
stream on dictionary i and table j against a plain engine built with (W_i, E_j): outputs, the per-column export items on the stream's
columns and rows < K_i, and the fill of the rows past K_i.
  - a one-entry bank against llhist and llbank engines, every synthesis mode, inference 0 and 5, P 0, 2 and 4, Lh 0 and 64;
  - K_i in {24, 64, 100, 128, 256} plus a second K = 100 content, unsorted over 37 streams and 3 tables, D = 16 (SIMT), 32, 64 and 128
    (grouped tensor-core GEMM), hops per call 1 and 3, mixed schedules, graph and kernel-by-kernel runs of the same case.  K_i = 24
    and 100 make the plain engine take the float64 argmax while the bank takes the tensor path with refinement;
  - 1056 streams over 64 dictionaries and 4 tables;
  - every per-stream setting on 130 streams in one call, against the host mirror;
  - assign_dictionary and load_dictionary between launches of a kept graph;
  - the gated float64 fallback on mono input;
  - records: lldict <-> llbank, permuted and duplicated entries, the lowest matching entry, refusals that leave every stream as it
    was, a refused record after an accepted run, a file."""
import ctypes

import numpy as np
import pytest

from gcc_nmf_b200 import lowlatency as ll
from gcc_nmf_b200 import records
from gcc_nmf_b200._lib import ParameterError

pytestmark = pytest.mark.gpu

SR = 16000
SPACINGS = [0.1, 0.3, 0.8, 0.5]
ATOMS = [24, 64, 100, 128, 256, 100]      # the last: another content of K = 100


def _setup(D, atoms=ATOMS, N=256, m=32, hop=32, seed=0):
    from gcc_nmf_b200 import gccNMFFunctions as fn
    from gcc_nmf_b200.online import getAsymmetricAnalysisWindow, getAsymmetricSynthesisWindow
    F = N // 2 + 1
    rng = np.random.RandomState(seed)
    Ws = [(rng.random_sample((F, k)) + 0.01).astype(np.float32) for k in atoms]
    E = [fn.getExpJOmegaTau(fn.getFrequenciesInHz(SR, F), fn.getTDOAsInSeconds(d, D)) for d in SPACINGS]
    return dict(N=N, hop=hop, D=D, Ws=Ws, E=E, win=getAsymmetricAnalysisWindow(N, m, 0), syn=getAsymmetricSynthesisWindow(N, m, 0))


def _audio(S, hops, hop, seed=1, mono=False):
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


def _eq(a, b):
    assert a.shape == b.shape
    assert np.array_equal(a, b, equal_nan=True)


def _engine(p, W, E, S, **kw):
    kw.setdefault('targetTDOAEpsilon', 2.5)
    return ll.LowLatencyEngine(W, E, p['win'], p['syn'], p['hop'], numStreams=S, **kw)


def _run(eng, x, h0, h1, schedule, use_graph, after=None):
    """Calls over hops [h0, h1) with the hop counts of `schedule` in turn; after(eng, call) is called after each call."""
    out, h, k = [], h0, 0
    while h < h1:
        c = min(schedule[k % len(schedule)], h1 - h)
        out.append(eng.process(x[:, :, h * eng.hop:(h + c) * eng.hop], use_graph=use_graph))
        if after:
            after(eng, k)
        h += c
        k += 1
    return np.concatenate(out, axis=-1)


def _items(P, inference):
    if P:
        w = [ll.EXPORT_SOURCE_VALUES, ll.EXPORT_SOURCE_MASKS, ll.EXPORT_SOURCE_TARGETS, ll.EXPORT_SOURCE_WIENER, ll.EXPORT_SOURCE_Y]
    else:
        w = [ll.EXPORT_ARGMAX, ll.EXPORT_MASKS, ll.EXPORT_TARGETS, ll.EXPORT_WIENER, ll.EXPORT_Y]
    return w + ([ll.EXPORT_H] if inference else []) + [ll.EXPORT_COHERENCE, ll.EXPORT_VALID]


def _compare_items(a, b, what, cols, T, K, P):
    """Item `what` of a bank (a) and of a plain engine (b) on the columns `cols`, rows < K; the bank's rows >= K hold the fill."""
    col_axis = {ll.EXPORT_ARGMAX: 1, ll.EXPORT_MASKS: 1, ll.EXPORT_H: 1, ll.EXPORT_SOURCE_VALUES: 2, ll.EXPORT_SOURCE_MASKS: 2}
    if what in col_axis:
        cc = np.concatenate([cols, cols + T]) if what == ll.EXPORT_H else cols
        if col_axis[what] == 1:
            _eq(a[:K][:, cc], b[:, cc])
            pad = a[K:][:, cc]
        else:
            _eq(a[:, :K][:, :, cc], b[:, :, cc])
            pad = a[:, K:][:, :, cc]
        assert (pad == (-1 if what == ll.EXPORT_ARGMAX else 0)).all()
    elif what in (ll.EXPORT_TARGETS, ll.EXPORT_VALID, ll.EXPORT_SOURCE_TARGETS):
        _eq(a[cols], b[cols])
    else:                                  # (..., F, T) items
        _eq(a[..., cols], b[..., cols])


def _check_against_plain(p, bank, dents, sents, x, kw, schedule, use_graph, items, atoms, after=None):
    """Every (dictionary, table) pair in use against a plain llhist engine built with it, on the same input and schedule."""
    yb = _run(bank, x, 0, x.shape[2] // p['hop'], schedule, use_graph, after)
    last = bank.last_hops
    eb = {w: bank.export(w) for w in items}
    T = bank.S * last
    for i, K in enumerate(atoms):
        for j in range(len(p['E'])):
            streams = np.flatnonzero((dents == i) & (sents == j))
            if len(streams) == 0:
                continue
            plain = _engine(p, p['Ws'][i], p['E'][j], bank.S, **kw)
            if kw.get('historyLength'):
                plain.set_localization(None, 8)
            yp = _run(plain, x, 0, x.shape[2] // p['hop'], schedule, use_graph)
            _eq(yb[streams], yp[streams])
            cols = (streams[:, None] * last + np.arange(last)).ravel()
            for w in items:
                _compare_items(eb[w], plain.export(w), w, cols, T, K, bank.P)
            plain.close()
    return yb


SYNTH = ['online', 'lowlatency', 'windowed']
ONE = [(s, inf, P, Lh) for s in SYNTH for inf in (0, 5) for P in (0, 2, 4) for Lh in (0, 64)]


@pytest.mark.parametrize('synthesis,inference,P,Lh', ONE, ids=['-'.join(map(str, c)) for c in ONE])
def test_one_entry_bank_is_the_plain_engine(synthesis, inference, P, Lh):
    p = _setup(32, atoms=[64])
    S, hops = 5, 8
    kw = dict(synthesis=synthesis, numInferenceIterations=inference, numSources=P, historyLength=Lh)
    x = _audio(S, hops, p['hop'], seed=3)
    bank = _engine(p, [p['Ws'][0]], p['E'][1], S, **kw)
    steer = _engine(p, p['Ws'][0], [p['E'][1]], S, **kw)
    plain = _engine(p, p['Ws'][0], p['E'][1], S, **kw)
    for e in (bank, steer, plain):
        if Lh:
            e.set_localization(None, 5)
    ys = [_run(e, x, 0, hops, [1], True) for e in (bank, steer, plain)]
    _eq(ys[0], ys[2])
    _eq(ys[1], ys[2])
    for w in _items(P, inference) + ([ll.EXPORT_WINDOW_MEANS] if Lh else []) + ([ll.EXPORT_CARRIED_TARGETS, ll.EXPORT_STREAM_STATUS] if P else [ll.EXPORT_CARRY]):
        ref = plain.export(w)
        _eq(bank.export(w), ref)
        _eq(steer.export(w), ref)
    for e in (bank, steer, plain):
        e.close()


MIXED = [(D, P, inf, Lh, C) for D in (16, 32, 64, 128) for (P, inf, Lh, C) in ((0, 0, 0, 1), (0, 5, 64, 3), (2, 0, 0, 3), (2, 5, 64, 1))]


@pytest.mark.parametrize('D,P,inference,Lh,C', MIXED, ids=['-'.join(map(str, c)) for c in MIXED])
def test_mixed_dictionaries_match_plain_engines(D, P, inference, Lh, C):
    p = _setup(D)
    p['E'] = p['E'][:3]
    S, hops = 37, 12
    rng = np.random.RandomState(D + 7 * P + C)
    dents = rng.randint(0, len(ATOMS), S)
    sents = rng.randint(0, 3, S)
    kw = dict(hopsPerCall=C, numSources=P, numInferenceIterations=inference, historyLength=Lh)
    x = _audio(S, hops, p['hop'])
    schedule = [1] if C == 1 else [3, 1, 2]
    outs = []
    refined, ran = [], []

    def counts(e, k):
        if not P:
            refined.append(int(e.export(ll.EXPORT_REFINED)[0]))
            ran.append(int(e.export(ll.EXPORT_STATUS)[0]))
    for use_graph in (True, False):           # the same case as graphs and kernel by kernel
        bank = _engine(p, p['Ws'], p['E'], S, **kw)
        bank.assign_dictionary(None, dents)
        bank.assign_steering(None, sents)
        if Lh:
            bank.set_localization(None, 8)
        _eq(bank._export_now(ll.EXPORT_DICTIONARY_ASSIGNMENT), dents.astype(np.int32))
        outs.append(_check_against_plain(p, bank, dents, sents, x, kw, schedule, use_graph, _items(P, inference), ATOMS, counts))
        bank.process(x[:, :, :p['hop']])
        _eq(bank.export(ll.EXPORT_DICTIONARY_ATOMS), np.array(ATOMS, np.int32))
        bank.close()
    _eq(outs[0], outs[1])
    if not P:
        assert max(ran) == 0                  # the gated fallback never ran: the decisions came from the argmax path itself
        if D >= 32:
            assert sum(refined) > 0           # the grouped tensor-core GEMM ran and flagged near-ties for the float64 refinement


def test_1056_streams_over_64_dictionaries_and_4_tables():
    atoms = [4 * (i + 1) for i in range(64)]        # 4 .. 256
    p = _setup(32, atoms=atoms)
    S, hops = 1056, 3
    rng = np.random.RandomState(5)
    dents, sents = rng.permutation(np.arange(S) % 64), rng.randint(0, 4, S)
    bank = _engine(p, p['Ws'], p['E'], S)
    bank.assign_dictionary(None, dents)
    bank.assign_steering(None, sents)
    x = _audio(S, hops, p['hop'], seed=9)
    yb = _run(bank, x, 0, hops, [1], True)
    am = bank.export(ll.EXPORT_ARGMAX)
    for i in range(64):
        streams = np.flatnonzero(dents == i)
        ref = _engine(p, p['Ws'][i], p['E'], len(streams))       # an llbank engine built with W_i, the streams on their tables
        ref.assign_steering(None, sents[streams])
        yr = _run(ref, x[streams], 0, hops, [1], True)
        _eq(yb[streams], yr)
        _eq(am[:atoms[i]][:, streams], ref.export(ll.EXPORT_ARGMAX))
        assert (am[atoms[i]:][:, streams] == -1).all()
        ref.close()
    bank.close()


def test_settings_of_130_streams_in_one_call():
    """set_targets (-1 included), set_localization, assign_dictionary and assign_steering on 130 streams, each in one call that
    takes three launches of at most 64 streams: after one call of the engine its exports equal the host mirror."""
    p = _setup(16, atoms=[24, 64])
    S, P, Lh = 130, 3, 8
    rng = np.random.RandomState(130)
    bank = _engine(p, p['Ws'], p['E'], S, numSources=P, historyLength=Lh)
    bank.set_targets(None, rng.randint(-1, p['D'], (S, P)))
    bank.set_localization(None, rng.randint(0, Lh + 1, S))
    bank.assign_dictionary(None, rng.randint(0, 2, S))
    bank.assign_steering(None, rng.randint(0, len(p['E']), S))
    assert (bank._targets == -1).any() and (bank._targets >= 0).any()
    bank.process(_audio(S, 1, p['hop']))
    _eq(bank.export(ll.EXPORT_WINDOWS), bank._window)
    _eq(bank.export(ll.EXPORT_DICTIONARY_ASSIGNMENT), bank._dassign)
    _eq(bank.export(ll.EXPORT_ASSIGNMENT), bank._assign)
    # one hop per call: column s is stream s, on its override where one is set, else on its carried target
    _eq(bank.export(ll.EXPORT_SOURCE_TARGETS), np.where(bank._targets >= 0, bank._targets, bank.export(ll.EXPORT_CARRIED_TARGETS)))
    bank.close()


@pytest.mark.parametrize('inference', [0, 5])
def test_assign_and_load_dictionary_between_launches_of_a_kept_graph(inference):
    """Stream 2 runs 5 hops on W_a = entry 1 (K 64), is moved to entry 4 (K 256) by assign_dictionary, runs 4 hops, then entry 4 is
    replaced by W_c (K 100) with load_dictionary.  The reference is a plain stream saved from an engine on W_a and loaded into one
    on W_b, then into one on W_c.  Its records carry the engine's num_atoms, so a K change needs the header's num_atoms rewritten;
    that is sound because no per-stream state depends on K (the payload is the same bytes whatever K is: asserted below)."""
    p = _setup(32)
    S = 4
    kw = dict(numInferenceIterations=inference)
    x = _audio(S, 13, p['hop'], seed=4)
    bank = _engine(p, p['Ws'], p['E'][0], S, **kw)
    bank.assign_dictionary([2], 1)
    g = bank.build_graph()
    y = [_run(bank, x, 0, 5, [1], True)]
    rec_bank = bank.save_streams([2])
    bank.assign_dictionary([2], 4)
    y.append(_run(bank, x, 5, 9, [1], True))
    Wc = (np.random.RandomState(11).random_sample((p['Ws'][0].shape[0], 100)) + 0.01).astype(np.float32)
    bank.load_dictionary(4, Wc)
    y.append(_run(bank, x, 9, 13, [1], True))
    assert bank.build_graph() is g and len(bank._graphs) == 1      # the graph was kept
    yb = np.concatenate(y, -1)[2]

    def moved(src, W, K):
        rec = src.save_streams([0])
        dst = _engine(p, W, p['E'][0], 1, **kw)
        data = rec.data.numpy()
        data[0, ll.ATOMS_OFFSET:ll.ATOMS_OFFSET + 4] = np.array([K], np.int32).view(np.uint8)
        dst.load_streams([0], rec)
        return dst, rec

    xa = x[2:3]
    a = _engine(p, p['Ws'][1], p['E'][0], 1, **kw)
    ya = _run(a, xa, 0, 5, [1], True)
    payload = rec_bank.data.numpy()[0, records.RECORD_HEADER_BYTES:]
    b, rec_a = moved(a, p['Ws'][4], 256)
    pa = rec_a.data.numpy()[0, records.RECORD_HEADER_BYTES:]
    live = np.ones(len(pa), bool)
    live[24:32] = False                  # the alignment gap after the 24-byte stream parameters: no record writes it
    _eq(pa[live], payload[live])
    yb2 = _run(b, xa, 5, 9, [1], True)
    c, _ = moved(b, Wc, 100)
    yc = _run(c, xa, 9, 13, [1], True)
    _eq(yb, np.concatenate([ya, yb2, yc], -1)[0])
    for e in (bank, a, b, c):
        e.close()


def test_gated_fallback_on_mono_input():
    """Mono input ties the two central TDOAs in most decisions: far past the refinement list's 65536 entries at S = 512."""
    atoms = [512, 448, 512, 384]
    p = _setup(32, atoms=atoms)
    p['E'] = p['E'][:2]
    S, hops = 512, 3
    rng = np.random.RandomState(2)
    dents, sents = rng.randint(0, len(atoms), S), rng.randint(0, 2, S)
    bank = _engine(p, p['Ws'], p['E'], S)
    bank.assign_dictionary(None, dents)
    bank.assign_steering(None, sents)
    x = _audio(S, hops, p['hop'], seed=6, mono=True)
    ran = []
    yb = _run(bank, x, 0, hops, [1], True, after=lambda e, k: ran.append(int(e.export(ll.EXPORT_STATUS)[0])))
    assert max(ran) == 1                      # the refinement list overflowed and the float64 launch redid every decision
    am = bank.export(ll.EXPORT_ARGMAX)
    for i, K in enumerate(atoms):
        for j in range(2):
            streams = np.flatnonzero((dents == i) & (sents == j))
            if len(streams) == 0:
                continue
            plain = _engine(p, p['Ws'][i], p['E'][j], S)
            _eq(yb[streams], _run(plain, x, 0, hops, [1], True)[streams])
            _eq(am[:K][:, streams], plain.export(ll.EXPORT_ARGMAX)[:, streams])
            plain.close()
    bank.close()


def _state_of(eng):
    """Every stream's record payload and both assignments: what a refused load must leave as it was."""
    rec = eng.save_streams()
    return rec.data.numpy()[:, records.RECORD_HEADER_BYTES:].copy(), eng._export_now(ll.EXPORT_DICTIONARY_ASSIGNMENT), \
        eng._export_now(ll.EXPORT_ASSIGNMENT)


def _same_state(a, b):
    for u, v in zip(a, b):
        _eq(u, v)


def test_records_between_banks(tmp_path):
    p = _setup(32)
    S = 8
    src = _engine(p, p['Ws'], p['E'], S)
    dents = np.array([1, 2, 0, 4, 3, 5, 1, 2])
    sents = np.array([0, 1, 2, 3, 0, 1, 2, 3])
    src.assign_dictionary(None, dents)
    src.assign_steering(None, sents)
    x = _audio(S, 10, p['hop'])
    _run(src, x, 0, 4, [1], True)
    # lldict -> llbank: the stream on (W_4, E_3) into an llbank engine built with W_4 holding E_3 at entry 1
    one = _engine(p, p['Ws'][4], [p['E'][0], p['E'][3]], 2)
    one.load_streams([1], src.save_streams([3]))
    assert one._export_now(ll.EXPORT_ASSIGNMENT)[1] == 1
    ya = _run(src, x, 4, 6, [1], True)[3]
    yo = _run(one, np.stack([x[0], x[3]]), 4, 6, [1], True)[1]
    _eq(ya, yo)
    rec = src.save_streams()                             # every stream at hop 6
    # llbank -> lldict, into a bank with permuted and duplicated entries: the lowest entries holding W_4 and E_3
    perm = [p['Ws'][i] for i in (2, 4, 0, 4, 1, 3, 5)]
    tables = [p['E'][i] for i in (3, 1, 3, 0, 2)]
    dst = _engine(p, perm, tables, 3)
    dst.load_streams([2], one.save_streams([1]))
    assert dst._export_now(ll.EXPORT_DICTIONARY_ASSIGNMENT)[2] == 1
    assert dst._export_now(ll.EXPORT_ASSIGNMENT)[2] == 0
    # every stream of the source through a file into the permuted bank at other slots, then on together
    path = str(tmp_path / 'streams')
    rec.save(path)
    back = records.load(path + '.npz')
    big = _engine(p, perm, tables, 12)
    slots = [11, 0, 5, 3, 7, 9, 2, 4]
    big.load_streams(slots, back)
    lowest_d = {1: 4, 2: 0, 0: 2, 4: 1, 3: 5, 5: 6}
    lowest_s = {0: 3, 1: 1, 2: 4, 3: 0}
    _eq(big._export_now(ll.EXPORT_DICTIONARY_ASSIGNMENT)[slots], np.array([lowest_d[d] for d in dents], np.int32))
    _eq(big._export_now(ll.EXPORT_ASSIGNMENT)[slots], np.array([lowest_s[s] for s in sents], np.int32))
    xb = np.zeros((12, 2, x.shape[2]), np.float32)
    xb[slots] = x
    ys = _run(src, x, 6, 10, [1], True)
    yg = _run(big, xb, 6, 10, [1], True)
    _eq(yg[slots], ys)
    for e in (src, one, dst, big):
        e.close()


def test_refusals_leave_every_stream_unchanged():
    p = _setup(32)
    S = 6
    src = _engine(p, p['Ws'], p['E'], S)
    src.assign_dictionary(None, [0, 1, 2, 3, 4, 5])
    x = _audio(S, 4, p['hop'])
    _run(src, x, 0, 4, [1], True)
    rec = src.save_streams([2, 3])                       # dictionaries 2 (K 100) and 3 (K 128)
    # the destination holds W_2 but not W_3; its Kmax (128) admits both, so the digest lookup decides
    dst = _engine(p, [p['Ws'][0], p['Ws'][2], p['Ws'][5]], p['E'], 5)
    dst.assign_dictionary(None, [2, 1, 0, 2, 1])
    _run(dst, x[:5], 0, 3, [1], True)
    before = _state_of(dst)
    with pytest.raises(ParameterError, match='holds the stream'):
        dst.load_streams([0, 3], rec)                    # a non-contiguous list: the first record fits, the second is refused
    _same_state(_state_of(dst), before)
    # K mismatch: the record's header names 100 atoms, rewritten to 64 (the digest still names W_2)
    bad = src.save_streams([2])
    bad.data.numpy()[0, ll.ATOMS_OFFSET:ll.ATOMS_OFFSET + 4] = np.array([64], np.int32).view(np.uint8)
    with pytest.raises(ParameterError, match='atoms'):
        dst.load_streams([1], bad)
    _same_state(_state_of(dst), before)
    # the library refuses the same records on its own, before it touches the device
    for r, first in ((rec, 3), (bad, 1)):
        with pytest.raises(ParameterError):
            dst._record_call('load_streams', np.arange(first, first + r.count), r)
        _same_state(_state_of(dst), before)
    for e in (src, dst):
        e.close()


def test_library_and_engine_refusals_leave_the_state_unchanged():
    p = _setup(32, atoms=[24, 64])
    S = 3
    eng = _engine(p, p['Ws'], p['E'][:2], S)
    _run(eng, _audio(S, 3, p['hop']), 0, 3, [1], True)
    before = _state_of(eng)
    lib, h, cfg = eng.h.lib, eng.h.h, ctypes.byref(eng.cfg)
    st, nb = eng.state.data_ptr(), eng.state_bytes
    cs = eng.stream.cuda_stream
    W = eng._dicts[0]
    big = eng.torch.zeros((p['Ws'][0].shape[0], 65), dtype=eng.torch.float32, device=eng.h.device)
    i32 = lambda *v: (ctypes.c_int32 * len(v))(*v)          # noqa: E731
    assert lib.gccnmf_lldict_load_dictionary(h, cfg, 0, 0, 2, 2, st, nb, 0, big.data_ptr(), 65, None, cs) != 0     # K_i > Kmax
    assert lib.gccnmf_lldict_load_dictionary(h, cfg, 0, 0, 2, 2, st, nb, 0, W.data_ptr(), 0, None, cs) != 0        # K_i < 1
    assert lib.gccnmf_lldict_load_dictionary(h, cfg, 0, 0, 2, 2, st, nb, 2, W.data_ptr(), 24, None, cs) != 0       # entry outside
    assert lib.gccnmf_lldict_load_dictionary(h, cfg, 0, 0, 2, 2, st, nb, 0, None, 24, None, cs) != 0               # no W
    assert lib.gccnmf_lldict_assign(h, cfg, 0, 0, 2, 2, st, nb, 0, 1, i32(2), None, cs) != 0
    assert lib.gccnmf_lldict_assign(h, cfg, 0, 0, 2, 2, st, nb, 0, 1, None, i32(2), cs) != 0
    assert lib.gccnmf_lldict_assign(h, cfg, 0, 0, 2, 2, st, nb, 0, 1, i32(-2), None, cs) != 0
    assert lib.gccnmf_lldict_assign(h, cfg, 0, 0, 2, 2, st, nb, 2, 2, i32(0, 0), None, cs) != 0                    # streams outside
    assert lib.gccnmf_lldict_export(h, cfg, 0, 0, 2, 2, st, nb, 1, 29, eng.torch.zeros(8).data_ptr(), cs) != 0
    for qd, qe in ((0, 2), (65, 2), (2, 0), (2, 65)):
        assert lib.gccnmf_lldict_assign(h, cfg, 0, 0, qd, qe, st, nb, 0, 1, i32(0), None, cs) != 0
    ptrs = (ctypes.c_void_p * 2)(W.data_ptr(), big.data_ptr())
    c = eng._const
    assert lib.gccnmf_lldict_init(h, cfg, 0, 0, 2, 2, ptrs, (ctypes.c_int * 2)(24, 65), None, c[1].data_ptr(), c[2].data_ptr(), c[3].data_ptr(),
                                  float(eng.gain), st, nb, cs) != 0
    assert lib.gccnmf_lldict_init(h, cfg, 0, 0, 65, 2, ptrs, (ctypes.c_int * 2)(24, 64), None, c[1].data_ptr(), c[2].data_ptr(), c[3].data_ptr(),
                                  float(eng.gain), st, nb, cs) != 0
    eng.stream.synchronize()
    _same_state(_state_of(eng), before)
    with pytest.raises(ValueError):
        eng.load_dictionary(0, np.ones((p['Ws'][0].shape[0], 65), np.float32))      # K > Kmax
    with pytest.raises(ValueError):
        eng.load_dictionary(0, np.ones((10, 24), np.float32))                      # another F
    with pytest.raises(ValueError):
        eng.load_dictionary(2, p['Ws'][0])
    with pytest.raises(ValueError):
        eng.assign_dictionary([0], 2)
    with pytest.raises(ValueError):
        eng.assign_dictionary([3], 0)
    _same_state(_state_of(eng), before)
    eng.close()
