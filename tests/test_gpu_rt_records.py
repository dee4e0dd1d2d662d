"""GPU: moving live slots of the real-time engines (save_streams / load_streams of RealtimeEngine and MultiStreamRealtimeEngine,
gccnmf_rtrec_*).  The reference is an engine in which no slot moved, fed the same blocks: every output block of every slot of the
engines involved, and the moved slot's target, history, history index, targets, status and bank assignment, must equal it bit for
bit (NaN-equal).  Moves happen at several block counts with a history ring that wraps, between graph and kernel-by-kernel engines,
between engine forms (single stream, rtm, rtsep, bank) and between banks whose entries sit at other indexes.  Refusals are checked
through Python (nothing launched) and through the C entry (host fields: nothing launched; digests: only the digest kernels, the
state unchanged)."""
import ctypes

import numpy as np
import pytest

from gcc_nmf_b200 import _lib

pytestmark = pytest.mark.gpu

N, HOP, NT, D, HIST = 256, 64, 2, 16, 5
B = HOP * NT
F = N // 2 + 1


def _steering(sep):
    from gcc_nmf_b200.realtime.gccNMFProcessor import steeringVectors
    freq = np.linspace(0, 8000, F).astype(np.float32)
    return steeringVectors(freq, sep, D)[2]


def _dicts(Ks, seed=0):
    rng = np.random.default_rng(seed)
    return [(rng.random((F, K)) ** 3).astype(np.float32) for K in Ks]


def _audio(S, blocks, seed=0):
    from gcc_nmf_b200.synth import synthetic_stereo
    n = blocks * B
    x = np.stack([synthetic_stereo(n / 16000.0 + 0.01, seed=seed + 17 * s)[:, :n] for s in range(S)])
    return np.ascontiguousarray(x.reshape(S, 2, blocks, B).transpose(2, 0, 1, 3)).astype(np.float32)


WIN = np.sqrt(np.hamming(N)).astype(np.float32)


def _engine(W, E, S, inference=0, P=0, win=WIN, **kw):
    from gcc_nmf_b200.realtime.multistream import MultiStreamRealtimeEngine
    return MultiStreamRealtimeEngine(W, E, win, win, HOP, B, NT, S, historyLength=HIST, numInferenceIterations=inference, numSources=P, **kw)


def _single(W, E, inference=0, **kw):
    from gcc_nmf_b200.realtime.engine import RealtimeEngine
    return RealtimeEngine(W, E, WIN, WIN, HOP, B, NT, historyLength=HIST, numInferenceIterations=inference, **kw)


def _params(s, loc, P, mode=1):
    p = dict(separationEnabled=True, localizationEnabled=loc, localizationWindowSize=2 + s % 3, epsilon=1.0 + s % 4, beta=1.0 + 0.5 * (s % 2))
    if not P:
        p.update(mode=mode, targetTDOAIndex=float((3 * s + 1) % D))
    return p


def _configure(e, streams, loc, P, mode=1):
    """Slot i of e gets the settings of stream streams[i]."""
    for i, s in enumerate(streams):
        e.set_params([i], **_params(s, loc, P, mode))
        if P and not loc:
            e.set_targets([i], [[(s + 5 * q) % D for q in range(P)]])


def _carried(e, slot, P):
    """Target, history and history index; with sources also the targets and the status."""
    from gcc_nmf_b200.realtime import multistream as ms
    items = [ms.EXPORT_TARGET, ms.EXPORT_HISTORY, ms.EXPORT_HISTORY_INDEX] + ([ms.EXPORT_TARGETS, ms.EXPORT_STATUS] if P else [])
    return [e.export(slot, i) for i in items]


def _order(e):
    """The `order` array of a bank state (rt_carve: the slots sorted by dictionary, which rt_atoms walks), read from the state."""
    up = lambda x: (x + 255) // 256 * 256          # noqa: E731
    Fp, K, used, off = (F + 3) & ~3, e.K, 0, 0
    for n in (4 * F * K, 4 * K * Fp, 4 * F, 4 * K, 8 * K):           # W, W^T, recV, colsumW, H0 of one entry
        used = up(used) + n
    for n in (8 * N, 4 * N, 4 * N, 4 * N, e.Qd * up(used), e.Qe * up(8 * D * Fp), 4 * 64):
        off = up(off) + n
    e.stream.synchronize()
    return e.state[up(off):up(off) + 4 * e.S].cpu().numpy().view(np.int32)


def _assert_sorted(e):
    """A load re-sorts the bank's slots by dictionary (stable), as assign does."""
    d = [e.assignment(s)[0] for s in range(e.S)]
    assert list(_order(e)) == list(np.argsort(d, kind='stable')), d


def _same(a, b, what):
    assert len(a) == len(b), what
    for i, (u, v) in enumerate(zip(a, b)):
        assert u.shape == v.shape and np.array_equal(u, v, equal_nan=True), (what, i)


# ------------------------------------------------------------------------------------------------ move timing
# (inference, mode, P, block count of the move, localisation)
CASES = [(0, 1, 0, 0, True), (5, 0, 0, 1, True), (0, 0, 0, 3, False), (5, 1, 0, 7, False), (0, 1, 0, 8, True), (5, 1, 0, 9, True),
         (0, 1, 2, 0, True), (5, 1, 2, 3, False), (0, 1, 2, 9, True), (0, 1, 8, 1, True), (5, 1, 8, 7, False), (0, 1, 8, 8, False)]


@pytest.mark.parametrize('inference,mode,P,m,loc', CASES, ids=['-'.join(map(str, c)) for c in CASES])
def test_move_and_back_equals_unmoved(inference, mode, P, m, loc):
    """Slot 5 of an 8-slot engine (by graph) moves to slot 0 of a 3-slot engine (kernel by kernel) after m blocks and back three
    blocks later; the source slot is reset in between, the destination slot ran other audio under other settings before."""
    W, E = _dicts([32])[0], _steering(0.1)
    m2, T = m + 3, m + 6
    x = _audio(8, T, seed=m + 10 * P)
    ref = _engine(W, E, 8, inference, P)
    _configure(ref, range(8), loc, P, mode)
    want, want_carried = [], [_carried(ref, 5, P)]
    for b in range(T):
        want.append(ref.process_blocks(x[b]).copy())
        want_carried.append(_carried(ref, 5, P))
    a = _engine(W, E, 8, inference, P)
    _configure(a, range(8), loc, P, mode)
    d = _engine(W, E, 3, inference, P)
    _configure(d, [2, 6, 7], loc, P, mode)
    for b in range(T):
        if b == m:
            rec = a.save_streams([5])
            a.reset_slots([5])
            d.load_streams([0], rec)
            _same(_carried(d, 0, P), want_carried[b], ('carried after the move', b))
            assert d._params[0] == ref._params[5]
        if b == m2:
            rec = d.save_streams([0])
            a.load_streams([5], rec)
            d.reset_slots([0])
            _same(_carried(a, 5, P), want_carried[b], ('carried after the move back', b))
        out_a = a.process_blocks(x[b]).copy()
        out_d = d.process_blocks(np.stack([x[b][5] if m <= b < m2 else x[b][2], x[b][6], x[b][7]]), use_graph=False).copy()
        for s in range(8):
            if s != 5 or not m <= b < m2:
                assert np.array_equal(out_a[s], want[b][s]), ('source engine', b, s)
        if m <= b < m2:
            assert np.array_equal(out_d[0], want[b][5]), ('moved slot', b)
        assert np.array_equal(out_d[1:], want[b][6:]), ('destination engine', b)
    _same(_carried(a, 5, P), want_carried[T], 'carried at the end')
    assert a._params == ref._params


# ------------------------------------------------------------------------------------------------ cross-form moves
def _run_move(src, src_slot, dst, dst_slot, ref, x, m, T):
    """ref and src run stream `src_slot` of x (T, S, 2, B) in slot src_slot (the other slots other streams); after m blocks the slot
    moves into dst_slot of dst (kernel by kernel), which runs the same stream there.  Every block of the moved stream equals ref's."""
    S = x.shape[1]

    def feed(e, b, slot, shift, **kw):
        blk = np.stack([x[b][src_slot] if i == slot else x[b][(i + shift) % S] for i in range(e.S)])
        return e.process_blocks(blk, **kw)[slot].copy()
    for b in range(T):
        want = feed(ref, b, src_slot, 1)
        if b == m:
            dst.load_streams([dst_slot], src.save_streams([src_slot]))
        got = feed(src, b, src_slot, 1) if b < m else feed(dst, b, dst_slot, 3, use_graph=False)
        assert np.array_equal(got, want), b


@pytest.mark.parametrize('inference', [0, 5])
def test_bank_slot_into_rtm_engine(inference):
    """A bank slot on (3, 1) goes into an rtm engine built with (W_3, E_1); its blocks equal that rtm engine's unmoved slot."""
    Ws, Es = _dicts([32, 48, 20, 40], seed=1), [_steering(0.1), _steering(0.2)]
    x = _audio(4, 10, seed=3)
    bank = _engine(Ws, Es, 4, inference)
    bank.assign([2], 3, 1)
    ref = _engine(Ws[3], Es[1], 4, inference)
    for e in (bank, ref):
        _configure(e, range(4), True, 0)
    dst = _engine(Ws[3], Es[1], 3, inference)
    _run_move(bank, 2, dst, 1, ref, x, 4, 10)


@pytest.mark.parametrize('inference', [0, 5])
def test_rtm_slot_into_bank_at_another_index(inference):
    """An rtm slot goes into slot 0 of a bank that holds its (W, E) at entries (2, 1): the exported assignment is (2, 1), the slot
    moves to the end of the dictionary order, and the blocks equal the unmoved rtm slot's."""
    from gcc_nmf_b200.realtime import multistream as ms
    Ws, Es = _dicts([32, 48, 40], seed=2), [_steering(0.1), _steering(0.2)]
    x = _audio(3, 10, seed=4)
    src = _engine(Ws[2], Es[1], 3, inference)
    ref = _engine(Ws[2], Es[1], 3, inference)
    for e in (src, ref):
        _configure(e, range(3), True, 0)
    dst = _engine(Ws, Es, 5, inference)
    _run_move(src, 1, dst, 0, ref, x, 5, 10)
    assert tuple(dst.export(0, ms.EXPORT_ASSIGNMENT)) == (2, 1) == dst.assignment(0)
    _assert_sorted(dst)                                                   # slot 0 now comes after the slots on entry 0


@pytest.mark.parametrize('inference', [0, 5])
def test_bank_into_permuted_bank_with_sources(inference):
    """P = 3: a slot on (1, 0) of one bank goes into a bank with the entries permuted, one more entry and a larger K_max; it lands
    on the entries holding the same content, and its blocks, targets and status equal the unmoved slot's."""
    from gcc_nmf_b200.realtime import multistream as ms
    Ws, Es = _dicts([32, 40, 24], seed=5), [_steering(0.1), _steering(0.25)]
    big = _dicts([64], seed=6)[0]
    x = _audio(4, 10, seed=5)
    src = _engine(Ws, Es, 4, inference, 3)
    ref = _engine(Ws, Es, 4, inference, 3)
    for e in (src, ref):
        e.assign([0], 1, 0)
        _configure(e, range(4), True, 3)
    dst = _engine([Ws[2], big, Ws[1], Ws[0], Ws[1]], [Es[1], Es[0], Es[0]], 2, inference, 3)
    m, T = 4, 10
    for b in range(T):
        want = ref.process_blocks(x[b])[0].copy()
        if b < m:
            got = src.process_blocks(x[b])[0].copy()
        else:
            if b == m:
                dst.load_streams([1], src.save_streams([0]))
                assert dst.assignment(1) == (2, 1) and tuple(dst.export(1, ms.EXPORT_ASSIGNMENT)) == (2, 1)
                _assert_sorted(dst)
            got = dst.process_blocks(np.stack([x[b][3], x[b][0]]), use_graph=b % 2 == 0)[1].copy()
        assert np.array_equal(got, want), b
    _same(_carried(dst, 1, 3), _carried(ref, 0, 3), 'carried')


@pytest.mark.parametrize('inference', [0, 5])
def test_single_stream_engine_to_slot_and_back(inference):
    """A RealtimeEngine's stream moves into slot 1 of an rtm engine and back into the (reset) RealtimeEngine."""
    W, E = _dicts([32], seed=7)[0], _steering(0.1)
    x = _audio(3, 12, seed=6)
    ref, src = _single(W, E, inference), _single(W, E, inference)
    for e in (ref, src):
        e.set_params(**_params(0, True, 0))
    multi = _engine(W, E, 3, inference)
    _configure(multi, [1, 1, 2], True, 0)
    for b in range(12):
        want = ref.process_block(x[b][0]).copy()
        if b == 3:
            multi.load_streams([1], src.save_streams())
            src.reset()
        if b == 7:
            src.load_streams(multi.save_streams([1]))
        if 3 <= b < 7:
            got = multi.process_blocks(np.stack([x[b][1], x[b][0], x[b][2]]))[1].copy()
        else:
            got = src.process_block(x[b][0], use_graph=b % 2 == 1).copy()
        assert np.array_equal(got, want), b
    _same([src.export(i) for i in (1, 7, 8)], [ref.export(i) for i in (1, 7, 8)], 'carried')


def test_records_identical_across_forms():
    """The same stream saved from an rtm slot, a bank slot and a RealtimeEngine gives byte-identical records."""
    Ws, Es = _dicts([32, 40], seed=8), [_steering(0.1), _steering(0.2)]
    x = _audio(3, 6, seed=7)
    rtm = _engine(Ws[1], Es[1], 3, 5)
    bank = _engine(Ws + [_dicts([48], seed=9)[0]], Es, 3, 5)
    bank.assign([1], 1, 1)
    single = _single(Ws[1], Es[1], 5)
    for e in (rtm, bank):
        _configure(e, [0, 1, 2], True, 0)
    single.set_params(**_params(1, True, 0))
    for b in range(6):
        rtm.process_blocks(x[b])
        bank.process_blocks(x[b], use_graph=False)
        single.process_block(x[b][1])
    a, c, s = rtm.save_streams([1]), bank.save_streams([1]), single.save_streams()
    assert np.array_equal(a.data.numpy(), c.data.numpy())
    assert np.array_equal(a.data.numpy(), s.data.numpy())
    assert a.header(0).dictionary_atoms == 40


# ------------------------------------------------------------------------------------------------ other cases
def test_in_place_inactive_file_and_mirrors(tmp_path, monkeypatch):
    """A save and load in place; an inactive slot that moves and resumes later; two slots parked in a file and restored in swapped
    order on a second handle; the moved slots' host mirrors under a neighbour's set_params / set_active."""
    from gcc_nmf_b200 import records
    W, E = _dicts([32], seed=10)[0], _steering(0.15)
    T = 12
    x = _audio(6, T, seed=8)
    ref, src = _engine(W, E, 6, 5), _engine(W, E, 6, 5)
    for e in (ref, src):
        _configure(e, range(6), True, 0)
    want = []
    for b in range(T):
        if b == 2:
            ref.set_active([3], False)
        if b == 8:
            ref.set_active([3], True)
        want.append(ref.process_blocks(x[b]).copy())
    for b in range(4):
        if b == 1:
            src.load_streams([2], src.save_streams([2]))
        if b == 2:
            src.set_active([3], False)
        assert np.array_equal(src.process_blocks(x[b]), want[b]), b
    path = str(tmp_path / 'parked')
    src.save_streams([1, 3]).save(path)
    monkeypatch.setitem(_lib._default_handles, 0, _lib.Handle(0))
    dst = _engine(W, E, 6, 5)
    assert dst.h is not src.h
    dst.load_streams([3, 1], records.load(path + '.npz'))        # slot 3 <- stream 1, slot 1 <- stream 3
    assert dst._params[1] == src._params[3] and dst._params[3] == src._params[1] and not dst.is_active(1)
    dst.set_params([0, 2], **_params(9, False, 0))                  # neighbours' settings change; the loaded slots keep theirs
    dst.set_active([2], True)
    for b in range(4, T):
        if b == 8:
            dst.set_active([1], True)
        out = dst.process_blocks(np.stack([x[b][0], x[b][3], x[b][2], x[b][1], x[b][4], x[b][5]]), use_graph=b % 2 == 0)
        assert np.array_equal(out[3], want[b][1]) and np.array_equal(out[1], want[b][3]), b
    assert dst._params[3] == ref._params[1] and dst._params[1] == ref._params[3]


def test_frames_path_carries_history_and_target():
    """process_frames: the history and the localised target travel with the record."""
    W, E = _dicts([32], seed=11)[0], _steering(0.1)
    rng = np.random.default_rng(0)
    frames = rng.standard_normal((8, 3, 2, N, NT)).astype(np.float32)
    ref, src, dst = _engine(W, E, 3), _engine(W, E, 3), _engine(W, E, 2)
    for e in (ref, src, dst):
        _configure(e, range(e.S), True, 0)
    for b in range(8):
        want = ref.process_frames(frames[b])[2].copy()
        if b == 5:
            dst.load_streams([0], src.save_streams([2]))
        got = (src.process_frames(frames[b]) if b < 5 else dst.process_frames(np.stack([frames[b][2], frames[b][0]])))
        assert np.array_equal(got[2 if b < 5 else 0], want), b
    _same(_carried(dst, 0, 0), _carried(ref, 2, 0), 'carried')


def test_second_device():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip('one GPU: the move to a second device is not run here')
    W, E = _dicts([32], seed=12)[0], _steering(0.1)
    x = _audio(2, 8, seed=9)
    ref, src, dst = _engine(W, E, 2), _engine(W, E, 2), _engine(W, E, 2, device=1)
    for e in (ref, src, dst):
        _configure(e, range(2), True, 0)
    for b in range(8):
        want = ref.process_blocks(x[b])[1].copy()
        if b == 4:
            dst.load_streams([1], src.save_streams([1]))
        got = (src if b < 4 else dst).process_blocks(x[b])[1]
        assert np.array_equal(got, want), b


# ------------------------------------------------------------------------------------------------ refusals
def _state(e):
    e.stream.synchronize()
    return e.state.cpu().numpy().copy()


def _c_load(e, rec, first=0, count=None, record_bytes=None, workspace=None, ws_bytes=None):
    count = rec.count if count is None else count
    n = int(e.h.lib.gccnmf_rtrec_workspace_bytes(ctypes.byref(e.cfg), *e._record_dims, max(count, 1)))
    ws = e.torch.empty(n + 16, dtype=e.torch.uint8, device=e.h.device) if workspace is None else workspace
    st = e.h.lib.gccnmf_rtrec_load_slots(e.h.h, ctypes.byref(e.cfg), *e._record_dims, e.state.data_ptr(), e.state_bytes, first, count,
                                         rec.data.data_ptr(), rec.data.numel() if record_bytes is None else record_bytes,
                                         ws.data_ptr(), n if ws_bytes is None else ws_bytes, e.stream.cuda_stream)
    e.stream.synchronize()
    return st


def _refused(e, rec, launches_c, slots=(0,)):
    """Python refuses without a launch; the C entry refuses with `launches_c` launches; the state is unchanged."""
    from gcc_nmf_b200._lib import ParameterError
    before, n0 = _state(e), e.h.launches
    with pytest.raises((ParameterError, ValueError)):
        e.load_streams(list(slots), rec)
    assert e.h.launches == n0
    if rec.data.shape[1] >= e.record_bytes:
        assert _c_load(e, rec) != 0
    assert e.h.launches - n0 == launches_c or (rec.data.shape[1] < e.record_bytes and e.h.launches == n0)
    assert np.array_equal(_state(e), before)


def _saved(e, slots=(0,)):
    e.process_blocks(_audio(e.S, 1, seed=1)[0])
    return e.save_streams(list(slots))


def _copy(rec):
    from gcc_nmf_b200.records import StreamRecord
    return StreamRecord(rec.kind, rec.num_sources, rec.data.clone().pin_memory(), {k: v.copy() for k, v in rec.mirrors.items()})


CONFIG_CHANGES = [dict(hop=HOP // 2), dict(B=2 * B), dict(nT=1), dict(D=D + 1), dict(hist=HIST + 1), dict(inference=3), dict(alpha=0.1),
                  dict(epsilon=1e-12)]


@pytest.mark.parametrize('change', CONFIG_CHANGES, ids=[list(c)[0] for c in CONFIG_CHANGES])
def test_refuses_other_configuration(change):
    from gcc_nmf_b200.realtime.gccNMFProcessor import steeringVectors
    from gcc_nmf_b200.realtime.multistream import MultiStreamRealtimeEngine
    W = _dicts([32], seed=13)[0]
    rec = _saved(_engine(W, _steering(0.1), 2, 5))
    c = dict(hop=HOP, B=B, nT=NT, D=D, hist=HIST, inference=5, alpha=0.0, epsilon=1e-16)
    c.update(change)
    E = steeringVectors(np.linspace(0, 8000, F).astype(np.float32), 0.1, c['D'])[2]
    if 'B' in change:
        c['nT'] = c['B'] // c['hop']
    e = MultiStreamRealtimeEngine(W, E, WIN, WIN, c['hop'], c['B'], c['nT'], 2, historyLength=c['hist'], numInferenceIterations=c['inference'],
                                  sparsityAlpha=c['alpha'], epsilon=c['epsilon'])
    _refused(e, rec, 0)


def test_refuses_other_window_size():
    W = _dicts([32], seed=13)[0]
    rec = _saved(_engine(W, _steering(0.1), 2))
    from gcc_nmf_b200.realtime.multistream import MultiStreamRealtimeEngine
    from gcc_nmf_b200.realtime.gccNMFProcessor import steeringVectors
    W2 = np.ascontiguousarray(np.concatenate([W, W[1:]], axis=0)[:2 * N // 2 + 1])
    E2 = steeringVectors(np.linspace(0, 8000, N + 1).astype(np.float32), 0.1, D)[2]
    win2 = np.sqrt(np.hamming(2 * N)).astype(np.float32)
    _refused(MultiStreamRealtimeEngine(W2, E2, win2, win2, HOP, B, 1, 2, historyLength=HIST), rec, 0)


def test_refuses_other_sources():
    W, E = _dicts([32], seed=14)[0], _steering(0.1)
    for P_src, P_dst in ((2, 3), (3, 2), (0, 2), (2, 0)):
        _refused(_engine(W, E, 2, 0, P_dst), _saved(_engine(W, E, 2, 0, P_src)), 0)


def test_refuses_other_content():
    """The windows, a dictionary or steering table the destination lacks, another seed with inference: Python launches nothing;
    the C entry runs only the two digest kernels and leaves the state bytes as they were."""
    Ws, Es = _dicts([32, 40], seed=15), [_steering(0.1), _steering(0.2)]
    rec = _saved(_engine(Ws, Es, 2, 5), (0, 1))
    rec0 = _copy(rec)
    rec0.data = rec.data[:1].clone().pin_memory()
    for k in rec0.mirrors:
        rec0.mirrors[k] = rec.mirrors[k][:1]
    other_win = np.sqrt(np.hanning(N)).astype(np.float32)
    _refused(_engine(Ws, Es, 2, 5, win=other_win), rec0, 2)
    _refused(_engine([Ws[1]], Es, 2, 5), rec0, 2)                    # slot 0 is on dictionary 0
    _refused(_engine(Ws, [Es[1]], 2, 5), rec0, 2)                    # and on steering 0
    _refused(_engine(Ws, Es, 2, 5, seedValue=1), rec0, 2)            # H0 differs
    _refused(_engine([np.ascontiguousarray(Ws[0][:, :31])], Es, 2, 5), rec0, 2)
    # a two-run load whose second record is refused changes no slot
    e = _engine(Ws, Es, 4, 5)
    e.assign([0, 1, 2, 3], 0, 0)
    bad = _copy(rec)
    bad.data.numpy()[1, 40] ^= 1                                      # steering digest of record 1
    _refused(e, bad, 2, slots=(0, 2))
    # after the refusals the untouched engine still loads the good record
    e.load_streams([0, 2], rec)


def test_refuses_header_fields_ranges_and_sizes():
    from gcc_nmf_b200._lib import RtRecordHeader
    W, E = _dicts([32], seed=16)[0], _steering(0.1)
    e = _engine(W, E, 3, 5, 2)
    rec = _saved(e)
    # every header field and config word: host fields refuse with nothing launched, digests after the digest kernels
    offsets = [(f, getattr(RtRecordHeader, f).offset) for f, _ in RtRecordHeader._fields_ if f != 'config']
    offsets += [('config[%d]' % i, RtRecordHeader.config.offset + 4 * i) for i in range(16)]     # num_atoms (word 4) travels as 0
    for name, off in offsets:
        bad = _copy(rec)
        bad.data.numpy()[0, off] ^= 0x10
        _refused(e, bad, 2 if name.endswith('_digest') or name == 'dictionary_atoms' else 0)
    # ranges, record size, workspace
    n0, before = e.h.launches, _state(e)
    for first, count in ((-1, 1), (3, 1), (2, 2), (0, 0), (0, 4)):
        assert _c_load(e, rec, first, count) != 0, (first, count)
    assert _c_load(e, rec, record_bytes=rec.data.numel() - 1) != 0
    assert _c_load(e, rec, ws_bytes=16) != 0
    ws = e.torch.empty(1 << 22, dtype=e.torch.uint8, device=e.h.device)
    assert _c_load(e, rec, workspace=ws[4:]) != 0
    assert e.h.launches == n0 and np.array_equal(_state(e), before)
    for bad_slots in ([3], [0, 0]):
        with pytest.raises((IndexError, ValueError)):
            e.load_streams(bad_slots, rec)
    with pytest.raises(ValueError):                                   # count mismatch
        e.load_streams([0, 1], rec)
    ll = _copy(rec)
    ll.kind = _lib.RECORD_KIND_LL
    with pytest.raises(ValueError):
        e.load_streams([0], ll)
