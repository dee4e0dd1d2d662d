"""GPU: moving live streams of the low-latency engine (LowLatencyEngine.save_streams / load_streams, gccnmf_llrec_*).  The reference
is an engine in which every stream stays where it started, fed the same hops: the moved stream, every other stream of both engines,
and the moved stream's carried maximum, carried targets and status must equal it bit for bit.  Also: a save / load round trip in
place, an inactive stream, a record through a file into an engine on a second handle, a second device, the host mirrors of the
settings, and refusals that launch nothing."""
import ctypes

import numpy as np
import pytest

from gcc_nmf_b200 import _lib
from gcc_nmf_b200 import lowlatency as ll
from gcc_nmf_b200 import records

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


def _audio(S, hops, hop, seed=1):
    """S different stereo streams: a delayed source per stream (delay s - S / 2 between the channels) plus a second one entering
    half way, so the running maximum and its peaks move while the streams run."""
    rng = np.random.RandomState(seed)
    n = hops * hop
    x = np.zeros((S, 2, n))
    for s in range(S):
        for i, d in enumerate((s % 7 - 3, 3 - s % 5)):
            v = rng.standard_normal(n + 16)
            part = np.stack([v[8:8 + n], v[8 - d:8 - d + n]])
            part[:, :i * n // 2] = 0
            x[s] += part
    return (x / np.abs(x).max()).astype(np.float32)


def _engine(p, S, C=1, P=0, synthesis='lowlatency', inference=0, **kw):
    return ll.LowLatencyEngine(p['W'], p['E'], p['win'], p['syn'], p['hop'], numStreams=S, hopsPerCall=C, synthesis=synthesis,
                               numSources=P, numInferenceIterations=inference, targetTDOAEpsilon=2.5, **kw)


def _feed(eng, x, h0, h1, use_graph):
    """Hops [h0, h1) of x (S, 2, n) through eng in calls of at most eng.C hops -> the outputs along the last axis."""
    hop, out = eng.hop, []
    h = h0
    while h < h1:
        c = min(eng.C, h1 - h)
        out.append(eng.process(x[:, :, h * hop:(h + c) * hop], use_graph=use_graph))
        h += c
    return np.concatenate(out, axis=-1) if out else None


def _eps_of(s):
    """Epsilon of stream s: only the atoms localised at the target (0.25) or every atom within 6 TDOAs of it.  Atoms of these
    broadband dictionaries localise at or next to the dominant TDOA, so a narrower wide epsilon would give the same masks."""
    return 0.25 if s % 2 else 6.0


def _settings(eng):
    """Per-stream settings that change the output, so that a setting that does not travel shows: epsilon and a target override
    (single target), or one source's target override (sources)."""
    S = eng.S
    if eng.P:
        eng.set_targets(range(S), [[-1] * (eng.P - 1) + [(3 * s) % eng.D] for s in range(S)])
    else:
        eng.set_params(range(S), targetTDOAEpsilon=[_eps_of(s) for s in range(S)])
        eng.set_params([S - 1], targetOverride=3)


def _carried(eng, s):
    out = [eng.export(ll.EXPORT_CARRY)[s]]
    if eng.P:
        out += [eng.export(ll.EXPORT_CARRIED_TARGETS)[s], eng.export(ll.EXPORT_STREAM_STATUS)[s]]
    return out


# (synthesis, P, inference iterations, hop count of the move as a multiple of Q plus an offset, direction)
CASES = [('lowlatency', 0, 0, (0, 0), 'down'), ('lowlatency', 0, 5, (0, 1), 'up'), ('online', 0, 0, (1, -1), 'down'),
         ('windowed', 0, 0, (1, 0), 'up'), ('windowed', 0, 5, (2, 5), 'down'), ('online', 2, 0, (1, 0), 'up'),
         ('windowed', 2, 5, (0, 1), 'down'), ('lowlatency', 2, 0, (2, 5), 'down'), ('lowlatency', 8, 0, (1, -1), 'up'),
         ('windowed', 8, 5, (2, 5), 'up')]


@pytest.mark.parametrize('synthesis,P,inference,at,direction', CASES, ids=['-'.join(map(str, c)) for c in CASES])
def test_move_equals_unmoved(synthesis, P, inference, at, direction):
    """Stream 5 of an 8-stream engine (3 hops per call) moves to stream 0 of a 3-stream engine (1 hop per call), or back; one engine
    runs by graph, the other kernel by kernel.  The source saves and reloads its own stream in place as well."""
    p = _setup()
    Q = -(-p['N'] // p['hop'])
    h0 = at[0] * Q + at[1]
    h1 = h0 + max(3 * Q, 8) + 2
    x = _audio(8, h1, p['hop'])
    big = dict(S=8, C=3, use_graph=True, slot=5, streams=list(range(8)))
    small = dict(S=3, C=1, use_graph=False, slot=0, streams=[5, 6, 7])     # small engine's streams of x (slot 0: x[5] once moved)
    src, dst = (big, small) if direction == 'down' else (small, big)
    # the unmoved reference: all 8 streams of x in one engine, settings as the engines below give them
    ref = _engine(p, 8, 1, P, synthesis, inference)
    _settings(ref)
    want = _feed(ref, x, 0, h1, True)
    want_carried = _carried(ref, 5)
    engines = {}
    for role, d in (('src', src), ('dst', dst)):
        e = engines[role] = _engine(p, d['S'], d['C'], P, synthesis, inference)
        # each engine's streams carry the settings of the reference's stream they stand for
        if P:
            e.set_targets(range(d['S']), [[-1] * (P - 1) + [(3 * s) % e.D] for s in d['streams']])
        else:
            e.set_params(range(d['S']), targetTDOAEpsilon=[_eps_of(s) for s in d['streams']])
            if 7 in d['streams']:
                e.set_params([d['streams'].index(7)], targetOverride=3)
    # before the move the destination's slot runs other audio (stream 0 of x in the big engine, stream 2 in the small one) under
    # settings of its own, which the load must replace
    before = {'src': [x[s] for s in src['streams']], 'dst': [x[s] for s in dst['streams']]}
    before['dst'][dst['slot']] = x[2] if dst is small else x[0]
    if P:
        engines['dst'].set_targets([dst['slot']], [[1] + [-1] * (P - 1)])
    else:
        engines['dst'].set_params([dst['slot']], targetTDOAEpsilon=6.0, targetOverride=2)
    got = {r: [_feed(engines[r], np.stack(before[r]), 0, h0, d['use_graph'])] for r, d in (('src', src), ('dst', dst))}
    rec = engines['src'].save_streams([src['slot']])
    engines['src'].load_streams([src['slot']], rec)            # in place: changes nothing
    launches = engines['dst'].h.launches
    engines['dst'].load_streams([dst['slot']], rec)
    assert engines['dst'].h.launches == launches + 1
    after = {'src': before['src'], 'dst': [x[s] for s in dst['streams']]}
    for r, d in (('src', src), ('dst', dst)):
        got[r].append(_feed(engines[r], np.stack(after[r]), h0, h1, d['use_graph']))
    for r, d in (('src', src), ('dst', dst)):
        y = np.concatenate([g for g in got[r] if g is not None], axis=-1)
        for i, s in enumerate(d['streams']):
            lo = h0 * p['hop'] if (r == 'dst' and i == d['slot']) else 0
            assert np.array_equal(y[i, ..., lo:], want[s, ..., lo:]), (r, i, s)
    for r, d in (('src', src), ('dst', dst)):
        for a, b in zip(_carried(engines[r], d['slot']), want_carried):
            assert np.array_equal(a, b, equal_nan=True), r


def test_inactive_stream_moves_and_resumes():
    """An inactive stream moves as it is (still inactive, zeros out) and, once active again, resumes where it stopped."""
    p = _setup()
    P, hop = 2, p['hop']
    x = _audio(2, 60, hop, seed=4)
    ref = _engine(p, 2, 1, P, 'windowed')
    want = [_feed(ref, x, 0, 13, True)]
    ref.set_active([1], False)
    want.append(_feed(ref, x, 13, 20, True))
    ref.set_active([1], True)
    want.append(_feed(ref, x, 20, 60, True))
    want = np.concatenate(want, axis=-1)
    a, b = _engine(p, 2, 2, P, 'windowed'), _engine(p, 4, 1, P, 'windowed')
    ya = [_feed(a, x, 0, 13, False)]
    a.set_active([1], False)
    ya.append(_feed(a, x, 13, 17, False))
    rec = a.save_streams([1])
    b.load_streams([3], rec)
    assert b._active[3] == 0
    xb = np.zeros((4, 2, x.shape[2]), np.float32)
    xb[3] = x[1]
    yb = [_feed(b, xb, 17, 20, True)]
    assert not yb[0][3].any()
    b.set_active([3], True)
    yb.append(_feed(b, xb, 20, 60, True))
    yb = np.concatenate(yb, axis=-1)
    assert np.array_equal(yb[3], want[1, ..., 17 * hop:])
    assert np.array_equal(np.concatenate(ya, axis=-1)[1], want[1, ..., :17 * hop])


def test_suspend_to_file_and_resume_on_another_handle(tmp_path, monkeypatch):
    """Two streams parked in a file and restored, in swapped order, into a new engine that runs on a handle of its own."""
    p = _setup()
    hop, Q = p['hop'], -(-p['N'] // p['hop'])
    x = _audio(3, 5 * Q, hop, seed=5)
    ref = _engine(p, 3, 1, 0, 'online', inference=5)
    _settings(ref)
    want = _feed(ref, x, 0, 5 * Q, True)
    a = _engine(p, 3, 4, 0, 'online', inference=5)
    _settings(a)
    _feed(a, x, 0, Q + 3, True)
    a.save_streams([2, 0]).save(str(tmp_path / 'parked'))
    a.close()
    del a
    monkeypatch.setitem(_lib._default_handles, 0, _lib.Handle(0))
    b = _engine(p, 2, 1, 0, 'online', inference=5)
    assert b.h is _lib._default_handles[0]
    b.load_streams([0, 1], records.load(str(tmp_path / 'parked.npz')))
    assert b._eps.tolist() == [ref._eps[2], ref._eps[0]] and b._override.tolist() == [3, -1]
    y = _feed(b, x[[2, 0]], Q + 3, 5 * Q, False)
    assert np.array_equal(y, want[[2, 0], ..., (Q + 3) * hop:])


def test_move_to_second_device():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip('needs two devices')
    p = _setup()
    hop = p['hop']
    x = _audio(2, 40, hop, seed=6)
    ref = _engine(p, 2, 1, 2, 'windowed')
    want = _feed(ref, x, 0, 40, True)
    a = _engine(p, 2, 1, 2, 'windowed', device=0)
    b = _engine(p, 1, 3, 2, 'windowed', device=1)
    _feed(a, x, 0, 11, True)
    b.load_streams([0], a.save_streams([1]))
    assert np.array_equal(_feed(b, x[1:], 11, 40, True)[0], want[1, ..., 11 * hop:])


def test_loaded_settings_survive_a_neighbours_update():
    """set_params rewrites a whole range of streams from the host mirrors: after a load, a neighbour's update must leave the loaded
    stream's epsilon and override as the record brought them."""
    p = _setup()
    hop = p['hop']
    x = _audio(3, 40, hop, seed=7)
    ref = _engine(p, 3, 1)
    ref.set_params([1], targetTDOAEpsilon=4.5, targetOverride=9)
    want = _feed(ref, x, 0, 40, True)
    a = _engine(p, 3, 1)
    a.set_params([1], targetTDOAEpsilon=4.5, targetOverride=9)
    _feed(a, x, 0, 12, True)
    b = _engine(p, 3, 1)
    b.load_streams([1], a.save_streams([1]))
    b.set_params([0, 2], targetTDOAEpsilon=2.5)            # sends streams 0 .. 2 from the mirrors
    y = _feed(b, x, 12, 40, True)
    assert np.array_equal(y[1], want[1, ..., 12 * hop:])
    # the check has teeth: the destination's own settings give another output
    c = _engine(p, 3, 1)
    c.load_streams([1], a.save_streams([1]))
    c.set_params([1], targetTDOAEpsilon=2.5, targetOverride=-1)
    assert not np.array_equal(_feed(c, x, 12, 40, True)[1], want[1, ..., 12 * hop:])


def _load_raw(eng, first, count, data, nbytes=None):
    ws = eng.h.torch.empty(max(1, int(eng.h.lib.gccnmf_llrec_workspace_bytes(ctypes.byref(eng.cfg), eng.P, max(count, 1)))),
                           dtype=eng.h.torch.uint8, device=eng.h.device)
    return eng.h.lib.gccnmf_llrec_load_streams(eng.h.h, ctypes.byref(eng.cfg), eng.P, eng.state.data_ptr(), eng.state_bytes, first, count,
                                              data.data_ptr(), data.numel() if nbytes is None else nbytes, ws.data_ptr(), ws.numel(),
                                              eng.stream.cuda_stream)


def _corrupt(rec, torch, field, index=None):
    """A copy of a one-stream record with one header field changed."""
    bad = records.StreamRecord(rec.kind, rec.num_sources, rec.data.clone().pin_memory(), rec.mirrors)
    head = bad.header(0)
    if field == 'config':
        head.config[index] += 1
    else:
        setattr(head, field, {'magic': 0x12345678, 'abi_version': 1, 'kind': 1, 'num_sources': 2, 'payload_bytes': 16,
                              'synthesis_digest': head.synthesis_digest ^ 1}[field])
    bad.data[0, :ctypes.sizeof(head)] = torch.frombuffer(bytearray(bytes(head)), dtype=torch.uint8)
    return bad


def _payloads(eng, streams):
    n = int(eng.h.lib.gccnmf_llrec_workspace_bytes(ctypes.byref(eng.cfg), eng.P, 1))
    return eng.save_streams(streams).data.numpy()[:, _lib.RECORD_HEADER_BYTES:_lib.RECORD_HEADER_BYTES + n].copy()


def test_refusals_launch_nothing():
    """Every incompatible record is refused by load_streams (on the host, before any library call) and by the C entry itself,
    and neither launches anything; a refused multi-stream load leaves every stream as it was."""
    p = _setup()
    a = _engine(p, 2, 1, 0, 'lowlatency')
    _feed(a, _audio(2, 10, p['hop']), 0, 10, True)
    rec = a.save_streams([0])
    assert bytes(rec.header(0)) == bytes(a._record_header())          # the host's header is the library's
    rec2 = _engine(p, 2, 1, 2, 'lowlatency').save_streams([0])
    q = _setup(N=128, m=16)
    others = [lambda: _engine(q, 2), lambda: _engine(p, 2, synthesis='online'), lambda: _engine(p, 2, synthesis='windowed'),
              lambda: _engine(_setup(hop=16), 2), lambda: _engine(_setup(K=72), 2), lambda: _engine(_setup(D=32), 2),
              lambda: _engine(p, 2, inference=5), lambda: _engine(p, 2, sparsityAlpha=0.5),
              lambda: _engine(p, 2, epsilon=1e-12), lambda: _engine(p, 2, P=2)]
    for make in others:
        e = make()
        n = e.h.launches
        with pytest.raises(_lib.ParameterError):
            e.load_streams([1], rec)
        assert _load_raw(e, 1, 1, rec.data) != 0
        assert e.h.launches == n
    e = _engine(p, 2, 1, 3)
    n = e.h.launches
    with pytest.raises(_lib.ParameterError):
        e.load_streams([0], rec2)                                 # P = 2 into P = 3
    assert _load_raw(e, 0, 1, rec2.data) != 0
    assert e.h.launches == n
    b = _engine(p, 4, 3, 0, 'lowlatency')                         # compatible: other S and C
    n = b.h.launches
    torch = b.h.torch
    bads = [_corrupt(rec, torch, f) for f in ('magic', 'abi_version', 'kind', 'num_sources', 'payload_bytes', 'synthesis_digest')]
    bads += [_corrupt(rec, torch, 'config', i) for i in range(16)]
    for bad in bads:
        with pytest.raises(_lib.ParameterError):
            b.load_streams([2], bad)
        assert _load_raw(b, 2, 1, bad.data) != 0
    with pytest.raises(ValueError):
        b.load_streams([4], rec)                                  # outside [0, S)
    with pytest.raises(ValueError):
        b.load_streams([0, 1], rec)                               # two streams, one record
    assert _load_raw(b, 3, 2, rec.data) != 0                      # streams [3, 5) of 4
    assert _load_raw(b, -1, 1, rec.data) != 0
    assert _load_raw(b, 0, 1, rec.data, nbytes=rec.data.numel() - 1) != 0          # record too short
    assert b.h.launches == n
    # two runs ([0], [2]) whose second record is bad: nothing is loaded, no mirror changes
    before, eps = _payloads(b, [0, 2]), b._eps.copy()
    two = records.StreamRecord(rec.kind, 0, torch.cat([rec.data, bads[-1].data]).pin_memory(),
                               {k: np.concatenate([v, v]) for k, v in rec.mirrors.items()})
    b.set_params([0, 2], targetTDOAEpsilon=6.0)
    eps[[0, 2]] = 6.0
    n = b.h.launches
    with pytest.raises(_lib.ParameterError):
        b.load_streams([0, 2], two)
    assert b.h.launches == n and np.array_equal(b._eps, eps)
    assert np.array_equal(_payloads(b, [0, 2])[:, 32:], before[:, 32:])      # past LLStream, whose epsilon set_params changed
    n = b.h.launches
    assert _load_raw(b, 0, 1, rec.data) == 0                      # and the good record loads
    assert b.h.launches == n + 1


def _payload_regions(eng):
    """Bytes of each region of a stream's record payload, in order (the low-latency carve without history)."""
    R = (-(-eng.N // eng.hop) - 1) * eng.hop
    sizes = [24, 8 * eng.D, 4 * 2 * R, 4 * 2 * eng.N * max(eng.P, 1)] + ([32, 32, 4] if eng.P else [])
    return [b for b in sizes if b]


@pytest.mark.parametrize('form', ['llrec-P0', 'llrec-P2', 'llbank'])
def test_saved_bytes_are_all_defined(form):
    """A save through the C entry writes every byte of its records: the padding after each payload region, the header past its
    struct and the record past its payload are zero, whatever the device staging and the host buffer held before, so two saves of
    the same state are byte-identical."""
    import torch
    p = _setup()
    P = 2 if form == 'llrec-P2' else 0
    if form == 'llbank':
        from gcc_nmf_b200 import gccNMFFunctions as fn
        E2 = fn.getExpJOmegaTau(fn.getFrequenciesInHz(SR, p['N'] // 2 + 1), fn.getTDOAsInSeconds(0.2, p['D']))
        eng = ll.LowLatencyEngine(p['W'], [p['E'], E2], p['win'], p['syn'], p['hop'], numStreams=3, targetTDOAEpsilon=2.5)
        head = _lib.LLBankRecordHeader
    else:
        eng = _engine(p, 3, P=P)
        head = _lib.RecordHeader
    _feed(eng, _audio(3, 12, p['hop']), 0, 12, True)
    rb, count = eng.record_bytes, 3
    ws_bytes = int(eng._rec('workspace_bytes')(count))
    saves = []
    for staging_fill, host_fill in ((0xFF, 0xAB), (0x00, 0xCD)):
        ws = torch.full((ws_bytes,), staging_fill, dtype=torch.uint8, device=eng.h.device)
        rec = torch.full((count, rb), host_fill, dtype=torch.uint8).pin_memory()
        eng._check(eng._rec('save_streams')(eng.state.data_ptr(), eng.state_bytes, 0, count, rec.data_ptr(), rec.numel(), ws.data_ptr(),
                                            ws.numel(), eng.stream.cuda_stream))
        eng.stream.synchronize()
        saves.append(rec.numpy().copy())
    assert np.array_equal(saves[0], saves[1])
    data, H = saves[0], _lib.RECORD_HEADER_BYTES
    assert not data[:, ctypes.sizeof(head):H].any()                              # the header past its struct
    at = H
    for b in _payload_regions(eng):
        pad = -(-b // 16) * 16
        assert not data[:, at + b:at + pad].any(), (at - H, b)                # the padding after each region
        at += pad
    assert at - H == eng._record_header().payload_bytes
    assert not data[:, at:].any()                                                 # the record past its payload
