"""GPU: the real-time path over a bank of dictionaries and steering tables (MultiStreamRealtimeEngine with sequences of W and
expJOmegaTau, gccnmf_rtbank_*).  Slot s on entries (i, j) must compute bit for bit what an engine built with (W_i, E_j) computes:
every output block and every export item, with and without the graph, inference and sources."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SLOT_PARAMS = [
    dict(separationEnabled=True, localizationEnabled=True, localizationWindowSize=6),
    dict(separationEnabled=True, localizationEnabled=False, localizationWindowSize=6, targetTDOAIndex=3.0, mode=0, epsilon=4.0),
    dict(separationEnabled=False, localizationEnabled=True, localizationWindowSize=4),
    dict(separationEnabled=True, localizationEnabled=True, localizationWindowSize=3, beta=2.0, noiseFloor=0.1),
]
EXPORTS = range(9)
SOURCE_EXPORTS = range(9, 14)


def _steering(N, D, sep, sr=16000):
    from gcc_nmf_b200.realtime.gccNMFProcessor import steeringVectors
    freq = np.linspace(0, sr / 2, N // 2 + 1).astype(np.float32)
    return steeringVectors(freq, sep, D)[2]


def _dicts(N, Ks, seed=0):
    rng = np.random.default_rng(seed)
    return [(rng.random((N // 2 + 1, K)) ** 3).astype(np.float32) for K in Ks]


def _audio(S, B, blocks, seed=0):
    from gcc_nmf_b200.synth import synthetic_stereo
    n = blocks * B
    x = np.stack([synthetic_stereo(n / 16000.0 + 0.01, seed=seed + 17 * s)[:, :n] for s in range(S)])
    return np.ascontiguousarray(x.reshape(S, 2, blocks, B).transpose(2, 0, 1, 3))


def _engine(W, E, N, hop, B, nT, S, inference, P=0, **kw):
    from gcc_nmf_b200.realtime.multistream import MultiStreamRealtimeEngine
    win = np.sqrt(np.hamming(N).astype(np.float32))
    return MultiStreamRealtimeEngine(W, E, win, win, hop, B, nT, S, numInferenceIterations=inference, numSources=P, **kw)


def _exports(e, s, P):
    return [e.export(s, i) for i in (list(EXPORTS) + (list(SOURCE_EXPORTS) if P else []))]


def _assert_same(a, b, what):
    assert len(a) == len(b)
    for i, (u, v) in enumerate(zip(a, b)):
        assert u.shape == v.shape and np.array_equal(u, v, equal_nan=True), (what, i)


# ------------------------------------------------------------------------------------------------ heterogeneous slots
@pytest.mark.parametrize('P', [0, 3])
@pytest.mark.parametrize('inference', [0, 3])
@pytest.mark.parametrize('nT', [1, 4])
def test_heterogeneous_slots_equal_single_engines(P, inference, nT):
    """7 slots over 3 dictionaries (K = 64, 77, 200; K_max = 200 is not a multiple of 16) and 2 spacings, mixed parameters:
    every block and every export item of every slot equals a one-slot engine built with the slot's (W_i, E_j)."""
    N, D, blocks = 512, 32, 8
    hop = N // 4
    B = nT * hop
    Ws = _dicts(N, [64, 77, 200], seed=nT + inference)
    Es = [_steering(N, D, 0.1), _steering(N, D, 0.23)]
    S = 7
    entries = [(s % 3, (s // 3) % 2) for s in range(S)]
    bank = _engine(Ws, Es, N, hop, B, nT, S, inference, P)
    bank.assign(range(S), [d for d, _ in entries], [e for _, e in entries])
    refs = []
    for s, (d, e) in enumerate(entries):
        params = dict(SLOT_PARAMS[s % len(SLOT_PARAMS)])
        if P:
            params.pop('targetTDOAIndex', None)
            params.pop('mode', None)
        bank.set_params(s, **params)
        r = _engine(Ws[d], Es[e], N, hop, B, nT, 1, inference, P)
        r.set_params(0, **params)
        refs.append(r)
    x = _audio(S, B, blocks, seed=P)
    for b in range(blocks):
        graph = b % 2 == 0
        y = bank.process_blocks(x[b], use_graph=graph).copy()
        for s in range(S):
            yr = refs[s].process_blocks(x[b][s:s + 1], use_graph=not graph)
            assert np.array_equal(y[s], yr[0]), (b, s)
            _assert_same(_exports(bank, s, P), _exports(refs[s], 0, P), (b, s))
            assert tuple(bank.export(s, 14)) == entries[s] == bank.assignment(s)
    K_of = [w.shape[1] for w in Ws]
    for s, (d, _) in enumerate(entries):
        assert bank.export(s, 6).shape == (K_of[d], 2 * nT)


def test_frames_mode_and_forced_masks_equal_single_engines():
    """process_frames with and without forced (S, K_max, nT) masks: rows at or beyond K_i are ignored."""
    N, D, nT = 256, 16, 2
    hop = N // 4
    Ws = _dicts(N, [48, 96], seed=5)
    Es = [_steering(N, D, 0.1)]
    bank = _engine(Ws, Es, N, hop, nT * hop, nT, 4, 0)
    bank.assign([1, 3], 1)
    refs = [_engine(Ws[s % 2], Es[0], N, hop, nT * hop, nT, 1, 0) for s in range(4)]
    rng = np.random.default_rng(2)
    for it in range(4):
        frames = rng.standard_normal((4, 2, N, nT)).astype(np.float32)
        forced = rng.random((4, 96, nT)) if it % 2 else None
        y = bank.process_frames(frames, forcedAtomMask=forced).copy()
        for s in range(4):
            f = None if forced is None else forced[s:s + 1, :Ws[s % 2].shape[1]]
            assert np.array_equal(y[s], refs[s].process_frames(frames[s:s + 1], forcedAtomMask=f)[0]), (it, s)
            _assert_same(_exports(bank, s, 0), _exports(refs[s], 0, 0), (it, s))


# ------------------------------------------------------------------------------------------------ wide atoms tile
@pytest.mark.parametrize('D,nT', [(64, 1), (32, 2)])
def test_wide_atoms_tile_straddling_entries(D, nT):
    """S = 141, slot s on dictionary s mod 3: the 128 x 128 atoms tile runs (>= 132 CTAs) and its CTAs hold pairs of several
    entries.  Every slot equals the same slot of a multi-stream engine with that slot's dictionary alone."""
    N, S, blocks = 512, 141, 3
    hop = N // 4
    B = nT * hop
    Ws = _dicts(N, [64, 77, 200], seed=D)
    Es = [_steering(N, D, 0.1)]
    bank = _engine(Ws, Es, N, hop, B, nT, S, 0)
    bank.assign(range(S), [s % 3 for s in range(S)])
    bank.set_params(range(S), **SLOT_PARAMS[0])
    refs = [_engine(w, Es[0], N, hop, B, nT, S, 0) for w in Ws]
    for r in refs:
        r.set_params(range(S), **SLOT_PARAMS[0])
    x = _audio(4, B, blocks, seed=D)
    for b in range(blocks):
        xb = x[b][np.arange(S) % 4]
        y = bank.process_blocks(xb).copy()
        yr = [r.process_blocks(xb).copy() for r in refs]
        for s in range(S):
            assert np.array_equal(y[s], yr[s % 3][s]), (b, s)
        for s in (0, 1, 2, 70, 71, 139, 140):
            _assert_same(_exports(bank, s, 0), _exports(refs[s % 3], s, 0), (b, s))


# ------------------------------------------------------------------------------------------------ switching between launches
@pytest.mark.parametrize('switch', ['dictionary', 'steering', 'load_dictionary', 'load_steering'])
def test_switching_between_graph_launches(switch):
    """assign / load_* between graph launches: the block path equals oracle.OverlapAddProcessorOracle around frames-mode engines
    that switch at the same block.  The twins run every block, so their histories do not depend on which one was used: a
    dictionary switch keeps localisation on (history and target checked), a steering switch keeps it off."""
    from oracle import gccnmf_oracle as orc
    N, D, nT, blocks, at = 512, 32, 2, 10, 5
    hop = N // 4
    B = nT * hop
    Ws = _dicts(N, [64, 120], seed=9)
    Es = [_steering(N, D, 0.1), _steering(N, D, 0.3)]
    localize = switch in ('dictionary', 'load_dictionary')
    params = dict(SLOT_PARAMS[0], localizationEnabled=localize)
    bank = _engine(Ws, Es, N, hop, B, nT, 2, 0)
    bank.set_params(range(2), **params)
    if switch == 'dictionary':
        before, after = (Ws[0], Es[0]), (Ws[1], Es[0])
    elif switch == 'steering':
        before, after = (Ws[0], Es[0]), (Ws[0], Es[1])
    elif switch == 'load_dictionary':
        before, after = (Ws[0], Es[0]), (Ws[1], Es[0])
    else:
        before, after = (Ws[0], Es[0]), (Ws[0], Es[1])
    twins = [_engine(w, e, N, hop, B, nT, 1, 0) for w, e in (before, after)]
    for t in twins:
        t.set_params(0, **params)
    ola = orc.OverlapAddProcessorOracle(2, N, hop, B, nT)
    x = _audio(2, B, blocks, seed=4)
    bank.build_graph()
    for b in range(blocks):
        if b == at:
            if switch in ('dictionary', 'steering'):
                bank.assign(0, *((1, None) if switch == 'dictionary' else (None, 1)))
            elif switch == 'load_dictionary':
                bank.load_dictionary(0, Ws[1])
            else:
                bank.load_steering(0, Es[1])
        y = bank.process_blocks(x[b]).copy()
        cur = twins[1 if b >= at else 0]

        def frames_fn(windowed):
            outs = [t.process_frames(windowed[None]).copy()[0] for t in twins]
            return outs[1 if b >= at else 0]
        ref = ola.processFrames(x[b][0], frames_fn)
        assert np.array_equal(y[0], ref), b
        for i in (1, 2, 5, 7, 8) if localize else (2, 5):
            assert np.array_equal(bank.export(0, i), cur.export(0, i), equal_nan=True), (b, i)
    # slot 1 stayed on its entries only for an assignment; a load changes entry 0 for every slot on it
    assert bank.assignment(1) == (0, 0)


# ------------------------------------------------------------------------------------------------ reset, activation, one entry
def test_reset_and_activation_keep_or_restore_entries():
    N, D, nT, blocks = 256, 16, 1, 4
    hop = N // 4
    Ws = _dicts(N, [32, 64], seed=1)
    Es = [_steering(N, D, 0.1), _steering(N, D, 0.2)]
    bank = _engine(Ws, Es, N, hop, hop, nT, 3, 2)
    bank.assign([0, 1, 2], [1, 1, 0], [1, 0, 1])
    bank.set_active(1, False)
    x = _audio(3, hop, blocks)
    for b in range(blocks):
        y = bank.process_blocks(x[b], use_graph=b % 2 == 0).copy()
        assert not y[1].any()
    assert tuple(bank.export(1, 14)) == (1, 0)
    bank.reset_slots([0, 1])
    assert tuple(bank.export(0, 14)) == (0, 0) == tuple(bank.export(1, 14)) and tuple(bank.export(2, 14)) == (0, 1)
    assert bank.export(0, 6).shape == (32, 2)
    ref = _engine(Ws[0], Es[0], N, hop, hop, nT, 1, 2)
    for b in range(blocks):
        y = bank.process_blocks(x[b]).copy()
        assert np.array_equal(y[0], ref.process_blocks(x[b][:1])[0]), b


def test_settings_of_130_slots_in_one_call():
    """assign and set_targets on 130 slots, each in one call that takes three launches of at most 64 slots, with a mix of -1
    (keep) and values, twice: every slot's EXPORT_ASSIGNMENT and EXPORT_TARGETS equal the host's expectation."""
    N, D, P, S = 256, 16, 3, 130
    hop = N // 4
    Ws = _dicts(N, [32, 64, 48], seed=6)
    Es = [_steering(N, D, 0.1), _steering(N, D, 0.2)]
    bank = _engine(Ws, Es, N, hop, hop, 1, S, 0, P)
    rng = np.random.default_rng(130)
    entries = np.zeros((S, 2), np.int64)
    targets = np.tile([(2 * q + 1) * D // (2 * P) for q in range(P)], (S, 1))
    for _ in range(2):
        d, e, t = rng.integers(-1, 3, S), rng.integers(-1, 2, S), rng.integers(-1, D, (S, P))
        bank.assign(range(S), d, e)
        bank.set_targets(range(S), t)
        entries = np.where(np.stack([d, e], 1) >= 0, np.stack([d, e], 1), entries)
        targets = np.where(t >= 0, t, targets)
    for s in range(S):
        assert tuple(bank.export(s, 14)) == tuple(entries[s]) == bank.assignment(s), s
        assert np.array_equal(bank.export(s, 9), targets[s]), s


@pytest.mark.parametrize('P', [0, 2])
def test_bank_of_one_entry_equals_multi_stream_engine(P):
    N, D, nT, S, blocks = 512, 64, 1, 5, 6
    hop = N // 4
    W = _dicts(N, [128], seed=3)[0]
    E = _steering(N, D, 0.1)
    bank = _engine([W], [E], N, hop, hop, nT, S, 3, P)
    ref = _engine(W, E, N, hop, hop, nT, S, 3, P)
    for e in (bank, ref):
        e.set_params(range(S), **SLOT_PARAMS[0])
    x = _audio(S, hop, blocks, seed=7)
    for b in range(blocks):
        assert np.array_equal(bank.process_blocks(x[b], use_graph=b % 2 == 0), ref.process_blocks(x[b], use_graph=b % 2 == 1)), b
        for s in range(S):
            _assert_same(_exports(bank, s, P), _exports(ref, s, P), (b, s))


def test_invalid_bank_arguments():
    N, D = 256, 16
    Ws = _dicts(N, [32, 64])
    Es = [_steering(N, D, 0.1)]
    with pytest.raises(ValueError):
        _engine(Ws, [_steering(N, 8, 0.1), Es[0]], N, 64, 64, 1, 2, 0)       # D differs
    with pytest.raises(ValueError):
        _engine([Ws[0], _dicts(512, [32])[0]], Es, N, 64, 64, 1, 2, 0)       # F differs
    bank = _engine(Ws, Es, N, 64, 64, 1, 2, 0)
    with pytest.raises(ValueError):
        bank.assign(0, 2)
    with pytest.raises(ValueError):
        bank.assign(0, None, 1)
    with pytest.raises(ValueError):
        bank.load_dictionary(0, _dicts(N, [65])[0])                            # K_i > K_max
    from gcc_nmf_b200 import _lib
    import ctypes
    st = bank.h.lib.gccnmf_rtbank_load_dictionary(bank.h.h, ctypes.byref(bank.cfg), 2, 0, 2, 1, bank.state.data_ptr(), bank.state_bytes, 0,
                                                  bank._dicts[0][0].data_ptr(), 65, None, bank.stream.cuda_stream)
    assert st == _lib.GCCNMF_ERR_INVALID_ARGUMENT
    bad = (ctypes.c_int32 * 1)(5)
    st = bank.h.lib.gccnmf_rtbank_assign(bank.h.h, ctypes.byref(bank.cfg), 2, 0, 2, 1, bank.state.data_ptr(), bank.state_bytes, 0, 1, bad, None,
                                         bank.stream.cuda_stream)
    assert st == _lib.GCCNMF_ERR_INVALID_ARGUMENT


# ------------------------------------------------------------------------------------------------ runner
def test_run_many_with_per_file_sizes_and_spacings(tmp_path):
    from scipy.io import wavfile
    from gcc_nmf_b200.realtime.runRealtimeGCCNMF import RealtimeGCCNMFNoGUI
    from gcc_nmf_b200.synth import synthetic_stereo
    from gcc_nmf_b200.wavio import float2pcm
    N, sizes, seps = 512, [64, 128, 64], [0.1, 0.1, 0.2]
    rng = np.random.default_rng(0)
    dicts = {'Pretrained': {k: (rng.random((N // 2 + 1, k)) ** 3).astype(np.float32) for k in (64, 128)}}
    paths = []
    for i, n in enumerate((9000, 7000, 8000)):
        p = str(tmp_path / ('in%d.wav' % i))
        wavfile.write(p, 16000, float2pcm(synthetic_stereo(n / 16000.0, seed=i)[:, :n].T))
        paths.append(p)
    kw = dict(dictionariesW=dicts, windowSize=N, hopSize=128, blockSize=128, numTDOAs=32, dictionarySizes=[64, 128])
    many = RealtimeGCCNMFNoGUI(paths[0], **kw).runMany(paths, dictionarySizes=sizes, microphoneSeparations=seps)
    for i, p in enumerate(paths):
        one = RealtimeGCCNMFNoGUI(p, dictionarySize=sizes[i], microphoneSeparationInMetres=seps[i], **kw).run()
        assert np.array_equal(many[i], one), i


# ------------------------------------------------------------------------------------------------ regressions
def test_grouped_inference_with_ragged_atom_count():
    """rtm engine (no bank) with inference, nT = 3 and K = 42 (not a multiple of the 8 atoms of an update CTA), with enough slots
    for the grouped inference and filter warps: every slot equals a one-slot engine fed the same blocks."""
    N, D, nT, S, blocks = 256, 16, 3, 180, 5
    hop = N // 4
    B = nT * hop
    W = _dicts(N, [42], seed=11)[0]
    E = _steering(N, D, 0.1)
    many = _engine(W, E, N, hop, B, nT, S, 3)
    refs = [_engine(W, E, N, hop, B, nT, 1, 3) for _ in range(4)]
    for e in [many] + refs:
        e.set_params(range(e.S), **SLOT_PARAMS[0])
    x = _audio(4, B, blocks, seed=13)
    for b in range(blocks):
        y = many.process_blocks(x[b][np.arange(S) % 4], use_graph=b % 2 == 0).copy()
        yr = [r.process_blocks(x[b][c:c + 1])[0].copy() for c, r in enumerate(refs)]
        for s in range(S):
            assert np.array_equal(y[s], yr[s % 4]), (b, s)
        for s in (0, 1, S - 2, S - 1):
            _assert_same(_exports(many, s, 0), _exports(refs[s % 4], 0, 0), (b, s))


def test_exports_keep_the_shape_of_the_block_they_come_from():
    """After an assign or a load that changes K_i, and before the next block, the K-shaped items are still the last block's, at
    its K_i; from the next block on they have the new K_i."""
    N, D, nT = 256, 16, 1
    hop = N // 4
    Ws = _dicts(N, [32, 80], seed=2)
    E = _steering(N, D, 0.1)
    bank = _engine(Ws, [E], N, hop, hop, nT, 2, 2)
    x = _audio(2, hop, 4, seed=1)
    assert bank.export(0, 6).shape == (32, 2)                  # no block yet: the current entry's K_i
    bank.process_blocks(x[0])
    before = [bank.export(0, i) for i in (2, 5, 6)]
    bank.assign(0, 1)
    bank.load_dictionary(0, _dicts(N, [48], seed=3)[0])         # slot 1 is on entry 0
    for i, v in zip((2, 5, 6), before):
        assert np.array_equal(bank.export(0, i), v, equal_nan=True), i
    assert bank.export(1, 6).shape == (32, 2)
    bank.process_blocks(x[1])
    assert bank.export(0, 6).shape == (80, 2) and bank.export(1, 6).shape == (48, 2)
    assert bank.export(0, 2).shape == (80, 1) and bank.export(1, 5).shape == (48, 1)
