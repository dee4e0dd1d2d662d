"""GPU: the real-time path with several sources per stream (MultiStreamRealtimeEngine(numSources=P), gccnmf_rtsep_*).

Every stage the sources add is checked bit for bit against the host model (oracle/rt_exact.py, oracle/rt_sources.py) from the
device's own exports of the stage before; each source's output is checked bit for bit against a single-target slot fed that
source's mask; the sources sum to the separation-off output; a slot of an S-slot engine equals a one-slot engine.  Every case
runs kernel by kernel and through the graph (alternating blocks)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _consts(g, K=None, D=None, seed=0, mirrored=False):
    """W, expJOmegaTau and the window of realtime_mini, or a random W of K atoms and D TDOAs.  mirrored: E[:, D-1-d] =
    conj(E[:, d]), so that a mono input gives bit-identical GCC rows at mirrored TDOAs."""
    from gcc_nmf_b200 import gccNMFFunctions as fn
    sr, N, K0, D0 = [int(v) for v in g['params']]
    W = g['W'] if K is None else (np.random.default_rng(seed).random((N // 2 + 1, K)) ** 3).astype(np.float32)
    D = D0 if D is None else D
    freq = np.linspace(0, sr / 2, N // 2 + 1).astype(np.float32)
    maxT = float(g['micSep']) / fn.SPEED_OF_SOUND_IN_METRES_PER_SECOND
    tdoas = np.linspace(-maxT, maxT, D).astype(np.float32)
    E = np.exp(np.outer(freq, -(2j * np.pi) * tdoas)).astype(np.complex64)
    if mirrored:
        E[:, D - 1 - np.arange(D // 2)] = np.conj(E[:, :D // 2])
    win = np.sqrt(np.hamming(N).astype(np.float32))
    return W, E, win, N


def _audio(S, B, blocks, seed=0):
    """(blocks, S, 2, B) float32: a different synthetic two-source mixture per slot."""
    from gcc_nmf_b200.synth import synthetic_stereo
    n = blocks * B
    x = np.stack([synthetic_stereo(n / 16000.0 + 0.01, seed=seed + 17 * s)[:, :n] for s in range(S)])
    return np.ascontiguousarray(x.reshape(S, 2, blocks, B).transpose(2, 0, 1, 3))


SLOT_PARAMS = [
    dict(separationEnabled=True, localizationEnabled=True, localizationWindowSize=6),
    dict(separationEnabled=True, localizationEnabled=False, localizationWindowSize=6),
    dict(separationEnabled=False, localizationEnabled=True, localizationWindowSize=4),
    dict(separationEnabled=True, localizationEnabled=True, localizationWindowSize=3),
    dict(separationEnabled=True, localizationEnabled=True, localizationWindowSize=10),
]


def _sep(W, E, win, hop, B, nT, S, P, inference, params=None):
    from gcc_nmf_b200.realtime.multistream import MultiStreamRealtimeEngine
    e = MultiStreamRealtimeEngine(W, E, win, win, hop, B, nT, S, numInferenceIterations=inference, numSources=P)
    params = params or SLOT_PARAMS[0]
    e.set_params(range(S), **params)
    return e


# ------------------------------------------------------------------------------------------------ 1: stages against the model
@pytest.mark.parametrize('inference', [0, 5])
@pytest.mark.parametrize('nT', [1, 4])
@pytest.mark.parametrize('D', [16, 64, 128])
@pytest.mark.parametrize('tile', ['narrow', 'wide'])
@pytest.mark.parametrize('P', [2, 3, 8])
def test_stages_bit_exact_against_model(golden, P, tile, D, nT, inference):
    from gcc_nmf_b200.realtime import multistream as ms
    from oracle import rt_exact as rx
    from oracle import rt_sources as rs
    g = golden('realtime_mini')
    K = 128
    W, E, win, N = _consts(g, K=K, D=D, seed=D + P)
    hop = N // 4
    B = nT * hop
    Dp = 32 if D <= 32 else 64 if D <= 64 else 128
    # wide: enough (slot, frame) pairs for K / 128 x pairs / (128 / Dp) >= 132 CTAs of the 128 x 128 tile
    S = 3 if tile == 'narrow' else -(-132 * (128 // Dp) // nT)
    check = [0, S - 1]
    blocks = 4
    x = _audio(min(S, 4), B, blocks, seed=P)
    e = _sep(W, E, win, hop, B, nT, S, P, inference)
    hist = {s: e.export(s, ms.EXPORT_HISTORY) for s in check}
    index = {s: int(e.export(s, ms.EXPORT_HISTORY_INDEX)[0]) for s in check}
    targets = {s: e.export(s, ms.EXPORT_TARGETS) for s in check}
    assert targets[0].tolist() == [(2 * q + 1) * D // (2 * P) for q in range(P)]
    for b in range(blocks):
        e.process_blocks(x[b][np.arange(S) % x.shape[1]], use_graph=b % 2 == 0)
        for s in check:
            X = e.export(s, ms.EXPORT_INPUT_SPEC)
            G = rx.real_gcc(X, E)
            tau = targets[s]
            C = np.zeros((nT, D, K), np.float32)
            C[:, tau, :] = rx.atoms(np.ascontiguousarray(G[:, tau, :]), W)       # each output is its own chain: rows are independent
            masks, values = rs.source_masks(C, tau)
            assert np.array_equal(e.export(s, ms.EXPORT_TARGET_VALUES), values, equal_nan=True), (b, s)
            assert np.array_equal(e.export(s, ms.EXPORT_SOURCE_MASKS), masks), (b, s)
            assert np.array_equal(e.export(s, ms.EXPORT_ATOM_MASK), masks[0]), (b, s)
            hist[s], index[s], targets[s], status = rs.localize_sources(hist[s], index[s], e.export(s, ms.EXPORT_GCCPHAT), 6, True, tau, P)
            assert np.array_equal(e.export(s, ms.EXPORT_HISTORY), hist[s], equal_nan=True), (b, s)
            assert int(e.export(s, ms.EXPORT_HISTORY_INDEX)[0]) == index[s]
            assert e.export(s, ms.EXPORT_TARGETS).tolist() == targets[s].tolist(), (b, s)
            if status:
                assert int(e.export(s, ms.EXPORT_STATUS)[0]) & ms.STATUS_FEW_PEAKS
    e.close()


# ------------------------------------------------------------------------------------------------ 2: source == single-target slot
@pytest.mark.parametrize('inference', [0, 3])
@pytest.mark.parametrize('nT', [1, 2])
def test_each_source_is_a_single_target_slot(golden, nT, inference):
    """Source q's output blocks and spectra == slot q of a MultiStreamRealtimeEngine (P slots, the same input in each) fed the
    exported masks of source q block by block, over 64 blocks with the localisation moving the targets."""
    from gcc_nmf_b200.realtime import multistream as ms
    g = golden('realtime_mini')
    W, E, win, N = _consts(g)
    hop, P, blocks = N // 4, 3, 64
    B = nT * hop
    x = _audio(1, B, blocks, seed=3)
    sep = _sep(W, E, win, hop, B, nT, 1, P, inference)
    ref = ms.MultiStreamRealtimeEngine(W, E, win, win, hop, B, nT, P, numInferenceIterations=inference)
    moved = set()
    for b in range(blocks):
        y = sep.process_blocks(x[b], use_graph=b % 2 == 0).copy()
        masks = sep.export(0, ms.EXPORT_SOURCE_MASKS)
        moved.add(tuple(sep.export(0, ms.EXPORT_TARGETS)))
        yr = ref.process_blocks(np.repeat(x[b], P, axis=0), forcedAtomMask=masks).copy()
        assert np.array_equal(y[0], yr), (b, float(np.abs(y[0] - yr).max()))
        spec = sep.export(0, ms.EXPORT_SOURCE_SPECS)
        for q in range(P):
            assert np.array_equal(spec[q], ref.export(q, ms.EXPORT_OUTPUT_SPEC)), (b, q)
    assert len(moved) > 1                    # the localisation changed the targets during the run
    sep.close()
    ref.close()


# ------------------------------------------------------------------------------------------------ 3: the sources sum to the mixture path
@pytest.mark.parametrize('inference', [0, 4])
def test_sources_sum_to_separation_off_output(golden, inference):
    from gcc_nmf_b200.realtime import multistream as ms
    g = golden('realtime_mini')
    W, E, win, N = _consts(g)
    hop, nT, P, blocks = N // 4, 2, 4, 24
    B = nT * hop
    x = _audio(1, B, blocks, seed=11)
    sep = _sep(W, E, win, hop, B, nT, 1, P, inference)
    off = ms.MultiStreamRealtimeEngine(W, E, win, win, hop, B, nT, 1, numInferenceIterations=inference)
    off.set_params(0, separationEnabled=False)
    worst = 0.0
    for b in range(blocks):
        y = sep.process_blocks(x[b], use_graph=b % 2 == 0).copy()
        yo = off.process_blocks(x[b]).copy()
        if b < 2:                             # the two blocks of latency emit nothing but the rings' rounding residue
            continue
        peak = float(np.abs(yo).max())
        worst = max(worst, float(np.abs(y[0].astype(np.float64).sum(axis=0) - yo).max()) / peak)
    print('sum of %d sources vs separation off (inference %d): %.2e of the block peak' % (P, inference, worst))
    assert worst < 1e-6, worst
    sep.close()
    off.close()


# ------------------------------------------------------------------------------------------------ 4: streams x sources
def _one_slot(W, E, win, hop, B, nT, P, inference, params):
    return _sep(W, E, win, hop, B, nT, 1, P, inference, params)


def _same(multi, single, s, y, ys, what):
    from gcc_nmf_b200.realtime import multistream as ms
    assert np.array_equal(y, ys), (what, s)
    for item in range(14):
        a, b = multi.export(s, item), single.export(0, item)
        assert np.array_equal(a, b, equal_nan=a.dtype.kind in 'fc'), (what, s, item)
    assert ms.EXPORT_STATUS == 13


@pytest.mark.parametrize('inference', [0, 2])
def test_slots_equal_one_slot_engines_with_lifecycle(golden, inference):
    """S = 5 heterogeneous slots == five one-slot engines, with set_targets, a slot switched off and on, and a reset between
    graph launches."""
    g = golden('realtime_mini')
    W, E, win, N = _consts(g)
    hop, nT, S, P, blocks = N // 4, 2, 5, 3, 16
    B = nT * hop
    x = _audio(S, B, blocks, seed=2)
    multi = _sep(W, E, win, hop, B, nT, S, P, inference)
    singles = []
    for s in range(S):
        multi.set_params(s, **SLOT_PARAMS[s])
        singles.append(_one_slot(W, E, win, hop, B, nT, P, inference, SLOT_PARAMS[s]))
    graph = multi.build_graph().value
    for b in range(blocks):
        if b == 3:
            multi.set_targets([1, 2], [[4, 20, -1], [30, 1, 17]])
            singles[1].set_targets(0, [4, 20, -1])
            singles[2].set_targets(0, [30, 1, 17])
        if b == 6:
            multi.set_active(3, False)
        if b == 9:
            multi.set_active(3, True)
        if b == 11:
            multi.reset_slots(4)
            multi.set_params(4, **SLOT_PARAMS[4])
            singles[4].close()
            singles[4] = _one_slot(W, E, win, hop, B, nT, P, inference, SLOT_PARAMS[4])
        y = multi.process_blocks(x[b]).copy()
        assert multi.build_graph().value == graph
        for s in range(S):
            if s == 3 and 6 <= b < 9:
                assert not y[s].any()
                continue
            _same(multi, singles[s], s, y[s], singles[s].process_blocks(x[b][s:s + 1], use_graph=b % 2 == 0)[0], 'block %d' % b)


def test_many_slots_wide_tile(golden):
    """S = 141 slots on the 128 x 128 atoms tile (K = 200: a partial atom tile, D = 20: padded TDOA rows), sampled slots against
    one-slot engines, one slot inactive."""
    g = golden('realtime_mini')
    W, E, win, N = _consts(g, K=200, D=20, seed=4)
    hop, nT, S, P, blocks = N // 4, 2, 141, 4, 5
    B = nT * hop
    x = _audio(S, B, blocks, seed=6)
    multi = _sep(W, E, win, hop, B, nT, S, P, 2)
    multi.set_active(70, False)
    check = [0, 1, 71, S - 1]
    singles = {s: _one_slot(W, E, win, hop, B, nT, P, 2, SLOT_PARAMS[0]) for s in check}
    for b in range(blocks):
        y = multi.process_blocks(x[b]).copy()
        assert not y[70].any()
        for s in check:
            _same(multi, singles[s], s, y[s], singles[s].process_blocks(x[b][s:s + 1])[0], 'block %d' % b)


# ------------------------------------------------------------------------------------------------ 5: edge cases
def test_duplicate_targets_lower_source_wins(golden):
    from gcc_nmf_b200.realtime import multistream as ms
    g = golden('realtime_mini')
    W, E, win, N = _consts(g)
    hop, nT, P = N // 4, 1, 3
    e = _sep(W, E, win, hop, hop, nT, 1, P, 0, dict(localizationEnabled=False))
    e.set_targets(0, [5, 5, 20])
    x = _audio(1, hop, 6, seed=8)
    for b in range(6):
        y = e.process_blocks(x[b], use_graph=b % 2 == 0)
        m = e.export(0, ms.EXPORT_SOURCE_MASKS)
        v = e.export(0, ms.EXPORT_TARGET_VALUES)
        assert not m[1].any() and not y[0, 1].any()
        assert np.array_equal(v[0], v[1])
        assert np.array_equal(m[0] + m[2], np.ones_like(m[0]))


def test_digital_silence_goes_to_source_zero(golden):
    from gcc_nmf_b200.realtime import multistream as ms
    from oracle import rt_sources as rs
    g = golden('realtime_mini')
    W, E, win, N = _consts(g)
    hop, nT, P = N // 4, 2, 3
    B = nT * hop
    e = _sep(W, E, win, hop, B, nT, 1, P, 0)
    targets = e.export(0, ms.EXPORT_TARGETS)
    for b in range(12):                       # after 8 silent blocks the rings hold nothing but zeros
        y = e.process_blocks(np.zeros((1, 2, B), np.float32), use_graph=b % 2 == 0)
        v = e.export(0, ms.EXPORT_TARGET_VALUES)
        C = np.full((nT, int(E.shape[1]), W.shape[1]), np.nan, np.float32)
        C[:, targets, :] = v.transpose(2, 0, 1)
        masks, _ = rs.source_masks(C, targets)
        assert np.array_equal(e.export(0, ms.EXPORT_SOURCE_MASKS), masks)
        if b >= 8:
            assert np.isnan(v).all() and (masks[0] == 1).all()
            assert not np.any(y[0, 1:])       # sources 1 .. P-1 own no atom
        targets = e.export(0, ms.EXPORT_TARGETS)
    # the all-NaN mean has no peak: the targets stay and the status says so
    assert int(e.export(0, ms.EXPORT_STATUS)[0]) & ms.STATUS_FEW_PEAKS


def test_mono_input_on_mirrored_tdoas_ties_to_the_lower_source(golden):
    from gcc_nmf_b200.realtime import multistream as ms
    g = golden('realtime_mini')
    W, E, win, N = _consts(g, mirrored=True)
    D = E.shape[1]
    hop, nT, P = N // 4, 1, 2
    e = _sep(W, E, win, hop, hop, nT, 1, P, 0, dict(localizationEnabled=False))
    e.set_targets(0, [D - 4, 3])                # mirrored pair: identical GCC rows for a mono input
    x = _audio(1, hop, 6, seed=12)
    x[:, :, 1] = x[:, :, 0]
    for b in range(6):
        e.process_blocks(x[b], use_graph=b % 2 == 0)
        v = e.export(0, ms.EXPORT_TARGET_VALUES)
        assert np.array_equal(v[0], v[1], equal_nan=True)
        assert (e.export(0, ms.EXPORT_SOURCE_MASKS)[0] == 1).all()


def test_fewer_peaks_than_sources_keeps_targets(golden):
    """D = 16 has at most 7 strict interior maxima: with P = 8 the localisation never finds enough peaks."""
    from gcc_nmf_b200.realtime import multistream as ms
    g = golden('realtime_mini')
    W, E, win, N = _consts(g, D=16)
    hop, nT, P = N // 4, 1, 8
    e = _sep(W, E, win, hop, hop, nT, 1, P, 0)
    first = e.export(0, ms.EXPORT_TARGETS)
    assert int(e.export(0, ms.EXPORT_STATUS)[0]) == 0
    x = _audio(1, hop, 4, seed=1)
    for b in range(4):
        e.process_blocks(x[b], use_graph=b % 2 == 0)
        assert np.array_equal(e.export(0, ms.EXPORT_TARGETS), first)
        assert int(e.export(0, ms.EXPORT_STATUS)[0]) == ms.STATUS_FEW_PEAKS
    e.reset_slots(0)
    assert int(e.export(0, ms.EXPORT_STATUS)[0]) == 0


def test_invalid_arguments_fail_before_enqueue(golden):
    from gcc_nmf_b200 import _lib
    g = golden('realtime_mini')
    W, E, win, N = _consts(g)
    e = _sep(W, E, win, N // 4, N // 4, 1, 2, 3, 0)
    D = E.shape[1]
    with pytest.raises(_lib.ParameterError):
        e.set_targets(0, [0, D, 1])
    with pytest.raises(_lib.ParameterError):
        e.set_targets(1, [0, -2, 1])
    with pytest.raises(ValueError):
        e.process_blocks(np.zeros((2, 2, N // 4), np.float32), forcedAtomMask=np.ones((2, W.shape[1], 1)))
    W2, E2, win2, _ = _consts(g, D=2)
    e2 = _sep(W2, E2, win2, N // 4, N // 4, 1, 1, 2, 0, dict(localizationEnabled=False))
    with pytest.raises(_lib.ParameterError):
        e2.set_params(0, localizationEnabled=True)


# ------------------------------------------------------------------------------------------------ 6: drop-in processor and runner
def _processor(g, W, nT, P, localize=True):
    from gcc_nmf_b200.realtime.gccNMFProcessor import TARGET_MODE_MULTIPLE, GCCNMFProcessor
    from gcc_nmf_b200.realtime.utils import CircularBuffer
    sr, N, K, D = [int(v) for v in g['params']]
    hist = CircularBuffer((D, 128)) if localize else None
    tdoa = CircularBuffer((1, 128)) if localize else None
    p = GCCNMFProcessor(sr, N, nT, {'Pretrained': {K: W}}, 'Pretrained', K, 0, float(g['micSep']), localize, 6, gccPHATHistory=hist,
                        tdoaHistory=tdoa)
    p.numTDOAs = D
    p.targetMode = TARGET_MODE_MULTIPLE
    p.numSources = P
    p.reset()
    return p


def test_processor_multiple_mode(golden):
    """processBlock / processFrames in TARGET_MODE_MULTIPLE == a one-slot engine with sources; targetTDOAIndexes mirrors the
    device and setTargetTDOAIndexes reaches it."""
    from gcc_nmf_b200.realtime import multistream as ms
    g = golden('realtime_mini')
    W, E, win, N = _consts(g)
    hop, nT, P = N // 4, 2, 3
    B = nT * hop
    proc = _processor(g, g['W'], nT, P)
    eng = _sep(W, E, win, hop, B, nT, 1, P, 0, dict(epsilon=2.0, localizationEnabled=True, localizationWindowSize=6))
    x = _audio(1, B, 20, seed=5)
    for b in range(20):
        if b == 7:
            proc.setTargetTDOAIndexes([2, 15, 29])
            eng.set_targets(0, [2, 15, 29])
        y = proc.processBlock(x[b][0], hop, B)
        assert y.shape == (P, 2, B)
        assert np.array_equal(y, eng.process_blocks(x[b])[0]), b
        assert list(proc.targetTDOAIndexes) == eng.export(0, ms.EXPORT_TARGETS).tolist()
    fr = _processor(g, g['W'], nT, P, localize=False)
    frames = (np.random.default_rng(0).standard_normal((2, N, nT)) * win[None, :, None]).astype(np.float32)
    assert fr.processFrames(frames).shape == (P, 2, N, nT)


def test_headless_runner_sources_sum_to_separation_off(golden, tmp_path):
    from scipy.io import wavfile
    from gcc_nmf_b200.realtime.runRealtimeGCCNMF import RealtimeGCCNMFNoGUI, getGCCNMFConfigParams, pcm2float
    import os
    g = golden('realtime_mini')
    sr, N, K, D = [int(v) for v in g['params']]
    hop, B, nT = [int(v) for v in g['ola_params']]
    wav = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'dev1_female3_liverec_130ms_1m_mix.wav')

    def params(P):
        return getGCCNMFConfigParams(wav, dictionariesW={'Pretrained': {K: g['W']}}, windowSize=N, hopSize=hop, blockSize=B, numTDOAs=D,
                                     dictionarySize=K, dictionarySizes=[K], sampleRate=sr, numSources=P)
    paths = [str(tmp_path / ('source%d.wav' % q)) for q in range(3)]
    srcs = RealtimeGCCNMFNoGUI(params=params(3)).run(paths)
    off_runner = RealtimeGCCNMFNoGUI(params=params(0))
    off_runner.gccNMFProcessor.separationEnabled = False
    off = off_runner.run(str(tmp_path / 'off.wav'))
    assert srcs.shape == (3,) + off.shape
    peak = float(np.abs(off).max())
    err = float(np.abs(srcs.astype(np.float64).sum(axis=0) - off).max()) / peak
    print('runner: 3 sources vs separation off: %.2e of the peak' % err)
    assert err < 1e-5, err
    files = np.stack([pcm2float(wavfile.read(p)[1]).T for p in paths])
    assert files.shape == srcs.shape
    assert float(np.abs(files.sum(axis=0) - pcm2float(wavfile.read(str(tmp_path / 'off.wav'))[1]).T).max()) <= 4 / 32768.0
