"""GPU: many independent audio streams in one real-time engine (MultiStreamRealtimeEngine, gccnmf_rtm_*).  Slot s must be
bit-identical to a single-stream RealtimeEngine fed the same blocks with the same parameters: every output block, every export
item and the target index, with and without a graph, with and without inference, through activation changes and slot resets.
The reference fixture (realtime_mini) must pass through a slot exactly as through a single engine."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

EXPORTS = range(9)


def _consts(g, K=None, D=None, seed=0):
    """W, expJOmegaTau and the window of realtime_mini (GCCNMFProcessor.buildConstants), or a random W of K atoms and D TDOAs."""
    from gcc_nmf_b200 import gccNMFFunctions as fn
    sr, N, K0, D0 = [int(v) for v in g['params']]
    W = g['W'] if K is None else (np.random.default_rng(seed).random((N // 2 + 1, K)) ** 3).astype(np.float32)
    D = D0 if D is None else D
    freq = np.linspace(0, sr / 2, N // 2 + 1).astype(np.float32)
    maxT = float(g['micSep']) / fn.SPEED_OF_SOUND_IN_METRES_PER_SECOND
    tdoas = np.linspace(-maxT, maxT, D).astype(np.float32)
    E = np.exp(np.outer(freq, -(2j * np.pi) * tdoas)).astype(np.complex64)
    win = np.sqrt(np.hamming(N).astype(np.float32))
    return W, E, win, N


# heterogeneous slot parameters: window / boxcar, separation off, localisation on for some, a noise floor
SLOT_PARAMS = [
    dict(targetTDOAIndex=9.6, epsilon=5.0, beta=2.0, noiseFloor=0.0, mode=1, separationEnabled=True, localizationEnabled=True, localizationWindowSize=6),
    dict(targetTDOAIndex=3.0, epsilon=2.0, beta=1.0, noiseFloor=0.0, mode=0, separationEnabled=True, localizationEnabled=False, localizationWindowSize=6),
    dict(targetTDOAIndex=5.0, epsilon=2.0, beta=1.0, noiseFloor=0.0, mode=1, separationEnabled=False, localizationEnabled=True, localizationWindowSize=4),
    dict(targetTDOAIndex=12.0, epsilon=3.0, beta=1.0, noiseFloor=0.1, mode=1, separationEnabled=True, localizationEnabled=True, localizationWindowSize=3),
    dict(targetTDOAIndex=7.0, epsilon=4.0, beta=1.0, noiseFloor=0.0, mode=0, separationEnabled=True, localizationEnabled=True, localizationWindowSize=10),
]


def _params(s):
    return SLOT_PARAMS[s % len(SLOT_PARAMS)]


def _audio(S, B, blocks, seed=0):
    """(blocks, S, 2, B) float32: a different synthetic two-source mixture per slot."""
    from gcc_nmf_b200.synth import synthetic_stereo
    n = blocks * B
    x = np.stack([synthetic_stereo(n / 16000.0 + 0.01, seed=seed + 17 * s)[:, :n] for s in range(S)])
    return np.ascontiguousarray(x.reshape(S, 2, blocks, B).transpose(2, 0, 1, 3))


def _engines(W, E, win, hop, B, nT, S, inference, slots):
    from gcc_nmf_b200.realtime.engine import RealtimeEngine
    from gcc_nmf_b200.realtime.multistream import MultiStreamRealtimeEngine
    multi = MultiStreamRealtimeEngine(W, E, win, win, hop, B, nT, S, numInferenceIterations=inference)
    multi.set_params(range(S), **{k: [_params(s)[k] for s in range(S)] for k in SLOT_PARAMS[0]})
    singles = {}
    for s in slots:
        e = RealtimeEngine(W, E, win, win, hop, B, nT, numInferenceIterations=inference)
        e.set_params(**_params(s))
        singles[s] = e
    return multi, singles


def _assert_same(multi, single, s, out_m, out_s, what='block'):
    assert np.array_equal(out_m, out_s), (what, s, float(np.abs(out_m - out_s).max()))
    for item in EXPORTS:
        a, b = multi.export(s, item), single.export(item)
        assert a.dtype == b.dtype and a.shape == b.shape
        assert np.array_equal(a, b, equal_nan=a.dtype.kind in 'fc'), (what, s, item)


@pytest.mark.parametrize('nT', [1, 4])
@pytest.mark.parametrize('inference', [0, 3])
@pytest.mark.parametrize('use_graph', [True, False])
def test_slots_bit_identical_to_single_engines(golden, nT, inference, use_graph):
    g = golden('realtime_mini')
    W, E, win, N = _consts(g)
    hop, S, blocks = N // 4, 5, 10
    B = nT * hop
    x = _audio(S, B, blocks)
    multi, singles = _engines(W, E, win, hop, B, nT, S, inference, range(S))
    for b in range(blocks):
        y = multi.process_blocks(x[b], use_graph=use_graph).copy()
        for s in range(S):
            _assert_same(multi, singles[s], s, y[s], singles[s].process_block(x[b, s], use_graph=use_graph), 'block %d' % b)


@pytest.mark.parametrize('nT', [1, 4])
@pytest.mark.parametrize('inference', [0, 2])
def test_process_frames_slots_bit_identical(golden, nT, inference):
    """processFrames entry (caller-cut windowed frames), with forced atom masks on every other call."""
    g = golden('realtime_mini')
    W, E, win, N = _consts(g)
    K, S = W.shape[1], 5
    multi, singles = _engines(W, E, win, N // 4, nT * N // 4, nT, S, inference, range(S))
    rng = np.random.default_rng(3)
    for b in range(8):
        frames = (rng.standard_normal((S, 2, N, nT)) * win[None, None, :, None]).astype(np.float32)
        forced = (rng.random((S, K, nT)) < 0.5).astype(np.float64) if b % 2 else None
        y = multi.process_frames(frames, forcedAtomMask=forced).copy()
        for s in range(S):
            ys = singles[s].process_frames(frames[s], forcedAtomMask=None if forced is None else forced[s])
            _assert_same(multi, singles[s], s, y[s], ys, 'frames %d' % b)


@pytest.mark.parametrize('D,nT,K,S,inference', [(64, 1, 256, 160, 2), (20, 2, 200, 141, 2), (20, 2, 200, 141, 0)])
def test_many_slots_wide_tile_bit_identical(golden, D, nT, K, S, inference):
    """Enough (slot, frame) rows for the 128 x 128 atoms tile (K / 128 x rows / 128 CTAs fill the H100) and for several slots per
    warp in the inference and filter kernels (the last slot group partial): sampled slots against single engines, with one slot
    inactive (zeros out) and padded TDOA rows (D = 20) / a partial atom tile (K = 200)."""
    g = golden('realtime_mini')
    W, E, win, N = _consts(g, K=K, D=D, seed=D)
    hop = N // 4
    B = nT * hop
    check = [0, 1, S // 2 + 1, S - 1]
    blocks = 6
    x = _audio(S, B, blocks, seed=5)
    multi, singles = _engines(W, E, win, hop, B, nT, S, inference, check)
    multi.set_active(S // 2, False)
    for b in range(blocks):
        y = multi.process_blocks(x[b]).copy()
        assert not y[S // 2].any()
        for s in check:
            _assert_same(multi, singles[s], s, y[s], singles[s].process_block(x[b, s]), 'block %d' % b)


def test_lifecycle_reset_and_deactivate_under_one_graph(golden):
    """reset_slots mid-run == a fresh single engine from that block on; a slot inactive for k blocks outputs zeros and then
    continues as a single engine that never saw those blocks; the other slots are undisturbed.  One graph throughout."""
    from gcc_nmf_b200.realtime.engine import RealtimeEngine
    g = golden('realtime_mini')
    W, E, win, N = _consts(g)
    hop, nT, S, blocks = N // 4, 2, 4, 20
    B = nT * hop
    x = _audio(S, B, blocks, seed=9)
    multi, singles = _engines(W, E, win, hop, B, nT, S, 0, range(S))
    graph = multi.build_graph().value
    reset_at, off = 6, range(8, 12)
    for b in range(blocks):
        if b == reset_at:
            multi.reset_slots(1)
            multi.set_params(1, **_params(1))
            singles[1] = RealtimeEngine(W, E, win, win, hop, B, nT)
            singles[1].set_params(**_params(1))
        if b == off[0]:
            multi.set_active(2, False)
        if b == off[-1] + 1:
            multi.set_active(2, True)
        blk = x[b].copy()
        if b in off:
            blk[2] = 1e3 * np.random.default_rng(b).standard_normal((2, B))     # ignored while inactive
        y = multi.process_blocks(blk).copy()
        assert multi.build_graph().value == graph
        for s in range(S):
            if s == 2 and b in off:
                assert not y[s].any()
                continue
            _assert_same(multi, singles[s], s, y[s], singles[s].process_block(x[b, s]), 'block %d' % b)


@pytest.mark.parametrize('use_graph', [True, False])
def test_reference_fixture_through_a_slot(golden, use_graph):
    """realtime_mini's overlap-add sequence in slot 2 of 4 (the other slots get other audio) meets the assertions of the
    single-stream ring test: per-block target decisions, teacher-forced and free-running error."""
    from gcc_nmf_b200.realtime.multistream import MultiStreamRealtimeEngine
    g = golden('realtime_mini')
    W, E, win, N = _consts(g)
    hop, B, nT = [int(v) for v in g['ola_params']]
    x, ref = g['ola_x'], g['ola_out']
    K, S, slot, nb = W.shape[1], 4, 2, x.shape[1] // B
    scale = float(np.abs(ref).max())
    others = _audio(S, B, nb, seed=21)
    fixture = dict(targetTDOAIndex=9.60, epsilon=5.0, beta=2.0, noiseFloor=0.0, mode=1, separationEnabled=True, localizationEnabled=True,
                   localizationWindowSize=6)

    def run(forced):
        e = MultiStreamRealtimeEngine(W, E, win, win, hop, B, nT, S)
        e.set_params(range(S), **{k: [fixture[k] if s == slot else _params(s)[k] for s in range(S)] for k in fixture})
        out = np.zeros_like(ref)
        for b in range(nb):
            blk = others[b].copy()
            blk[slot] = x[:, b * B:(b + 1) * B]
            m = None
            if forced:
                m = np.ones((S, K, nT))
                m[slot] = g['ola_hmask'][b]
            out[:, b * B:(b + 1) * B] = e.process_blocks(blk, use_graph=use_graph and not forced, forcedAtomMask=m)[slot]
            if not forced:
                assert float(e.export(slot, 1)[0]) == g['ola_target'][b]
        return out
    free = float(np.abs(run(False) - ref).max() / scale)
    tf = float(np.abs(run(True) - ref).max() / scale)
    print('fixture through slot %d of %d (graph=%s): free-running %.2e, teacher-forced %.2e' % (slot, S, use_graph, free, tf))
    assert tf < 1e-5, tf
    assert free < 5e-3, free


@pytest.mark.parametrize('S', [1, 64])
@pytest.mark.parametrize('inference', [0, 2])
def test_kernel_launches_per_block(golden, S, inference):
    g = golden('realtime_mini')
    W, E, win, N = _consts(g)
    hop, nT = N // 4, 1
    B = nT * hop
    multi, _ = _engines(W, E, win, hop, B, nT, S, inference, [])
    x = _audio(S, B, 3)
    h = multi.h
    n0 = h.launches
    multi.process_blocks(x[0], use_graph=False)
    assert h.launches - n0 == 5 + 2 * inference
    multi.build_graph()
    n1 = h.launches
    multi.process_blocks(x[1])
    multi.process_blocks(x[2])
    assert h.launches - n1 == 2


def test_headless_runner_many_files(golden, tmp_path):
    """runMany: two wav files of different lengths as two slots of one engine == two single `run` calls (arrays and int16 files)."""
    from scipy.io import wavfile
    from gcc_nmf_b200.realtime.runRealtimeGCCNMF import RealtimeGCCNMFNoGUI, float2pcm, getGCCNMFConfigParams
    from gcc_nmf_b200.synth import synthetic_stereo
    g = golden('realtime_mini')
    sr, N, K, D = [int(v) for v in g['params']]
    hop, B, nT = [int(v) for v in g['ola_params']]
    clips = [g['ola_x'], synthetic_stereo(0.23, seed=4)]
    srcs = [str(tmp_path / ('in%d.wav' % i)) for i in range(2)]
    for p, c in zip(srcs, clips):
        wavfile.write(p, sr, float2pcm(np.ascontiguousarray(c.T)))

    def params(path):
        return getGCCNMFConfigParams(path, dictionariesW={'Pretrained': {K: g['W']}}, windowSize=N, hopSize=hop, blockSize=B, numTDOAs=D,
                                     dictionarySize=K, dictionarySizes=[K], sampleRate=sr)
    single = []
    for i, p in enumerate(srcs):
        single.append(RealtimeGCCNMFNoGUI(params=params(p)).run(str(tmp_path / ('single%d.wav' % i))))
    many = RealtimeGCCNMFNoGUI(params=params(None)).runMany(srcs, [str(tmp_path / ('many%d.wav' % i)) for i in range(2)])
    assert len(many) == 2
    for i in range(2):
        assert many[i].shape == single[i].shape
        assert np.array_equal(many[i], single[i]), i
        assert open(str(tmp_path / ('many%d.wav' % i)), 'rb').read() == open(str(tmp_path / ('single%d.wav' % i)), 'rb').read()
