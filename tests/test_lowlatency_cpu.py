"""CPU: the streaming schedule of the low-latency engine (oracle/ll_stream.py) against the notebook loop's fixture for every call
size, the latency formula and synthesis modes, the state-size carve and argument validation of the C ABI, and the header
against the bindings."""
import ctypes
import os
import re

import numpy as np
import pytest

from oracle import ll_stream as model

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _lib():
    from gcc_nmf_b200 import _lib
    try:
        return _lib.load_library()
    except ImportError:
        pytest.skip('library not built')


@pytest.mark.parametrize('tag', ['sym_', 'asym_'])
@pytest.mark.parametrize('schedule', [[1], [2], [3], [8], [1, 5, 8, 2, 3, 7]])
def test_schedule_model_equals_notebook_loop(golden, tag, schedule):
    """Fed the notebook's own frames (its Wiener filters on rfft(frame x window)), the streamed emit is the notebook's
    targetEstimateSamplesOLA delayed by the latency, bit for bit."""
    g = golden('lowlatency_mini')
    sr, N, hop, D, K, synth = [int(v) for v in g['params']]
    win = g['symmetricWindow'] if tag == 'sym_' else g['analysisWindow']
    wf = g[tag + 'wienerFilters']
    T = wf.shape[2]

    def frame_fn(frames, js):
        Xf = np.fft.rfft(frames * win, axis=-1)
        out = [np.fft.irfft(wf[:, :, j] * Xf[k], axis=-1) if j < T else np.full((2, N), np.nan) for k, j in enumerate(js)]
        return np.zeros((D, len(js))), np.stack(out)

    x = g['samples'][:, :g['samples'].shape[1] // hop * hop]
    y, _ = model.stream(x, N, hop, np.ones(N), hop / float(N) * 2, D, frame_fn, schedule)
    L = model.latency(np.ones(N), hop)
    assert L == -(-N // hop) * hop - hop
    assert not np.any(y[:, :L])
    assert np.array_equal(y[:, L:L + T * hop], g[tag + 'output'][:, :T * hop])


def test_schedule_model_carries_the_running_max():
    rng = np.random.RandomState(0)
    N, hop, D = 64, 16, 8
    ang = rng.standard_normal((D, 40))
    ang[3, 17] = np.nan

    def frame_fn(frames, js):
        return ang[:, js], np.zeros((len(js), 2, N))

    ref = None
    for sched in ([1], [4], [3, 1, 7]):
        _, t = model.stream(np.zeros((2, 43 * hop), np.float32), N, hop, np.ones(N), 1.0, D, frame_fn, sched)
        acc = np.maximum.accumulate(np.where(np.isnan(ang), np.inf, ang), axis=1)
        expect = [int(np.argmax(np.where(np.isinf(acc[:, j]) & np.isnan(ang[:, :j + 1]).any(axis=1), np.nan, acc[:, j]))) for j in range(40)]
        assert t == expect
        ref = t if ref is None else ref
        assert t == ref


def test_synthesis_modes_and_latency():
    from gcc_nmf_b200.lowlatency import batchArguments, latencyOf, synthesisWeights
    from gcc_nmf_b200.online import getAsymmetricSynthesisWindow
    N, m, hop = 1024, 64, 64
    syn = getAsymmetricSynthesisWindow(N, m, 0)
    gf = hop / float(N) * 2
    w, g = synthesisWeights('online', syn, hop)
    assert np.all(w == gf) and g == np.float32(1.0)
    w, g = synthesisWeights('lowlatency', syn, hop)
    assert np.all(w == 1) and g == np.float32(gf)
    assert latencyOf(w, hop) == N - hop
    w, g = synthesisWeights('windowed', syn, hop)
    assert np.array_equal(w, syn) and g == np.float32(gf)
    assert syn[N - 2 * m] == 0 and syn[N - 2 * m + 1] != 0          # the rising half starts at hanning's zero
    assert latencyOf(w, hop) == 2 * m - hop - 1 == 63
    assert latencyOf(np.ones(256), 24) == 264 - 24
    with pytest.raises(ValueError):
        synthesisWeights('other', syn, hop)
    with pytest.raises(ValueError):
        latencyOf(np.zeros(8), 2)
    assert batchArguments('windowed') == dict(gainPerFrame=False, applySynthesisWindow=True)


def _cfg(**kw):
    from gcc_nmf_b200._lib import LLConfig
    c = dict(window_size=1024, hop_size=64, hops_per_call=1, num_atoms=256, num_tdoas=128, num_streams=4, inference_iterations=0,
             sparsity_alpha=0.0, epsilon=1e-16)
    c.update(kw)
    return LLConfig(*[c[f] for f, _ in LLConfig._fields_])


def test_state_carve():
    lib = _lib()
    size = lambda **kw: lib.gccnmf_ll_state_bytes(ctypes.byref(_cfg(**kw)))      # noqa: E731
    sizes = [size(num_streams=s) for s in (1, 2, 3, 64, 1024, 4096)]
    assert all(a < b for a, b in zip(sizes, sizes[1:]))
    assert size(hops_per_call=8) > size(hops_per_call=1)
    assert size(inference_iterations=5) > size()
    N, hop, F, K, D, S = 1024, 64, 513, 256, 128, 4
    per_stream = 2 * (N - hop) * 4 + 2 * N * 4 + D * 8 + 2 * N * 4      # rings, carry, staging (C = 1) and one frame pair at least
    assert size(num_streams=S + 1) - size(num_streams=S) >= per_stream
    assert size() % 256 == 0


@pytest.mark.parametrize('bad', [dict(window_size=1000), dict(window_size=16), dict(hop_size=0), dict(hop_size=2048),
                                 dict(hops_per_call=0), dict(hops_per_call=65), dict(num_atoms=0), dict(num_tdoas=100),
                                 dict(num_tdoas=256), dict(num_tdoas=2), dict(num_streams=0), dict(num_streams=4097),
                                 dict(inference_iterations=-1), dict(num_atoms=60000, inference_iterations=5)])
def test_invalid_configurations(bad):
    lib = _lib()
    assert lib.gccnmf_ll_state_bytes(ctypes.byref(_cfg(**bad))) == 0


def test_valid_edges():
    lib = _lib()
    for ok in (dict(hop_size=24, window_size=256), dict(num_streams=4096), dict(hops_per_call=64, num_streams=1), dict(num_tdoas=4),
               dict(hop_size=1024), dict(num_atoms=60000), dict(num_atoms=57000, inference_iterations=5)):
        assert lib.gccnmf_ll_state_bytes(ctypes.byref(_cfg(**ok))) > 0, ok
    assert lib.gccnmf_ll_state_bytes(None) == 0


def test_header_agrees_with_bindings():
    from gcc_nmf_b200 import _lib
    header = open(os.path.join(ROOT, 'include', 'gccnmf_b200.h')).read()
    declared = set(re.findall(r'GCCNMF_API\s+[\w\s\*]+?\b(gccnmf_ll_\w+)\s*\(', header))
    bound = {n for n in _lib.SIGNATURES if n.startswith('gccnmf_ll_')}
    assert declared == bound and len(bound) == 7
    fields = re.search(r'typedef struct gccnmf_ll_config \{(.*?)\} gccnmf_ll_config;', header, re.S).group(1)
    names = re.findall(r'(?:int|float)\s+(\w+);', fields)
    assert names == [f for f, _ in _lib.LLConfig._fields_]
