"""GPU: gccnmf_klnmf_batched -- B clips of one shape in one call -- against gccnmf_klnmf run on each clip alone, NaN-equal bit for
bit: ragged shapes, every batch size class, both numerator forms, every schedule option, strided V read in place, silent frames,
a NaN-filled workspace, the float32 SIMT shapes and the refusals; then performKLNMFBatch and the pipeline's batch flows against
their single-clip counterparts."""
import ctypes

import numpy as np
import pytest

from test_gpu_klnmf import DEFAULT_OPTIONS, NEUTRAL, options, tile_plan

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def h():
    from gcc_nmf_b200._lib import default_handle
    hd = default_handle()
    yield hd
    for name, value in DEFAULT_OPTIONS.items():
        hd.set_option(name, value)


@pytest.fixture(scope='module')
def sm_count(h):
    import torch
    return torch.cuda.get_device_properties(h.device).multi_processor_count


def inputs(h, B, F, T2, K, seed=0, ld=None):
    """B distinct V clips (as a (B, F, T2) view whose rows sit `ld` apart when given: clip b at column b * T2 of an (F, B * T2)
    matrix, the layout h.stft leaves), one seeded W0, H0 per clip."""
    import torch
    rng = np.random.default_rng(seed)
    V = (rng.random((B, F, T2)) ** 3 + 1e-3).astype(np.float32)
    if ld == 'stft':
        flat = h.to_device(np.ascontiguousarray(V.transpose(1, 0, 2).reshape(F, B * T2)))
        Vd = flat.view(F, B, T2).permute(1, 0, 2)
    else:
        Vd = h.to_device(V)
    W0 = torch.from_numpy((rng.random((B, F, K)) + 0.1).astype(np.float32))
    H0 = torch.from_numpy((rng.random((B, K, T2)) + 0.1).astype(np.float32))
    return Vd, W0, H0


def solo(h, V, W0, H0, iters, alpha, eps, update_W):
    Ws, Hs = [], []
    for b in range(V.shape[0]):
        W, H = h.to_device(W0[b]), h.to_device(H0[b])
        h.klnmf(V[b].contiguous(), W, H, iters, alpha, eps, update_W=update_W)
        Ws.append(W)
        Hs.append(H)
    import torch
    return torch.stack(Ws), torch.stack(Hs)


def batched(h, V, W0, H0, iters, alpha, eps, update_W):
    W, H = h.to_device(W0), h.to_device(H0)
    h.klnmf_batched(V, W, H, iters, alpha, eps, update_W=update_W)
    return W, H


def nan_equal(a, b):
    import torch
    return bool(torch.all((a == b) | (torch.isnan(a) & torch.isnan(b))))


def assert_same(h, V, W0, H0, iters=5, alpha=0.1, eps=1e-16, update_W=True, what=''):
    W, H = batched(h, V, W0, H0, iters, alpha, eps, update_W)
    Ws, Hs = solo(h, V, W0, H0, iters, alpha, eps, update_W)
    for b in range(V.shape[0]):
        assert nan_equal(W[b], Ws[b]) and nan_equal(H[b], Hs[b]), (what, 'clip', b)
    return W, H


# (F, T2, K): ragged F (tail rows 1 and 8, a partial m tile, 16 m tiles + 1), 2T from 128 to 3744, K in {32, 40, 72, 128, 1024}
SHAPES = [(129, 128, 32), (136, 250, 40), (200, 622, 72), (513, 622, 128), (2049, 600, 128), (513, 3744, 1024)]
RUNS = [(1, 0.0, 1e-16, True), (5, 0.1, 1e-16, True), (5, 0.1, 1e-3, False)]


@pytest.mark.parametrize('shape', SHAPES, ids=lambda s: '%dx%dx%d' % s)
@pytest.mark.parametrize('B', [1, 2, 3, 7])
def test_batch_equals_solo(h, shape, B):
    F, T2, K = shape
    if K == 1024 and B > 3:
        pytest.skip('covered by test_batch_beyond_resident_clusters')
    assert h.klnmf_uses_tensor_cores(F, T2, K)
    V, W0, H0 = inputs(h, B, F, T2, K, seed=B)
    for iters, alpha, eps, update_W in RUNS:
        assert_same(h, V, W0, H0, iters, alpha, eps, update_W, what=(shape, B, iters, alpha, eps, update_W))


def test_numerator_with_k_splits_is_covered(h, sm_count):
    assert any(tile_plan(h, sm_count, *s)[3] >= 2 for s in SHAPES)


def test_batch_of_33_in_place_stft_layout(h):
    """B = 33 clips read in place from an (F, 33 T2) matrix (row pitch 33 T2, clip stride T2)."""
    V, W0, H0 = inputs(h, 33, 513, 622, 128, seed=33, ld='stft')
    assert V.stride() == (622, 33 * 622, 1)
    assert_same(h, V, W0, H0, 5, 0.1, 1e-16, True)


def test_batch_beyond_resident_clusters(h, sm_count):
    """K = 1024: the batch's k-split clusters outnumber what the device holds at once, where one clip's do not."""
    F, T2, K = 513, 1250, 1024
    plan = tile_plan(h, sm_count, F, T2, K)
    B = 9
    assert plan[3] >= 2 and B * plan[7] > sm_count, plan
    V, W0, H0 = inputs(h, B, F, T2, K, seed=5)
    for wcr in (1, 0):
        with options(h, w_cluster_reduce=wcr):
            assert_same(h, V, W0, H0, 3, 0.1, 1e-16, True, what=('w_cluster_reduce', wcr))


OPTIONS = NEUTRAL + [('w_cluster_reduce', 1), ('force_simt_nmf', 1), ('wh_split2', 1), ('wh_tile', 112)]


def test_every_option(h, sm_count):
    F, T2, K = 2049, 600, 128
    assert tile_plan(h, sm_count, F, T2, K)[3] >= 2
    for ld in (None, 'stft'):
        V, W0, H0 = inputs(h, 3, F, T2, K, seed=11, ld=ld)
        for opt in OPTIONS:
            kw = dict(opt) if isinstance(opt[0], tuple) else dict([opt])
            with options(h, **kw):
                assert_same(h, V, W0, H0, 3, 0.1, 1e-16, True, what=(kw, ld))


def test_silent_frame_stays_in_its_clip(h):
    """A silent frame makes W.H vanish there and the clip's ratios NaN: the clip matches its solo NaNs, the others stay finite."""
    import torch
    V, W0, H0 = inputs(h, 3, 513, 622, 128, seed=3)
    V[1, :, 100] = 0.0
    W, H = assert_same(h, V, W0, H0, 5, 0.0, 1e-16, True)
    assert not bool(torch.isfinite(H[1]).all()) or not bool(torch.isfinite(W[1]).all())
    for b in (0, 2):
        assert bool(torch.isfinite(W[b]).all()) and bool(torch.isfinite(H[b]).all())


def test_nan_filled_workspace(h):
    """Every workspace word the batch reads is written by it first."""
    B, F, T2, K = 3, 200, 622, 72
    V, W0, H0 = inputs(h, B, F, T2, K, seed=7)
    nbytes = h.lib.gccnmf_klnmf_batched_workspace_bytes(B, F, T2, K)
    h.workspace('klnmf_batched', nbytes).fill_(0xFF)            # all-ones words: float32 NaN
    assert_same(h, V, W0, H0, 5, 0.1, 1e-16, True)


@pytest.mark.parametrize('shape', [(64, 100, 20), (130, 100, 24), (513, 622, 36)], ids=lambda s: '%dx%dx%d' % s)
@pytest.mark.parametrize('ld', [None, 'stft'])
def test_simt_shapes(h, shape, ld):
    F, T2, K = shape
    assert not h.klnmf_uses_tensor_cores(F, T2, K)
    V, W0, H0 = inputs(h, 3, F, T2, K, seed=9, ld=ld)
    for iters, alpha, eps, update_W in RUNS:
        assert_same(h, V, W0, H0, iters, alpha, eps, update_W)


def test_workspace_is_b_times_single_clip(h):
    for F, T2, K in SHAPES:
        for B in (1, 3, 33):
            assert h.lib.gccnmf_klnmf_batched_workspace_bytes(B, F, T2, K) == B * h.lib.gccnmf_klnmf_workspace_bytes(F, T2, K)


def test_refusals(h):
    import torch
    from gcc_nmf_b200._lib import GCCNMF_OK
    lib, B, F, T2, K = h.lib, 2, 200, 622, 72
    V, W0, H0 = inputs(h, B, F, T2, K)
    W, H = h.to_device(W0), h.to_device(H0)
    nbytes = lib.gccnmf_klnmf_batched_workspace_bytes(B, F, T2, K)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=h.device)
    p = lambda t: t.data_ptr()

    def call(v=p(V), ld=T2, cs=F * T2, b=B, f=F, t2=T2, w=p(W), hh=p(H), k=K, it=3, wsp=p(ws), n=nbytes):
        return lib.gccnmf_klnmf_batched(h.h, v, ld, cs, b, f, t2, w, hh, k, it, 0.0, 1e-16, 1, wsp, n, h.stream)
    before = h.launches
    bad = [dict(b=0), dict(b=-1), dict(b=8192), dict(v=None), dict(w=None), dict(hh=None), dict(f=0), dict(t2=-1), dict(k=0),
           dict(ld=T2 - 1), dict(cs=-1), dict(it=-1), dict(wsp=None), dict(n=nbytes - 1)]
    for kw in bad:
        assert call(**kw) != GCCNMF_OK, kw
    assert h.launches == before                 # refused before anything was enqueued
    assert lib.gccnmf_klnmf_batched_workspace_bytes(0, F, T2, K) == 0
    assert call(it=0) == GCCNMF_OK and h.launches == before
    assert call() == GCCNMF_OK
    from gcc_nmf_b200._lib import ParameterError
    with pytest.raises(ParameterError):
        h.klnmf_batched(V, W[:, :, :8], H, 1)
    with pytest.raises(ParameterError):
        h.klnmf_batched(V.transpose(1, 2), W, H, 1)


def test_perform_klnmf_batch(h):
    from gcc_nmf_b200 import gccNMFFunctions as fn
    rng = np.random.default_rng(1)
    Vs = (rng.random((3, 513, 622)) ** 3 + 1e-3).astype(np.float32)
    W, H = fn.performKLNMFBatch(Vs, 128, 10, 0.1)
    for b in range(3):
        Wb, Hb = fn.performKLNMF(Vs[b], 128, 10, 0.1)
        assert np.array_equal(W[b], Wb, equal_nan=True) and np.array_equal(H[b], Hb, equal_nan=True)


def clips_c1():
    """The shipped recording's first 10 s and two synthetic clips of the same length (configs[0]: 16 kHz, 10 s)."""
    import os
    from gcc_nmf_b200.synth import synthetic_stereo
    from gcc_nmf_b200.wavio import wavread
    here = os.path.dirname(os.path.abspath(__file__))
    rec, sr = wavread(os.path.join(here, 'golden', 'dev1_female3_liverec_130ms_1m_mix.wav'))
    n = 10 * sr
    rec = np.ascontiguousarray(np.asarray(rec, dtype=np.float32)[:2, :n])
    return sr, np.stack([rec, synthetic_stereo(10.0, sr, seed=21), synthetic_stereo(10.0, sr, seed=22, num_sources=3)])


SIGNAL_KEYS = ['W', 'H', 'V', 'X', 'coherence', 'angularSpectrogram', 'meanAngularSpectrum', 'targetCoefficientMasks',
               'targetSpectrogramEstimates', 'targetSignalEstimates']


def _equal(a, b):
    import torch
    if a.is_complex():
        return torch.equal(torch.view_as_real(a), torch.view_as_real(b))
    if a.is_floating_point():
        return nan_equal(a, b)
    return torch.equal(a, b)


@pytest.mark.parametrize('flow', ['enhance', 'separate'])
def test_pipeline_batch_flows(h, flow):
    """configs[0] settings: N = 1024, hop = 512 (F = 513, 2T = 622), K = 128, 64 TDOAs, 100 iterations."""
    from gcc_nmf_b200.pipeline import GCCNMFPipeline
    sr, x = clips_c1()
    pipe = GCCNMFPipeline(sr, 1024, 512, 64, 1.0, 128, 100, handle=h)
    keep = lambda r: {k: (v.clone() if hasattr(v, 'clone') else v) for k, v in r.items()}     # results are views of reused buffers
    if flow == 'enhance':
        batch = [keep(r) for r in pipe.enhance_batch(h.to_device(x))]
        singles = [keep(pipe.enhance(h.to_device(x[b]))) for b in range(3)]
        extra = ['argMaxGCCNMF']
    else:
        batch = [keep(r) for r in pipe.separate_batch(h.to_device(x), 2)]
        singles = [keep(pipe.separate(h.to_device(x[b]), 2)) for b in range(3)]
        extra = ['targetTDOAGCCNMFs']
    assert len(batch) == 3
    for b in range(3):
        assert batch[b]['targetTDOAIndexes'] == singles[b]['targetTDOAIndexes'], b
        for k in SIGNAL_KEYS + extra:
            assert batch[b][k].shape == singles[b][k].shape and _equal(batch[b][k], singles[b][k]), (flow, b, k)
