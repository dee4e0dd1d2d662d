"""GPU: gccnmf_klnmf_ragged -- B clips of different lengths in one call -- against gccnmf_klnmf run on each clip alone, NaN-equal bit
for bit: lengths that share one tile width per contraction, lengths whose solo plans differ in every width and k-split count,
duplicate lengths, B = 1, B = 33 read in place, tensor-core and SIMT clips mixed, every run and schedule option, a NaN-filled
workspace, a silent frame, the launch count and the refusals; then performKLNMFBatch and the pipeline's batch flows on lists."""
import ctypes

import numpy as np
import pytest

from test_gpu_klnmf import DEFAULT_OPTIONS, options, tile_plan
from test_gpu_klnmf_batch import OPTIONS, RUNS, SIGNAL_KEYS, _equal, nan_equal

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


def inputs(h, F, T2s, K, seed=0, flat=False):
    """One V per clip (flat: column ranges of one (F, sum T2) device matrix, read in place), one seeded W0 (B, F, K) and H0 per clip."""
    import torch
    rng = np.random.default_rng(seed)
    Vh = [(rng.random((F, t)) ** 3 + 1e-3).astype(np.float32) for t in T2s]
    if flat:
        M = h.to_device(np.ascontiguousarray(np.concatenate(Vh, axis=1)))
        offs = np.cumsum([0] + list(T2s))
        Vs = [M[:, offs[b]:offs[b + 1]] for b in range(len(T2s))]
    else:
        Vs = [h.to_device(v) for v in Vh]
    W0 = torch.from_numpy((rng.random((len(T2s), F, K)) + 0.1).astype(np.float32))
    H0 = [torch.from_numpy((rng.random((K, t)) + 0.1).astype(np.float32)) for t in T2s]
    return Vs, W0, H0


def ragged(h, Vs, W0, H0, iters, alpha, eps, update_W):
    W, Hs = h.to_device(W0), [h.to_device(x) for x in H0]
    h.klnmf_ragged(Vs, W, Hs, iters, alpha, eps, update_W=update_W)
    return W, Hs


def assert_same(h, Vs, W0, H0, iters=3, alpha=0.1, eps=1e-16, update_W=True, what=''):
    W, Hs = ragged(h, Vs, W0, H0, iters, alpha, eps, update_W)
    for b, V in enumerate(Vs):
        Wb, Hb = h.to_device(W0[b]), h.to_device(H0[b])
        h.klnmf(V.contiguous(), Wb, Hb, iters, alpha, eps, update_W=update_W)
        assert nan_equal(W[b], Wb) and nan_equal(Hs[b], Hb), (what, 'clip', b, V.shape)
    return W, Hs


def widths(h, sm, F, T2, K):
    p = tile_plan(h, sm, F, T2, K)
    return p[0], p[1], p[2], p[3]          # W.H width, G2 width, G4 width, G4 k-splits


# configs[0]: F = 513, K = 128, hop 512; 2T of clips from about 2 to 30 s at 16 kHz
SHARED = [130, 250, 622, 938, 1250, 1874]


def test_lengths_sharing_widths(h, sm_count):
    F, K = 513, 128
    plans = [widths(h, sm_count, F, t, K) for t in SHARED]
    assert len({p[:3] for p in plans}) == 1, plans
    Vs, W0, H0 = inputs(h, F, SHARED, K, seed=1)
    for iters, alpha, eps, update_W in RUNS:
        assert_same(h, Vs, W0, H0, iters, alpha, eps, update_W, what=(iters, alpha, eps, update_W))


def mixed_lengths(h, sm, F, K, candidates):
    """The first length of each new W.H width, G2 width and G4 (width, k-splits) among the candidates."""
    seen, picked = [set(), set(), set()], []
    for t in candidates:
        p = widths(h, sm, F, t, K)
        keys = [p[0], p[1], (p[2], p[3])]
        if any(k not in s for k, s in zip(keys, seen)):
            picked.append(t)
            for k, s in zip(keys, seen):
                s.add(k)
    return picked, seen


def test_lengths_with_different_plans(h, sm_count):
    """Clips whose solo plans differ in the W.H width, the G2 width, the G4 width and its k-split count, in one call."""
    F, K = 513, 1024
    T2s, seen = mixed_lengths(h, sm_count, F, K, range(128, 4096, 6))
    assert all(len(s) >= 2 for s in seen), seen
    Vs, W0, H0 = inputs(h, F, T2s, K, seed=2)
    for iters, alpha, eps, update_W in RUNS:
        assert_same(h, Vs, W0, H0, iters, alpha, eps, update_W, what=(T2s, iters, update_W))


def plane_launches(h, sm, F, T2s, K):
    p = [widths(h, sm, F, t, K) for t in T2s]
    return 2 * len({x[0] for x in p}) + len({x[1] for x in p}) + len({x[2] for x in p})


@pytest.mark.parametrize('K,T2s', [(128, SHARED), (1024, None)], ids=['shared', 'mixed'])
def test_launch_count(h, sm_count, K, T2s):
    """Launches per iteration: one per distinct tile width of each contraction (G1 and G3 count apart) plus the W update; with
    every width shared, exactly the launches of an equal-length gccnmf_klnmf_batched call."""
    F, iters = 513, 3
    if T2s is None:
        T2s = mixed_lengths(h, sm_count, F, K, range(128, 4096, 6))[0]
    Vs, W0, H0 = inputs(h, F, T2s, K, seed=3)
    before = h.launches
    ragged(h, Vs, W0, H0, iters, 0.1, 1e-16, True)
    got = h.launches - before
    assert got == 3 + 1 + iters * (plane_launches(h, sm_count, F, T2s, K) + 1) + 2, (got, T2s)
    if K == 128:
        V = h.to_device(np.ones((len(T2s), F, 622), dtype=np.float32))
        W, H = h.to_device(W0), h.to_device(np.ones((len(T2s), K, 622), dtype=np.float32))
        before = h.launches
        h.klnmf_batched(V, W, H, iters, 0.1, 1e-16, update_W=True)
        assert got == h.launches - before


def test_duplicate_lengths(h):
    Vs, W0, H0 = inputs(h, 513, [622, 300, 622, 622, 300], 128, seed=4)
    assert_same(h, Vs, W0, H0)


def test_single_clip(h):
    Vs, W0, H0 = inputs(h, 513, [938], 128, seed=5)
    assert_same(h, Vs, W0, H0, 5)


def test_33_clips_in_place_from_one_matrix(h):
    T2s = [130 + 37 * b for b in range(33)]
    Vs, W0, H0 = inputs(h, 513, T2s, 128, seed=6, flat=True)
    assert Vs[1].stride() == (sum(T2s), 1)
    assert_same(h, Vs, W0, H0)


def test_tensor_core_and_simt_clips_mixed(h):
    F, K, T2s = 513, 128, [100, 622, 64, 300, 127]
    assert [h.klnmf_uses_tensor_cores(F, t, K) for t in T2s] == [False, True, False, True, False]
    for flat in (False, True):
        Vs, W0, H0 = inputs(h, F, T2s, K, seed=7, flat=flat)
        for iters, alpha, eps, update_W in RUNS:
            assert_same(h, Vs, W0, H0, iters, alpha, eps, update_W, what=(flat, iters, update_W))


def test_every_option(h):
    F, K, T2s = 2049, 128, [300, 600, 1250]
    for flat in (False, True):
        Vs, W0, H0 = inputs(h, F, T2s, K, seed=8, flat=flat)
        for opt in OPTIONS:
            kw = dict(opt) if isinstance(opt[0], tuple) else dict([opt])
            with options(h, **kw):
                assert_same(h, Vs, W0, H0, 3, 0.1, 1e-16, True, what=(kw, flat))


def test_nan_filled_workspace(h):
    """Every workspace word the call reads is written by it first."""
    from test_klnmf_ragged_cpu import lengths
    F, K, T2s = 200, 72, [622, 150, 400]
    Vs, W0, H0 = inputs(h, F, T2s, K, seed=9)
    nbytes = h.lib.gccnmf_klnmf_ragged_workspace_bytes(len(T2s), F, lengths(*T2s), K)
    h.workspace('klnmf_ragged', nbytes).fill_(0xFF)
    assert_same(h, Vs, W0, H0, 5)


def test_silent_frame_stays_in_its_clip(h):
    import torch
    Vs, W0, H0 = inputs(h, 513, [622, 300, 938], 128, seed=10)
    Vs[1][:, 100] = 0.0
    W, Hs = assert_same(h, Vs, W0, H0, 5, 0.0, 1e-16, True)
    assert not bool(torch.isfinite(Hs[1]).all()) or not bool(torch.isfinite(W[1]).all())
    for b in (0, 2):
        assert bool(torch.isfinite(W[b]).all()) and bool(torch.isfinite(Hs[b]).all())


def test_refusals(h):
    import torch
    from gcc_nmf_b200._lib import GCCNMF_OK, ParameterError
    from test_klnmf_ragged_cpu import lengths
    lib, F, K, T2s = h.lib, 200, 72, [622, 300]
    Vs, W0, H0 = inputs(h, F, T2s, K)
    W, Hs = h.to_device(W0), [h.to_device(x) for x in H0]
    nbytes = lib.gccnmf_klnmf_ragged_workspace_bytes(2, F, lengths(*T2s), K)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=h.device)
    ptrs = lambda ts: (ctypes.c_void_p * len(ts))(*[t.data_ptr() if t is not None else None for t in ts])

    def call(v=Vs, ld=(622, 300), t2=tuple(T2s), b=2, f=F, w=W.data_ptr(), hh=Hs, k=K, it=3, wsp=ws.data_ptr(), n=nbytes):
        return lib.gccnmf_klnmf_ragged(h.h, ptrs(v) if v is not None else None, (ctypes.c_int64 * 2)(*ld) if ld is not None else None,
                                       lengths(*t2) if t2 is not None else None, b, f, w, ptrs(hh) if hh is not None else None, k, it, 0.0,
                                       1e-16, 1, wsp, n, h.stream)
    before = h.launches
    bad = [dict(b=0), dict(b=-1), dict(b=8192), dict(v=None), dict(ld=None), dict(t2=None), dict(w=None), dict(hh=None),
           dict(v=[Vs[0], None]), dict(hh=[None, Hs[1]]), dict(f=0), dict(k=0), dict(t2=(622, 0)), dict(t2=(-1, 300)),
           dict(ld=(621, 300)), dict(ld=(622, 299)), dict(it=-1), dict(wsp=None), dict(n=nbytes - 1)]
    for kw in bad:
        assert call(**kw) != GCCNMF_OK, kw
    assert h.launches == before                 # refused before anything was enqueued
    assert call(it=0) == GCCNMF_OK and h.launches == before
    assert call() == GCCNMF_OK
    with pytest.raises(ParameterError):
        h.klnmf_ragged(Vs, W[:, :, :8], Hs, 1)
    with pytest.raises(ParameterError):
        h.klnmf_ragged([Vs[0].t(), Vs[1]], W, Hs, 1)
    with pytest.raises(ParameterError):
        h.klnmf_ragged(Vs, W, Hs[:1], 1)


def test_perform_klnmf_batch_on_a_list(h):
    from gcc_nmf_b200 import gccNMFFunctions as fn
    rng = np.random.default_rng(11)
    Vs = [(rng.random((513, t)) ** 3 + 1e-3).astype(np.float32) for t in (622, 90, 1250, 300)]
    W, Hs = fn.performKLNMFBatch(Vs, 128, 10, 0.1)
    assert W.shape == (4, 513, 128) and [x.shape for x in Hs] == [(128, V.shape[1]) for V in Vs]
    for b, V in enumerate(Vs):
        Wb, Hb = fn.performKLNMF(V, 128, 10, 0.1)
        assert np.array_equal(W[b], Wb, equal_nan=True) and np.array_equal(Hs[b], Hb, equal_nan=True), b


def clips_ragged():
    """The shipped recording cut to 6 s and 10 s, and synthetic clips of 1.5 s (a SIMT-path NMF), 4 s and 14 s."""
    import os
    from gcc_nmf_b200.synth import synthetic_stereo
    from gcc_nmf_b200.wavio import wavread
    here = os.path.dirname(os.path.abspath(__file__))
    rec, sr = wavread(os.path.join(here, 'golden', 'dev1_female3_liverec_130ms_1m_mix.wav'))
    rec = np.asarray(rec, dtype=np.float32)[:2]
    cut = lambda s: np.ascontiguousarray(rec[:, :int(s * sr)])
    return sr, [cut(6.0), synthetic_stereo(1.5, sr, seed=31), cut(10.0), synthetic_stereo(4.0, sr, seed=32),
                synthetic_stereo(14.0, sr, seed=33, num_sources=3)]


@pytest.mark.parametrize('flow', ['enhance', 'separate'])
def test_pipeline_batch_flows_on_a_list(h, flow):
    """configs[0] settings: N = 1024, hop = 512 (F = 513), K = 128, 64 TDOAs, 100 iterations."""
    from gcc_nmf_b200.pipeline import GCCNMFPipeline
    sr, xs = clips_ragged()
    pipe = GCCNMFPipeline(sr, 1024, 512, 64, 1.0, 128, 100, handle=h)
    keep = lambda r: {k: (v.clone() if hasattr(v, 'clone') else v) for k, v in r.items()}     # results are views of reused buffers
    clips = [h.to_device(x) for x in xs]
    if flow == 'enhance':
        batch = [keep(r) for r in pipe.enhance_batch(clips)]
        singles = [keep(pipe.enhance(c)) for c in clips]
        extra = ['argMaxGCCNMF']
    else:
        batch = [keep(r) for r in pipe.separate_batch(clips, 2)]
        singles = [keep(pipe.separate(c, 2)) for c in clips]
        extra = ['targetTDOAGCCNMFs']
    assert len(batch) == len(xs)
    for b in range(len(xs)):
        assert batch[b]['targetTDOAIndexes'] == singles[b]['targetTDOAIndexes'], b
        for k in SIGNAL_KEYS + extra:
            assert batch[b][k].shape == singles[b][k].shape and _equal(batch[b][k], singles[b][k]), (flow, b, k)
