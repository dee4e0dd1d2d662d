"""CPU: the host side of the real-time path with several sources per stream (gccnmf_rtsep_*): state sizing, argument checks, no
CPU fallback, and the host model of the source stages (oracle/rt_sources.py) against the reference's own multi-target rule."""
import ctypes

import numpy as np
import pytest


@pytest.fixture(scope='module')
def lib():
    import __graft_entry__ as entry
    entry.build()
    from gcc_nmf_b200 import _lib
    return _lib.load_library()


def _cfg(**kw):
    from gcc_nmf_b200._lib import RtConfig
    c = dict(window_size=512, hop_size=128, block_size=128, windows_per_block=1, num_atoms=1024, num_tdoas=64, history_length=128,
             inference_iterations=10, sparsity_alpha=0.0, epsilon=1e-16)
    c.update(kw)
    return RtConfig(**c)


@pytest.mark.parametrize('P', [2, 3, 8])
def test_state_bytes_grows_linearly_in_streams(lib, P):
    cfg = _cfg()
    streams = (1, 2, 3, 8, 64, 1024)
    sizes = [lib.gccnmf_rtsep_state_bytes(ctypes.byref(cfg), s, P) for s in streams]
    per_slot = sizes[1] - sizes[0]
    assert per_slot > 0 and per_slot % 256 == 0
    for s, v in zip(streams, sizes):
        assert v == sizes[0] + (s - 1) * per_slot
    # a slot holds at least P output rings, P masks and P output spectra on top of a single-target slot
    single = lib.gccnmf_rtm_state_bytes(ctypes.byref(cfg), 2) - lib.gccnmf_rtm_state_bytes(ctypes.byref(cfg), 1)
    assert per_slot >= single + P * (4 * 2 * 8 * 128 + 8 * 1024 + 8 * 2 * 257)
    assert lib.gccnmf_rtsep_state_bytes(ctypes.byref(cfg), 5, P) < lib.gccnmf_rtsep_state_bytes(ctypes.byref(cfg), 5, P + 1) or P == 8


def test_zero_sources_is_the_multi_stream_layout(lib):
    for kw in (dict(), dict(num_tdoas=16, windows_per_block=4, hop_size=32), dict(inference_iterations=0, num_atoms=200)):
        cfg = _cfg(**kw)
        for s in (1, 7, 256):
            assert lib.gccnmf_rtsep_state_bytes(ctypes.byref(cfg), s, 0) == 0      # the rtsep entries need sources
            # the P = 0 carve is the one gccnmf_rtm_* use, and it is unchanged by the source regions
            assert lib.gccnmf_rtsep_state_bytes(ctypes.byref(cfg), s, 2) > lib.gccnmf_rtm_state_bytes(ctypes.byref(cfg), s) > 0


def test_state_bytes_rejects_invalid_input(lib):
    cfg = _cfg()
    for P in (-1, 1, 9, 100):
        assert lib.gccnmf_rtsep_state_bytes(ctypes.byref(cfg), 4, P) == 0, P
    assert lib.gccnmf_rtsep_state_bytes(ctypes.byref(cfg), 0, 2) == 0
    assert lib.gccnmf_rtsep_state_bytes(ctypes.byref(cfg), 4097, 2) == 0
    assert lib.gccnmf_rtsep_state_bytes(None, 4, 2) == 0
    for bad in (dict(num_tdoas=0), dict(num_tdoas=129), dict(window_size=500), dict(windows_per_block=9), dict(num_atoms=0),
                dict(history_length=0), dict(block_size=16)):
        assert lib.gccnmf_rtsep_state_bytes(ctypes.byref(_cfg(**bad)), 4, 3) == 0, bad


def test_engine_with_sources_has_no_cpu_fallback(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip('GPU present')
    from gcc_nmf_b200 import _lib
    from gcc_nmf_b200.realtime.multistream import MultiStreamRealtimeEngine
    F, K, D, N = 257, 16, 8, 512
    W = np.ones((F, K), np.float32)
    E = np.ones((F, D), np.complex64)
    with pytest.raises(ValueError):
        MultiStreamRealtimeEngine(W, E, np.ones(N, np.float32), np.ones(N, np.float32), 128, 128, 1, 4, numSources=1)
    with pytest.raises(_lib.GCCNMFError):
        MultiStreamRealtimeEngine(W, E, np.ones(N, np.float32), np.ones(N, np.float32), 128, 128, 1, 4, numSources=3)


# ------------------------------------------------------------------------------------------------ host model vs the reference
def _values(rng, P, K, T, kind):
    v = rng.standard_normal((P, K, T)).astype(np.float32)
    if kind == 'tied':
        v[:, ::3] = v[0, ::3]                      # every source equal on a third of the atoms
        v[1:, 1::5] = v[:1, 1::5].max() + 1.0      # sources 1 .. P-1 tie at the top on a fifth
    elif kind == 'plateau':
        v[:] = np.round(v * 2) / 2                 # few distinct values: many ties
    elif kind == 'nan':
        v[:, 2::7, 1] = np.nan                     # all-NaN columns (what digital silence gives: every target row is NaN)
    return v


@pytest.mark.parametrize('kind', ['random', 'tied', 'plateau', 'nan'])
@pytest.mark.parametrize('P', [2, 3, 8])
def test_source_masks_match_reference_rule(P, kind):
    """source_masks == gccNMFFunctions.getTargetCoefficientMasks (numpy nanargmax, first maximum) on every column the reference
    accepts; an all-NaN column, which the reference rejects, goes to source 0."""
    from oracle import gccnmf_oracle as orc
    from oracle import rt_sources as rs
    rng = np.random.default_rng(P * 10 + len(kind))
    K, T, D = 96, 3, 24
    targets = rng.choice(D, P, replace=False)
    v = _values(rng, P, K, T, kind)
    C = rng.standard_normal((T, D, K)).astype(np.float32)
    C[:, targets, :] = v.transpose(2, 0, 1)
    masks, values = rs.source_masks(C, targets)
    assert masks.dtype == np.float64 and masks.shape == (P, K, T)
    assert np.array_equal(values, v, equal_nan=True)
    assert np.array_equal(masks.sum(axis=0), np.ones((K, T)))              # a partition of the atoms
    dead = np.isnan(v).all(axis=0)
    if dead.any():
        with pytest.raises(ValueError):
            orc.getTargetCoefficientMasks(v, P)
        assert (masks[0][dead] == 1).all()
        v = np.where(dead[None], 0.0, v)                                   # the reference on the columns it accepts
        ref = orc.getTargetCoefficientMasks(v, P)
        assert np.array_equal(masks[:, ~dead], ref[:, ~dead])
    else:
        assert np.array_equal(masks, orc.getTargetCoefficientMasks(v, P).astype(np.float64))


def test_source_masks_duplicate_targets_go_to_the_lower_source():
    from oracle import rt_sources as rs
    C = np.random.default_rng(1).standard_normal((2, 10, 32)).astype(np.float32)
    masks, _ = rs.source_masks(C, [4, 7, 4])
    assert not masks[2].any()
    assert np.array_equal(masks[0] + masks[1], np.ones((32, 2)))


def _spectrum(rng, D, kind):
    x = rng.standard_normal(D)
    if kind == 'plateau':
        x[3:6] = x[3]                              # a plateau is not a strict maximum
    elif kind == 'tied':
        x[:] = -1.0
        x[2::4] = 1.0                              # equal peaks: argsort order, the higher index counts as larger
    elif kind == 'nan':
        x[::5] = np.nan
    elif kind == 'flat':
        x[:] = 0.5                                 # no peak at all
    return x


@pytest.mark.parametrize('kind', ['random', 'plateau', 'tied', 'nan', 'flat'])
@pytest.mark.parametrize('P', [2, 3, 8])
def test_localize_sources_match_reference_peak_picking(P, kind):
    """History push, windowed nanmean and top-P peaks against gccnmf_oracle.estimateTargetTDOAIndexesFromAngularSpectrum
    (argrelmax, largest P, ascending) applied to the nanmean of the same columns; fewer peaks keep the targets and flag it."""
    from oracle import gccnmf_oracle as orc
    from oracle import rt_exact as rx
    from oracle import rt_sources as rs
    rng = np.random.default_rng(P + 7 * len(kind))
    D, L, nT, window = 32, 12, 2, 5
    hist = np.zeros((D, L))
    index, targets = 0, np.arange(P, dtype=np.int32)
    for block in range(9):
        gcc = np.stack([_spectrum(rng, D, kind) for _ in range(nT)], axis=1).astype(np.float32)
        h_ref, i_ref, _ = rx.localize(hist, index, gcc, window, False, 0.0)
        hist, index, new, status = rs.localize_sources(hist, index, gcc, window, True, targets, P)
        assert np.array_equal(hist, h_ref, equal_nan=True) and index == i_ref
        cols = [(index - 1 - j) % L for j in range(min(window, L))]
        with np.errstate(all='ignore'), __import__('warnings').catch_warnings():
            __import__('warnings').simplefilter('ignore', RuntimeWarning)
            mean = np.nanmean(hist[:, cols], axis=1)
        try:
            ref = [int(i) for i in orc.estimateTargetTDOAIndexesFromAngularSpectrum(mean, 0.1, D, P)]
        except ValueError:
            ref = None
        if ref is None:
            assert status == rs.STATUS_FEW_PEAKS and np.array_equal(new, targets)
        else:
            assert status == 0 and new.tolist() == ref
        targets = new
    # localisation off: the history moves, the targets do not
    _, _, kept, status = rs.localize_sources(hist, index, gcc, window, False, targets, P)
    assert status == 0 and np.array_equal(kept, targets)
