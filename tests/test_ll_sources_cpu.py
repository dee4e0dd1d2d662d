"""CPU: the low-latency engine with several sources per stream (gccnmf_llsep_*): the state carve, configuration checks, the header
against the bindings, and the host model of the per-frame target decisions (oracle/ll_sources.py) against the reference's own
multi-target peak rule."""
import ctypes
import os
import re

import numpy as np
import pytest

from oracle import ll_sources as model

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _lib():
    from gcc_nmf_b200 import _lib
    try:
        return _lib.load_library()
    except ImportError:
        pytest.skip('library not built')


def _cfg(**kw):
    from gcc_nmf_b200._lib import LLConfig
    c = dict(window_size=1024, hop_size=64, hops_per_call=1, num_atoms=256, num_tdoas=128, num_streams=4, inference_iterations=0,
             sparsity_alpha=0.0, epsilon=1e-16)
    c.update(kw)
    return LLConfig(*[c[f] for f, _ in LLConfig._fields_])


def test_state_carve_grows_with_sources():
    lib = _lib()
    N = 1024
    for kw in (dict(), dict(inference_iterations=5, hops_per_call=3), dict(num_tdoas=16, window_size=256, hop_size=32)):
        cfg = _cfg(**kw)
        n = kw.get('window_size', N)
        single = lib.gccnmf_ll_state_bytes(ctypes.byref(cfg))
        sizes = [lib.gccnmf_llsep_state_bytes(ctypes.byref(cfg), P) for P in range(2, 9)]
        assert sizes[0] > single > 0
        assert all(a < b for a, b in zip(sizes, sizes[1:]))
        assert all(v % 256 == 0 for v in sizes)
        for P in range(2, 9):
            more = _cfg(**dict(kw, num_streams=5))
            per_stream = lib.gccnmf_llsep_state_bytes(ctypes.byref(more), P) - lib.gccnmf_llsep_state_bytes(ctypes.byref(cfg), P)
            assert per_stream >= P * 2 * n * 4, (kw, P)                 # P output rings of 2 x N float32 at least


def test_invalid_sources_and_configurations():
    lib = _lib()
    cfg = _cfg()
    for P in (-1, 0, 1, 9, 100):
        assert lib.gccnmf_llsep_state_bytes(ctypes.byref(cfg), P) == 0, P
    assert lib.gccnmf_llsep_state_bytes(None, 2) == 0
    for bad in (dict(window_size=1000), dict(hop_size=0), dict(hops_per_call=65), dict(num_atoms=0), dict(num_tdoas=100),
                dict(num_streams=0), dict(num_streams=4097), dict(inference_iterations=-1)):
        assert lib.gccnmf_llsep_state_bytes(ctypes.byref(_cfg(**bad)), 3) == 0, bad
    # P x K x T must stay within int32: 8 sources x 60000 atoms x 4096 streams x 2 hops does not
    assert lib.gccnmf_llsep_state_bytes(ctypes.byref(_cfg(num_atoms=60000, num_streams=4096, hops_per_call=2)), 8) == 0
    assert lib.gccnmf_ll_state_bytes(ctypes.byref(_cfg(num_atoms=60000, num_streams=4096, hops_per_call=2))) > 0


def test_entry_points_refuse_before_enqueueing():
    """With a NULL handle every entry fails on its arguments (nothing can have been enqueued)."""
    lib = _lib()
    cfg = _cfg()
    assert lib.gccnmf_llsep_process(None, ctypes.byref(cfg), 2, None, 0, 1, None, None, None) != 0
    assert lib.gccnmf_llsep_set_targets(None, ctypes.byref(cfg), 2, None, 0, 0, 1, None, None) != 0


def test_header_agrees_with_bindings():
    from gcc_nmf_b200 import _lib
    from gcc_nmf_b200 import lowlatency as ll
    header = open(os.path.join(ROOT, 'include', 'gccnmf_b200.h')).read()
    declared = set(re.findall(r'GCCNMF_API\s+[\w\s\*]+?\b(gccnmf_llsep_\w+)\s*\(', header))
    bound = {n for n in _lib.SIGNATURES if n.startswith('gccnmf_llsep_')}
    assert declared == bound and len(bound) == 8
    defines = dict(re.findall(r'#define (GCCNMF_LLSEP_\w+) (\d+)', header))
    assert int(defines['GCCNMF_LLSEP_MAX_SOURCES']) == ll.MAX_SOURCES
    assert int(defines['GCCNMF_LLSEP_STATUS_FEW_PEAKS']) == ll.STATUS_FEW_PEAKS == model.STATUS_FEW_PEAKS
    assert int(defines['GCCNMF_LLSEP_STATUS_ALL_NAN']) == ll.STATUS_ALL_NAN == model.STATUS_ALL_NAN
    for name, value in (('TARGETS', ll.EXPORT_SOURCE_TARGETS), ('VALUES', ll.EXPORT_SOURCE_VALUES), ('MASKS', ll.EXPORT_SOURCE_MASKS),
                        ('WIENER', ll.EXPORT_SOURCE_WIENER), ('Y', ll.EXPORT_SOURCE_Y), ('STREAM_STATUS', ll.EXPORT_STREAM_STATUS),
                        ('CARRIED_TARGETS', ll.EXPORT_CARRIED_TARGETS), ('CALL_STATUS', ll.EXPORT_CALL_STATUS)):
        assert int(defines['GCCNMF_LLSEP_EXPORT_' + name]) == value, name


def test_engine_rejects_bad_source_counts():
    from gcc_nmf_b200.lowlatency import LowLatencyEngine
    F, K, D, N = 129, 8, 8, 256
    for P in (1, 9, -2):
        with pytest.raises(ValueError):
            LowLatencyEngine(np.ones((F, K), np.float32), np.ones((F, D), np.complex128), np.ones(N), np.ones(N), 32, numSources=P)


# ------------------------------------------------------------------------------------------------ host model vs the reference
def _column(rng, D, peaks):
    """A running-maximum column with `peaks` strict interior maxima of distinct values."""
    x = -5.0 + np.arange(D) * 1e-3                # rising: no maximum of its own
    where = np.sort(rng.choice(np.arange(1, D - 1, 2), peaks, replace=False))
    x[where] = rng.permutation(np.linspace(1.0, 2.0, peaks))
    return x


@pytest.mark.parametrize('D', [16, 128])
@pytest.mark.parametrize('P', [2, 3, 8])
def test_peak_rule_matches_reference(P, D):
    """pick_peaks == gccnmf_oracle.estimateTargetTDOAIndexesFromAngularSpectrum(numSources=P) on columns with distinct peak values
    and at least P peaks; with fewer, the reference finds too few and the model holds the targets and sets the status."""
    from oracle import gccnmf_oracle as orc
    rng = np.random.default_rng(P * 1000 + D)
    most = (D - 2 + 1) // 2                      # interior odd positions: the most peaks _column places
    for i in range(60 if P <= most else 0):
        x = _column(rng, D, int(rng.integers(P, most + 1)))
        ref = [int(v) for v in orc.estimateTargetTDOAIndexesFromAngularSpectrum(x, 0.1, D, P)]
        assert model.pick_peaks(x, P).tolist() == ref
    for i in range(20):
        x = _column(rng, D, int(rng.integers(0, P)))
        with pytest.raises(ValueError):
            orc.estimateTargetTDOAIndexesFromAngularSpectrum(x, 0.1, D, P)
        assert model.pick_peaks(x, P) is None


@pytest.mark.parametrize('P', [2, 3, 8])
def test_stream_model_holds_defaults_and_overrides(P):
    from oracle import gccnmf_oracle as orc
    D = 32
    rng = np.random.default_rng(P)
    m = model.SourceTargets(D, P)
    assert m.column_targets().tolist() == [(2 * q + 1) * D // (2 * P) for q in range(P)]
    # the running maximum is carried: a column that falls everywhere leaves the previous maximum and its targets
    hi = _column(rng, D, P + 2)
    acc, t = m.frame(hi)
    assert np.array_equal(acc, hi) and t.tolist() == [int(v) for v in orc.estimateTargetTDOAIndexesFromAngularSpectrum(hi, 0.1, D, P)]
    acc2, t2 = m.frame(hi - 10.0)
    assert np.array_equal(acc2, hi) and np.array_equal(t2, t) and m.status == 0
    # a NaN sticks in the running maximum: no peak next to it, and with all of it NaN no peak at all
    m.frame(np.full(D, np.nan))
    assert np.isnan(m.carry).all() and m.status == model.STATUS_FEW_PEAKS and np.array_equal(m.column_targets(), t)
    m.frame(_column(rng, D, P + 3))
    assert m.status == model.STATUS_FEW_PEAKS and np.array_equal(m.column_targets(), t)     # sticky, and the targets held
    over = np.full(P, -1, np.int32)
    over[P - 1] = 5
    m.set_override(over)
    assert m.column_targets()[:P - 1].tolist() == t[:P - 1].tolist() and m.column_targets()[P - 1] == 5
    m.reset()
    assert m.status == 0 and np.isneginf(m.carry).all() and m.column_targets()[P - 1] == 5
    assert m.targets.tolist() == model.default_targets(D, P).tolist()
