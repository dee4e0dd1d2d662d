"""CPU: the localisation window of the low-latency engine (gccnmf_llhist_*).  The host model (oracle/ll_window.py) against a plain
loop over the frames a stream has seen; the state and record sizes against a restatement of the carve (Lh = 0 giving the ll /
llsep / llrec sizes); the header's history field; the bindings; and refusals that need no device."""
import ctypes
import os
import re

import numpy as np
import pytest

from oracle import ll_window as lw
from oracle.ll_sources import default_targets, pick_peaks

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _lib():
    from gcc_nmf_b200 import _lib
    try:
        return _lib.load_library()
    except ImportError:
        pytest.skip('library not built')


# ---------------------------------------------------------------------------------------------- the model against a plain loop
def _plain_mean(seen, Lh, w):
    """Newest-first float64 nanmean of the last w of (Lh zero columns, then every column seen), NaN when all are NaN."""
    cols = [np.zeros(len(seen[0]) if seen else 0)] * Lh + list(seen)
    out = []
    for d in range(len(cols[-1])):
        s, n = 0.0, 0
        for c in reversed(cols[-w:]):
            if c[d] == c[d]:
                s += float(c[d])
                n += 1
        out.append(s / n if n else float('nan'))
    return np.array(out)


def _plain_argmax(x):
    best = 0
    for d in range(1, len(x)):
        a, b = x[d], x[best]
        if (a != a and b == b) or (a == a and b == b and a > b):
            best = d
    return best


def _columns(D, n, seed):
    rng = np.random.RandomState(seed)
    ang = rng.standard_normal((n, D))
    ang[rng.random_sample(n) < 0.15] = np.nan          # a silent frame is NaN in every TDOA
    return ang


@pytest.mark.parametrize('Lh,w', [(5, 1), (5, 3), (5, 5), (8, 8), (8, 2), (1, 1)])
@pytest.mark.parametrize('P', [0, 2, 3])
def test_model_equals_plain_loop(Lh, w, P):
    """Ring wraps (frames = 4 Lh + 3), w = Lh, w larger than the frames seen (the first frames), NaN columns and invalid frames."""
    D = 12
    n = 4 * Lh + 3
    ang = _columns(D, n, seed=Lh * 10 + w + P)
    valid = np.ones(n, bool)
    valid[[2, 3, n // 2]] = False
    m = lw.WindowTargets(D, Lh, P)
    m.window = w
    seen = []
    targets = default_targets(D, P) if P else None
    status = 0
    carry = np.full(D, -np.inf)
    for t in range(n):
        if valid[t]:
            seen.append(ang[t])
            carry = np.array([v if (v > c or v != v) else c for v, c in zip(ang[t], carry)])
        mean, got = m.frame(ang[t], valid[t])
        want = _plain_mean(seen, Lh, w)
        assert np.array_equal(mean, want, equal_nan=True), t
        assert len(seen) % Lh == m.index
        if not P:
            assert got == _plain_argmax(want), t
            continue
        if valid[t]:
            picked = pick_peaks(want, P)
            if picked is None:
                status |= lw.STATUS_FEW_PEAKS
            else:
                targets = picked
        assert np.array_equal(got, targets), t
        assert m.status == status
    assert np.array_equal(m.carry, carry, equal_nan=True)


def test_model_window_zero_is_running_maximum():
    D, Lh = 8, 4
    ang = _columns(D, 20, seed=3)
    m = lw.WindowTargets(D, Lh)
    carry = np.full(D, -np.inf)
    for t in range(20):
        with np.errstate(invalid='ignore'):
            carry = np.where((ang[t] > carry) | np.isnan(ang[t]), ang[t], carry)
        mean, got = m.frame(ang[t])
        assert np.isnan(mean).all() and got == np.argmax(carry)


def test_model_recovers_after_w_clean_frames():
    """A NaN frame decides nothing once w frames without NaN followed it."""
    D, Lh, w = 8, 16, 6
    m = lw.WindowTargets(D, Lh)
    m.window = w
    m.frame(np.full(D, np.nan))
    col = np.zeros(D)
    col[5] = 1.0
    for i in range(w):
        mean, got = m.frame(col)
    assert not np.isnan(mean).any() and got == 5


# ---------------------------------------------------------------------------------------------- sizes, header, bindings, refusals
def _cfg(**kw):
    from gcc_nmf_b200._lib import LLConfig
    c = dict(window_size=256, hop_size=32, hops_per_call=1, num_atoms=64, num_tdoas=16, num_streams=4, inference_iterations=0,
             sparsity_alpha=0.0, epsilon=1e-16)
    c.update(kw)
    return LLConfig(*[c[f] for f, _ in LLConfig._fields_])


def _up(x, a):
    return (x + a - 1) // a * a


def _state_bytes(lib, c, P, Lh):
    """ll_carve restated: every region 256-aligned, in carve order, the history (ring + index + window + 8 bytes per stream, then
    the call's (D, T) means) last."""
    S, N, hop, C, K, D = c.num_streams, c.window_size, c.hop_size, c.hops_per_call, c.num_atoms, c.num_tdoas
    F, R, T, inf, Pm = N // 2 + 1, (-(-N // hop) - 1) * hop, S * C, c.inference_iterations > 0, max(P, 1)
    regions = [8, 24 * S, 16, 8 * N, 8 * N, 8 * 2 * F * D, 4 * F * K, 4 * K * F * inf, 4 * K * inf, 4 * 2 * K * inf, 4 * S * 2 * R,
               4 * S * Pm * 2 * N, 8 * S * D, 4 * 2 * S * (R + C * hop), 4 * 4 * F * T, 4 * 2 * F * T * inf, 4 * 2 * F * T, 8 * D * T,
               8 * D * T, 4 * T, 4 * T, 4 * K * T, 4 * K * T, 4 * Pm * (2 if inf else 1) * F * T, 4 * Pm * 4 * F * T, 4 * 2 * K * T * inf,
               4 * Pm * 2 * T * N, lib.gccnmf_wiener_apply_workspace_bytes(F) // 4 * 4, lib.gccnmf_tdoa_argmax_workspace_bytes(F, T, D, K),
               4 * S * 8 * (P > 0), 4 * S * 8 * (P > 0), 4 * S * (P > 0), 4 * T * P, 4 * P * K * T, 4 * P * K * T,
               S * (8 * D * Lh + 16) * (Lh > 0), 8 * D * T * (Lh > 0)]
    used = 0
    for r in regions:
        used = _up(used, 256) + r
    return _up(used, 256)


def _payload(c, P, Lh):
    N, hop, D = c.window_size, c.hop_size, c.num_tdoas
    R = (-(-N // hop) - 1) * hop
    sizes = [24, 8 * D, 4 * 2 * R, 4 * max(P, 1) * 2 * N] + ([32, 32, 4] if P else []) + ([8 * D * Lh + 16] if Lh else [])
    return sum(_up(s, 16) for s in sizes if s)


SWEEP = [dict(), dict(window_size=1024, hop_size=64, num_tdoas=128, num_atoms=256, num_streams=1024, hops_per_call=3),
         dict(hop_size=24), dict(hop_size=256), dict(hop_size=100, num_tdoas=4), dict(inference_iterations=5, hops_per_call=7),
         dict(window_size=4096, hop_size=1000, num_tdoas=128, num_streams=4096)]


@pytest.mark.parametrize('kw', SWEEP, ids=[str(i) for i in range(len(SWEEP))])
def test_state_and_record_sizes(kw):
    lib = _lib()
    c = _cfg(**kw)
    for P in (0, 2, 3, 8):
        base = lib.gccnmf_llsep_state_bytes(ctypes.byref(c), P) if P else lib.gccnmf_ll_state_bytes(ctypes.byref(c))
        assert lib.gccnmf_llhist_state_bytes(ctypes.byref(c), P, 0) == base
        assert lib.gccnmf_llhist_record_bytes(ctypes.byref(c), P, 0) == lib.gccnmf_llrec_record_bytes(ctypes.byref(c), P)
        assert lib.gccnmf_llhist_workspace_bytes(ctypes.byref(c), P, 0, 3) == lib.gccnmf_llrec_workspace_bytes(ctypes.byref(c), P, 3)
        for Lh in (0, 1, 5, 64, 1024):
            assert lib.gccnmf_llhist_state_bytes(ctypes.byref(c), P, Lh) == _state_bytes(lib, c, P, Lh), (P, Lh)
            assert lib.gccnmf_llhist_record_bytes(ctypes.byref(c), P, Lh) == 256 + _up(_payload(c, P, Lh), 256), (P, Lh)
            for count in (1, 3):
                assert lib.gccnmf_llhist_workspace_bytes(ctypes.byref(c), P, Lh, count) == count * _payload(c, P, Lh), (P, Lh)


def test_header_history_field():
    from gcc_nmf_b200 import _lib as L
    assert ctypes.sizeof(L.LLConfig) == 4 * L.LLHIST_RECORD_CONFIG_HISTORY
    assert L.LLHIST_RECORD_CONFIG_HISTORY < len(L.RecordHeader().config)
    header = open(os.path.join(ROOT, 'include', 'gccnmf_b200.h')).read()
    defines = dict(re.findall(r'#define (GCCNMF_LLHIST_\w+) (\d+)', header))
    assert int(defines['GCCNMF_LLHIST_MAX_HISTORY']) == L.LLHIST_MAX_HISTORY == 1024
    from gcc_nmf_b200 import lowlatency as ll
    assert [int(defines['GCCNMF_LLHIST_EXPORT_' + k]) for k in ('RING', 'INDEX', 'WINDOWS', 'MEANS')] == \
        [ll.EXPORT_HISTORY, ll.EXPORT_HISTORY_INDEX, ll.EXPORT_WINDOWS, ll.EXPORT_WINDOW_MEANS]


def test_header_agrees_with_bindings():
    from gcc_nmf_b200 import _lib as L
    header = open(os.path.join(ROOT, 'include', 'gccnmf_b200.h')).read()
    declared = set(re.findall(r'GCCNMF_API\s+[\w\s\*]+?\b(gccnmf_llhist_\w+)\s*\(', header))
    bound = {n for n in L.SIGNATURES if n.startswith('gccnmf_llhist_')}
    assert declared == bound == {'gccnmf_llhist_' + n for n in (
        'state_bytes', 'init', 'reset_streams', 'set_params', 'set_targets', 'set_window', 'process', 'graph_create', 'export',
        'record_bytes', 'workspace_bytes', 'save_streams', 'load_streams')}
    for name in bound:
        decl = re.search(r'GCCNMF_API\s+[\w\s\*]+?\b%s\s*\((.*?)\);' % name, header, re.S).group(1)
        assert len(decl.split(',')) == len(L.SIGNATURES[name][1]), name


def test_host_refusals():
    lib = _lib()
    c = _cfg()
    for Lh in (-1, 1025, 4096):
        assert lib.gccnmf_llhist_state_bytes(ctypes.byref(c), 0, Lh) == 0, Lh
        assert lib.gccnmf_llhist_record_bytes(ctypes.byref(c), 2, Lh) == 0, Lh
        assert lib.gccnmf_llhist_workspace_bytes(ctypes.byref(c), 0, Lh, 1) == 0, Lh
    for P in (-1, 1, 9):
        assert lib.gccnmf_llhist_state_bytes(ctypes.byref(c), P, 8) == 0, P
    assert lib.gccnmf_llhist_workspace_bytes(ctypes.byref(c), 0, 8, 0) == 0
    assert lib.gccnmf_llhist_state_bytes(None, 0, 8) == 0
    w = (ctypes.c_int32 * 1)(1)
    assert lib.gccnmf_llhist_set_window(None, ctypes.byref(c), 0, 8, None, 0, 0, 1, w, None) != 0
    assert lib.gccnmf_llhist_save_streams(None, ctypes.byref(c), 0, 8, None, 0, 0, 1, None, 0, None, 0, None) != 0
    assert lib.gccnmf_llhist_load_streams(None, ctypes.byref(c), 0, 8, None, 0, 0, 1, None, 0, None, 0, None) != 0


def test_engine_refuses_history_length_on_the_host():
    from gcc_nmf_b200 import lowlatency as ll
    for Lh in (-1, 1025):
        with pytest.raises(ValueError, match='historyLength'):
            ll.LowLatencyEngine(np.ones((129, 8), np.float32), np.ones((129, 8), complex), np.ones(256), np.ones(256), 32, historyLength=Lh)
