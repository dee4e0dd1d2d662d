"""CPU: the host model of the offline window targets (oracle/offline_window.py) against a plain per-frame loop, the tracked
pipeline's workspace formula, the new bindings against the header, and the refusals the library makes without a device."""
import ctypes
import os
import re

import numpy as np
import pytest

from oracle import offline_window as ow

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_ENTRIES = ('gccnmf_window_targets', 'gccnmf_target_gccnmf', 'gccnmf_argmax_mask_frames', 'gccnmf_pipeline_tracked_workspace_bytes',
               'gccnmf_separate_tracked')


@pytest.fixture(scope='module')
def lib():
    import __graft_entry__ as entry
    entry.build()
    from gcc_nmf_b200 import _lib
    return _lib.load_library()


def plain_loop(A, w, P):
    """The rule written out frame by frame and term by term, with no helper of the oracle."""
    D, T = A.shape
    means = np.empty((D, T))
    targets = np.empty((T, P), np.int32)
    last = [(2 * q + 1) * D // (2 * P) for q in range(P)]
    status = 0
    for t in range(T):
        for d in range(D):
            s, n = 0.0, 0
            for u in range(t, max(0, t - w + 1) - 1, -1):
                v = A[d, u]
                if v == v:
                    s += v
                    n += 1
            means[d, t] = s / n if n else np.nan
        m = means[:, t]
        peaks = [d for d in range(1, D - 1) if m[d] > m[d - 1] and m[d] > m[d + 1]]
        if len(peaks) < P:
            status = 1
        else:
            ranked = sorted(peaks, key=lambda d: (m[d], d), reverse=True)
            last = sorted(ranked[:P])
        targets[t] = last
    return means, targets, status


def spectrogram(D, T, seed, moving=True):
    """Two bumps over TDOA; the first moves across the array half way through the clip."""
    rng = np.random.default_rng(seed)
    d = np.arange(D)[:, None]
    centre = np.where(np.arange(T) < T // 2, D // 4, 3 * D // 4) if moving else np.full(T, D // 4)
    A = np.exp(-0.5 * ((d - centre[None]) / 1.5) ** 2) + 0.6 * np.exp(-0.5 * ((d - D // 2 - 2) / 1.5) ** 2)
    return A + 0.05 * rng.standard_normal((D, T))


def equal(a, b):
    return np.array_equal(np.asarray(a), np.asarray(b), equal_nan=True)


@pytest.mark.parametrize('w', [1, 3, 8, 40, 45])
@pytest.mark.parametrize('P', [1, 2, 3])
def test_oracle_matches_plain_loop(w, P):
    A = spectrogram(16, 40, seed=w * 10 + P)
    means, targets, status = ow.window_targets(A, w, P)
    pm, pt, ps = plain_loop(A, w, P)
    assert equal(means, pm) and equal(targets, pt) and status == ps


def test_nan_columns_and_silence():
    """NaN columns are skipped; a window of only NaN columns is NaN, has no peaks and holds."""
    A = spectrogram(12, 30, seed=3)
    A[:, 0:4] = np.nan              # digital silence at the start: no peaks, the defaults
    A[:, 15] = np.nan               # one NaN column in the middle, bridged by the window
    A[5, 20:23] = np.nan            # one TDOA row NaN for a while
    for w in (1, 2, 6, 31):
        means, targets, status = ow.window_targets(A, w, 2)
        pm, pt, ps = plain_loop(A, w, 2)
        assert equal(means, pm) and equal(targets, pt) and status == ps == 1
        assert np.isnan(means[:, :4]).all()
        assert (targets[:4] == [3, 9]).all()                       # floor((2q + 1) 12 / 4)
    means, targets, _ = ow.window_targets(A, 1, 2)
    assert np.isnan(means[:, 15]).all() and (targets[15] == targets[14]).all()


def test_hold_in_the_middle():
    """A flat stretch (no strict maxima) holds the targets of the frame before it, not the defaults."""
    A = spectrogram(16, 30, seed=4)
    A[:, 10:14] = 1.0
    means, targets, status = ow.window_targets(A, 1, 2)
    assert status == 1
    for t in range(10, 14):
        assert (targets[t] == targets[9]).all()
    assert not (targets[9] == ow.frame_targets(np.ones((16, 1)), 2)[0][0]).all()


def test_window_longer_than_clip_is_the_running_mean():
    A = spectrogram(10, 12, seed=5)
    means = ow.window_means(A, 1000)
    for t in range(12):
        ref = np.zeros(10)
        for u in range(t, -1, -1):
            ref = ref + A[:, u]
        assert equal(means[:, t], ref / (t + 1))


def test_mask_frames_is_the_static_lut_per_frame():
    from oracle import offline_exact as ox
    rng = np.random.default_rng(6)
    D, K, T = 16, 5, 9
    tdoas = np.linspace(-3e-4, 3e-4, D)
    argmax = rng.integers(0, D, (K, T)).astype(np.int32)
    targets = rng.integers(0, D, T).astype(np.int32)
    window = 0.05 * (tdoas[-1] - tdoas[0]) * 3
    mask = ow.mask_frames(argmax, tdoas, targets, window)
    for t in range(T):
        assert equal(mask[:, t], ox.argmax_mask(argmax[:, t], ox.tdoa_lut(tdoas, targets[t], window)))
    same = ow.mask_frames(argmax, tdoas, np.full(T, 7, np.int32), window)
    assert equal(same, ox.argmax_mask(argmax, ox.tdoa_lut(tdoas, 7, window)))


def _align(x, a=256):
    return (x + a - 1) // a * a


@pytest.mark.parametrize('N,hop,D,K,S,n', [(1024, 512, 64, 128, 2, 16000 * 4), (256, 64, 16, 32, 0, 8000), (512, 128, 128, 64, 3, 12345),
                                             (2048, 512, 1024, 1024, 1, 16000 * 30)])
def test_workspace_formula(lib, N, hop, D, K, S, n):
    """The tracked workspace is the static one followed by the angular spectrogram and the window means, (D, T) float64 each, and
    the (D, D) TDOA table, each on a 256-byte boundary."""
    from gcc_nmf_b200._lib import PipelineConfig
    cfg = PipelineConfig(N, hop, D, K, 10, S, 0.0, 1e-16, 1e-5)
    T = lib.gccnmf_stft_num_frames(n, N, hop)
    static = lib.gccnmf_pipeline_workspace_bytes(ctypes.byref(cfg), n)
    expect = _align(_align(_align(static + 8 * D * T) + 8 * D * T) + D * D)
    for w in (1, 64, 10 ** 6):
        assert lib.gccnmf_pipeline_tracked_workspace_bytes(ctypes.byref(cfg), w, n) == expect
    for w in (0, -1):
        assert lib.gccnmf_pipeline_tracked_workspace_bytes(ctypes.byref(cfg), w, n) == 0
    assert lib.gccnmf_pipeline_tracked_workspace_bytes(ctypes.byref(cfg), 8, N - 1) == 0
    assert lib.gccnmf_pipeline_tracked_workspace_bytes(None, 8, n) == 0


def test_bindings_match_the_header(lib):
    """Each new entry is declared once, bound with as many arguments as the header gives it, and exported."""
    from gcc_nmf_b200 import _lib
    text = open(os.path.join(ROOT, 'include', 'gccnmf_b200.h')).read()
    for name in NEW_ENTRIES:
        decls = re.findall(r'GCCNMF_API [\w\s\*]+?\b' + name + r'\(([^)]*)\);', text)
        assert len(decls) == 1, name
        assert len(decls[0].split(',')) == len(_lib.SIGNATURES[name][1]), name
        assert hasattr(lib, name)
    ret = {name: _lib.SIGNATURES[name][0] for name in NEW_ENTRIES}
    assert ret['gccnmf_pipeline_tracked_workspace_bytes'] is ctypes.c_size_t
    assert all(ret[n] is ctypes.c_int for n in NEW_ENTRIES if n != 'gccnmf_pipeline_tracked_workspace_bytes')
    assert _lib.SIGNATURES['gccnmf_argmax_mask_frames'][1][7] is ctypes.c_double


def test_null_handle_is_refused(lib):
    from gcc_nmf_b200._lib import GCCNMF_ERR_INVALID_ARGUMENT, PipelineConfig
    cfg = PipelineConfig(256, 64, 16, 32, 1, 0, 0.0, 1e-16, 1e-5)
    p = ctypes.c_void_p(256)
    assert lib.gccnmf_window_targets(None, p, 16, 10, 4, 2, p, p, p, None) == GCCNMF_ERR_INVALID_ARGUMENT
    assert lib.gccnmf_target_gccnmf(None, p, 9, 10, p, 16, p, 8, p, 2, p, None) == GCCNMF_ERR_INVALID_ARGUMENT
    assert lib.gccnmf_argmax_mask_frames(None, p, 8, 10, p, 16, p, 1e-5, p, p, None) == GCCNMF_ERR_INVALID_ARGUMENT
    assert lib.gccnmf_separate_tracked(None, ctypes.byref(cfg), 4, p, 8000, p, p, p, p, p, p, p, p, p, p, 1 << 20, None) == GCCNMF_ERR_INVALID_ARGUMENT
