"""CPU: the host side of the multi-stream real-time path (gccnmf_rtm_*): state sizing and no CPU fallback."""
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


def test_state_bytes_grows_linearly_in_streams(lib):
    cfg = _cfg()
    sizes = [lib.gccnmf_rtm_state_bytes(ctypes.byref(cfg), s) for s in (1, 2, 3, 8, 64, 1024)]
    assert all(v > 0 for v in sizes)
    per_slot = sizes[1] - sizes[0]
    assert per_slot > 0 and per_slot % 256 == 0
    for s, v in zip((1, 2, 3, 8, 64, 1024), sizes):
        assert v == sizes[0] + (s - 1) * per_slot
    assert sizes[0] >= lib.gccnmf_rt_state_bytes(ctypes.byref(cfg))
    # a slot holds at least its rings, its GCC-PHAT history and its GCC rows
    assert per_slot >= 4 * 2 * 8 * 128 * 2 + 8 * 64 * 128 + 4 * 64 * 257


def test_state_bytes_rejects_invalid_input(lib):
    cfg = _cfg()
    assert lib.gccnmf_rtm_state_bytes(ctypes.byref(cfg), 0) == 0
    assert lib.gccnmf_rtm_state_bytes(ctypes.byref(cfg), -3) == 0
    assert lib.gccnmf_rtm_state_bytes(None, 4) == 0
    for bad in (dict(window_size=500), dict(window_size=0), dict(num_tdoas=129), dict(windows_per_block=9), dict(num_atoms=0),
                dict(history_length=0), dict(block_size=16)):
        assert lib.gccnmf_rtm_state_bytes(ctypes.byref(_cfg(**bad)), 4) == 0, bad


def test_slot_params_layout_matches_header(lib):
    from gcc_nmf_b200._lib import RtmSlotParams
    assert ctypes.sizeof(RtmSlotParams) == 40
    assert [f[0] for f in RtmSlotParams._fields_] == ['target_index', 'set_target', 'epsilon', 'beta', 'noise_floor', 'mode',
                                                     'separation_enabled', 'localization_enabled', 'localization_window', 'active']


def test_multistream_engine_has_no_cpu_fallback(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip('GPU present')
    from gcc_nmf_b200 import _lib
    from gcc_nmf_b200.realtime.multistream import MultiStreamRealtimeEngine
    F, K, D, N = 257, 16, 8, 512
    W = np.ones((F, K), np.float32)
    E = np.ones((F, D), np.complex64)
    with pytest.raises(_lib.GCCNMFError):
        MultiStreamRealtimeEngine(W, E, np.ones(N, np.float32), np.ones(N, np.float32), 128, 128, 1, 4)
