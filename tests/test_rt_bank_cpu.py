"""CPU: the host side of the real-time path over a bank of dictionaries and steering tables (gccnmf_rtbank_*): state sizing,
argument checks and no CPU fallback."""
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


def _align(n):
    return (n + 255) // 256 * 256


CONFIGS = (dict(), dict(num_tdoas=16, windows_per_block=4, hop_size=32), dict(inference_iterations=0, num_atoms=200))


@pytest.mark.parametrize('kw', CONFIGS)
def test_empty_bank_is_the_rtm_and_rtsep_layout(lib, kw):
    cfg = _cfg(**kw)
    for S in (1, 7, 256):
        assert lib.gccnmf_rtbank_state_bytes(ctypes.byref(cfg), S, 0, 0, 0) == lib.gccnmf_rtm_state_bytes(ctypes.byref(cfg), S) > 0
        for P in (2, 3, 8):
            assert lib.gccnmf_rtbank_state_bytes(ctypes.byref(cfg), S, P, 0, 0) == lib.gccnmf_rtsep_state_bytes(ctypes.byref(cfg), S, P) > 0


@pytest.mark.parametrize('kw', CONFIGS)
def test_state_grows_as_the_carve_says(lib, kw):
    """Each further dictionary entry adds W, W^T, recV, colsumW and H0 at K_max (256-aligned each); each further steering entry
    adds E^T; a bank adds the K_i table and the sorted slot order to the shared region and one 256-byte word block per slot."""
    cfg = _cfg(**kw)
    K, D, N = cfg.num_atoms, cfg.num_tdoas, cfg.window_size
    F = N // 2 + 1
    Fp = (F + 3) & ~3
    dict_entry = _align(F * K * 4) + _align(K * Fp * 4) + _align(F * 4) + _align(K * 4) + _align(K * 2 * 4)
    steer_entry = _align(D * Fp * 8)

    def size(S, P, Qd, Qe):
        return lib.gccnmf_rtbank_state_bytes(ctypes.byref(cfg), S, P, Qd, Qe)
    for P in (0, 3):
        base = size(4, P, 1, 1)
        assert size(4, P, 2, 1) - base == dict_entry
        assert size(4, P, 5, 1) - base == 4 * dict_entry
        assert size(4, P, 1, 2) - base == steer_entry
        assert size(4, P, 64, 64) - base == 63 * (dict_entry + steer_entry)
        per_slot = size(5, P, 1, 1) - base
        plain = lib.gccnmf_rtm_state_bytes(ctypes.byref(cfg), 5) - lib.gccnmf_rtm_state_bytes(ctypes.byref(cfg), 4) if P == 0 else \
            lib.gccnmf_rtsep_state_bytes(ctypes.byref(cfg), 5, P) - lib.gccnmf_rtsep_state_bytes(ctypes.byref(cfg), 4, P)
        assert per_slot - plain == 256                            # the (dictionary, steering) word, after the slot's regions
        for S in (1, 9, 4096):
            assert size(S, P, 3, 2) - size(1, P, 3, 2) == (S - 1) * per_slot + _align(4 * S) - _align(4)


def test_state_bytes_rejects_invalid_banks(lib):
    cfg = _cfg()
    for Qd, Qe in ((1, 0), (0, 1), (65, 1), (1, 65), (-1, 1), (1, -1)):
        assert lib.gccnmf_rtbank_state_bytes(ctypes.byref(cfg), 4, 0, Qd, Qe) == 0, (Qd, Qe)
    assert lib.gccnmf_rtbank_state_bytes(ctypes.byref(cfg), 4, 1, 2, 2) == 0
    assert lib.gccnmf_rtbank_state_bytes(ctypes.byref(cfg), 4097, 0, 2, 2) == 0
    assert lib.gccnmf_rtbank_state_bytes(None, 4, 0, 2, 2) == 0
    assert lib.gccnmf_rtbank_state_bytes(ctypes.byref(cfg), 4, 0, 64, 64) > 0


def test_bank_engine_validates_shapes_and_has_no_cpu_fallback(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip('GPU present')
    from gcc_nmf_b200 import _lib
    from gcc_nmf_b200.realtime.multistream import MultiStreamRealtimeEngine
    F, N = 257, 512
    win = np.ones(N, np.float32)
    Ws = [np.ones((F, 16), np.float32), np.ones((F, 40), np.float32)]
    Es = [np.ones((F, 8), np.complex64), np.ones((F, 8), np.complex64)]
    with pytest.raises(ValueError):              # D differs
        MultiStreamRealtimeEngine(Ws, [Es[0], np.ones((F, 9), np.complex64)], win, win, 128, 128, 1, 4)
    with pytest.raises(ValueError):              # F differs
        MultiStreamRealtimeEngine([Ws[0], np.ones((F + 1, 4), np.float32)], Es, win, win, 128, 128, 1, 4)
    with pytest.raises(ValueError):              # too many entries
        MultiStreamRealtimeEngine(Ws * 33, Es, win, win, 128, 128, 1, 4)
    with pytest.raises(_lib.GCCNMFError):
        MultiStreamRealtimeEngine(Ws, Es, win, win, 128, 128, 1, 4)


def test_header_and_signatures_list_the_bank_family():
    import os
    import re
    from gcc_nmf_b200 import _lib
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    header = open(os.path.join(root, 'include', 'gccnmf_b200.h')).read()
    declared = set(re.findall(r'GCCNMF_API\s+[\w\s\*]+?\b(gccnmf_rtbank_\w+)\s*\(', header))
    bound = {n for n in _lib.SIGNATURES if n.startswith('gccnmf_rtbank_')}
    assert declared == bound and len(bound) == 12


def test_bank_argument_checks():
    """K_i above K_max, F mismatch, entries outside the bank and malformed assignments are rejected before anything is sent."""
    from gcc_nmf_b200.realtime import multistream as ms
    F = 257
    assert ms.check_bank_dictionary(np.ones((F, 40)), F, 64).shape == (F, 40)
    assert ms.check_bank_dictionary(np.ones((F, 64)), F, 64).dtype == np.float32
    for bad in (np.ones((F, 65)), np.ones((F, 0)), np.ones((F + 1, 16)), np.ones(F)):
        with pytest.raises(ValueError):
            ms.check_bank_dictionary(bad, F, 64)
    assert ms.check_bank_index(2, 3, 'dictionary') == 2
    for bad in (-1, 3, 64):
        with pytest.raises(ValueError):
            ms.check_bank_index(bad, 3, 'dictionary')
    assert ms.check_bank_entries(None, 3, 2, 'steering') == [-1, -1, -1]
    assert ms.check_bank_entries(1, 2, 2, 'steering') == [1, 1]
    assert ms.check_bank_entries([0, -1, 4], 3, 5, 'dictionary') == [0, -1, 4]
    for values, count, entries in (([0, 5], 2, 5),       # outside the bank
                                   ([-2], 1, 5),         # below -1
                                   ([0, 1, 2], 2, 3),    # three values for two slots
                                   ([0.5], 1, 5)):       # not an integer
        with pytest.raises(ValueError):
            ms.check_bank_entries(values, count, entries, 'dictionary')
