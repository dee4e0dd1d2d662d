"""CPU: the C-ABI library loads without a GPU, exports every symbol include/gccnmf_b200.h declares,
host-only helpers behave, and the product path refuses to run without a device (no CPU fallback)."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope='module')
def lib():
    import __graft_entry__ as entry
    entry.build()
    from gcc_nmf_b200 import _lib
    return _lib.load_library()


def header_symbols():
    text = open(os.path.join(ROOT, 'include', 'gccnmf_b200.h')).read()
    return sorted(set(re.findall(r'GCCNMF_API [\w\s\*]+?\b(gccnmf_\w+)\(', text)))


def test_every_declared_symbol_is_exported_and_bound(lib):
    from gcc_nmf_b200 import _lib
    names = header_symbols()
    assert len(names) >= 20
    for name in names:
        assert hasattr(lib, name), 'missing export: ' + name
    assert sorted(_lib.SIGNATURES) == names


def test_host_helpers(lib):
    assert lib.gccnmf_abi_version() == 2
    assert lib.gccnmf_stft_num_frames(160000, 1024, 512) == 311          # config 1
    assert lib.gccnmf_stft_num_frames(480000, 1024, 256) == 1872         # config 2
    assert lib.gccnmf_stft_num_frames(100, 1024, 256) < 0                # buffer too short
    assert lib.gccnmf_stft_num_frames(4096, 1024, 0) < 0                 # invalid hop
    assert lib.gccnmf_istft_length(1024, 256, 1872, 1) == 478976
    assert lib.gccnmf_istft_length(1024, 512, 311, 1) == 158720
    assert lib.gccnmf_klnmf_workspace_bytes(513, 3744, 1024) > 513 * 3744 * 4
    assert lib.gccnmf_status_string(-5).decode().startswith('no CUDA device')


def test_tdoa_argmax_host_helpers(lib):
    """gccnmf_tdoa_argmax_workspace_bytes: 256 (the float64 kernel runs, no workspace) for every shape the tensor-core argmax does
    not cover -- D not a power of two in [8, 128], K % 8 != 0, K < 64, F < 32, T D < 256 -- and a real workspace at the edges it
    does; gccnmf_tdoa_argmax_refine_capacity: min(K T, max(65536, K T / 8)) decisions."""
    ws = lib.gccnmf_tdoa_argmax_workspace_bytes
    F, T, D, K = 513, 100, 64, 128
    assert ws(F, T, D, K) > 2 * T * D * 520 * 2                         # the G planes alone: 2 x T D x Fp bf16
    for edge in [(32, T, D, K), (F, 4, 64, K), (F, 32, 8, K), (F, T, 128, K), (F, T, D, 64), (F, T, D, 72)]:
        assert ws(*edge) > 256, edge
    for uncovered in [(F, T, 48, K), (F, T, 4, K), (F, T, 256, K), (F, T, 96, K),    # D
                      (F, T, D, 132), (F, T, D, 1020),                                # K % 8 != 0
                      (F, T, D, 56), (F, T, D, 8),                                    # K < 64
                      (31, T, D, K), (1, T, D, K),                                    # F < 32
                      (F, 3, 64, K), (F, 31, 8, K), (F, 1, 128, K)]:                  # T D < 256
        assert ws(*uncovered) == 256, uncovered
    assert ws(0, T, D, K) == 0 and ws(F, T, D, 0) == 0
    cap = lib.gccnmf_tdoa_argmax_refine_capacity
    for K, T in [(1, 1), (64, 100), (128, 500), (128, 512), (128, 1024), (1024, 1872), (4096, 37494)]:
        assert cap(K, T) == min(K * T, max(65536, K * T // 8)), (K, T)
    assert cap(0, 10) == 0 and cap(10, 0) == 0


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip('GPU present')
    from gcc_nmf_b200 import _lib
    with pytest.raises(_lib.GCCNMFError):
        _lib.Handle(0)
    import gcc_nmf_b200.gccNMFFunctions as fn
    import numpy as np
    with pytest.raises(_lib.GCCNMFError):
        fn.performKLNMF(np.ones((8, 8), np.float32), 2, 1, 0)


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, 'gcc-nmf_b200')
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith('.py'):
                src = open(os.path.join(dirpath, f)).read()
                assert not re.search(r'^\s*(from|import)\s+oracle', src, re.M), f


def test_klnmf_tile_plan_fills_the_chip(lib):
    """Host-side tile planner of the TMA KL-NMF path (klnmf_tma.cu make_plan): one wave on 148 SMs at the headline shape (the planner takes the SM count),
    and sane choices at the other BASELINE.json shapes."""
    import ctypes
    out = (ctypes.c_int * 8)()
    assert lib.gccnmf_klnmf_tile_plan(148, 513, 3744, 1024, out) == 0            # config 2
    bn_wh, bn_h, bn_w, splits_w, slots, c_wh, c_h, c_w = list(out)
    assert (bn_h, bn_w, splits_w) == (208, 176, 6)
    assert bn_wh in (104, 112, 128) and c_wh == 4 * ((3744 + bn_wh - 1) // bn_wh)  # W.H: dual-N loop, 2 MMAs of N = 2 bn per k-step
    assert slots == 18 and (c_h, c_w) == (144, 144) and c_wh <= 148                # every launch is one wave of <= 148 CTAs
    assert lib.gccnmf_klnmf_tile_plan(148, 513, 622, 128, out) == 0               # config 1: few tiles -> k-splits for the numerator
    assert out[3] >= 2 and max(out[5], out[6], out[7]) <= 148
    assert lib.gccnmf_klnmf_tile_plan(148, 1025, 37494, 4096, out) == 0           # config 4: many waves, widest tiles
    assert out[0] == 256 and out[1] in (208, 256) and out[3] == 1
    for bn in (out[0], out[1], out[2]):
        assert bn in (112, 128, 176, 208, 256)
    assert lib.gccnmf_klnmf_tile_plan(148, 513, 3744, 1020, out) < 0              # K % 8 != 0: float32 SIMT path
    assert lib.gccnmf_klnmf_tile_plan(0, 513, 3744, 1024, out) < 0
    # fewer SMs -> the planner may not use more CTAs than a wave when a single-wave choice exists
    assert lib.gccnmf_klnmf_tile_plan(132, 513, 3744, 1024, out) == 0
    assert out[7] <= 132
    # F = 129 .. 136 (a 256-point FFT): the m tile of a 256-column W.H tile cannot share its columns among the SIMT tail rows (at
    # most 128 each), so the launch runs two m tiles; the planner must cost and count the same CTAs
    for F in (129, 136):
        for T2 in range(16000, 36000, 250):
            assert lib.gccnmf_klnmf_tile_plan(132, F, T2, 32, out) == 0
            assert out[5] == (2 if out[0] > 128 else 1) * -(-T2 // out[0]), (F, T2, list(out))


def test_pull_exchange_buffer_layout(lib):
    """Size of the symmetric buffer of the pull exchange (gccnmf_klnmf_step_pull): 2 x (numerator + packed row sums), 2 x row-sum slots,
    the slice-owner buffer, the arrival counters and one flag per 32 x 128 tile of U; identical on every rank when built from the largest
    shard (host logic only)."""
    F, T2, K = 513, 3744, 1024
    n = lib.gccnmf_klnmf_pull_buffer_floats(F, T2, K)
    slots = (T2 + 127) // 128
    tiles = ((F + 31) // 32) * ((K + 127) // 128)
    assert n == 2 * (F * K + K) + 2 * slots * K + F * K + 64 + (tiles + 63) // 64 * 64
    assert lib.gccnmf_klnmf_pull_buffer_floats(F, T2 + 2, K) >= n           # uneven shards: every rank uses the largest 2T
    assert lib.gccnmf_klnmf_pull_buffer_floats(1025, 4688, 4096) > 3 * 1025 * 4096
    assert lib.gccnmf_klnmf_pull_buffer_floats(0, T2, K) == 0


def test_documented_options_are_the_accepted_ones():
    """Every option gccnmf_set_option accepts (csrc/api.cu) is listed in the header's option block, and vice versa."""
    api = open(os.path.join(ROOT, 'gcc-nmf_b200', 'csrc', 'api.cu')).read()
    accepted = set(re.findall(r'strcmp\(name, "([a-z_0-9]+)"\)', api))
    hdr = open(os.path.join(ROOT, 'include', 'gccnmf_b200.h')).read()
    block = hdr[hdr.index('Options (A/B switches'):hdr.index('GCCNMF_API int gccnmf_set_option')]
    documented = set(re.findall(r'^ \*   "([a-z_0-9]+)"', block, re.M))
    assert accepted == documented, (sorted(accepted - documented), sorted(documented - accepted))
