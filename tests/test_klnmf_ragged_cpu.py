"""CPU: the ragged KL-NMF entry points -- workspace size, bindings, the refusals made on the host before anything is enqueued -- and the
seeded-prefix property of the initial H that lets one draw serve clips of every length."""
import ctypes
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TABLE_PER_CLIP, TABLE_EXTRA = 1280, 256


@pytest.fixture(scope='module')
def lib():
    import __graft_entry__ as entry
    entry.build()
    from gcc_nmf_b200 import _lib
    return _lib.load_library()


def lengths(*t2):
    return (ctypes.c_int * len(t2))(*t2)


def test_workspace_is_table_plus_each_clips_region(lib):
    """A per-call table of 1280 B + 256 bytes, then each clip's region of a batched run on its own shape: nothing is padded to the
    longest clip, and at tensor-core shapes each region is the single-clip workspace."""
    for F, K, t2 in [(513, 128, (122, 130, 622, 1874, 622)), (513, 1024, (250, 1250, 3744)), (200, 72, (622,)), (64, 20, (100, 37))]:
        got = lib.gccnmf_klnmf_ragged_workspace_bytes(len(t2), F, lengths(*t2), K)
        regions = [lib.gccnmf_klnmf_batched_workspace_bytes(1, F, t, K) for t in t2]
        assert got == TABLE_PER_CLIP * len(t2) + TABLE_EXTRA + sum(regions), (F, K, t2)
        for t, r in zip(t2, regions):
            if t >= 128 and F >= 128 and K % 8 == 0 and K >= 32:         # tensor-core shapes
                assert r == lib.gccnmf_klnmf_workspace_bytes(F, t, K)
    many = lengths(*([622] * 8191))
    assert lib.gccnmf_klnmf_ragged_workspace_bytes(8191, 513, many, 128) == \
        8191 * (TABLE_PER_CLIP + lib.gccnmf_klnmf_workspace_bytes(513, 622, 128)) + TABLE_EXTRA


def test_workspace_refuses_bad_sizes(lib):
    t2 = lengths(622, 300)
    for B, F, T, K in [(0, 513, t2, 128), (-1, 513, t2, 128), (8192, 513, lengths(*([622] * 8192)), 128), (2, 0, t2, 128), (2, 513, t2, 0),
                       (2, 513, None, 128), (2, 513, lengths(622, 0), 128), (2, 513, lengths(-1, 622), 128)]:
        assert lib.gccnmf_klnmf_ragged_workspace_bytes(B, F, T, K) == 0, (B, F, K)


def test_header_prototypes_match_bindings():
    from gcc_nmf_b200 import _lib
    text = open(os.path.join(ROOT, 'include', 'gccnmf_b200.h')).read()
    ctype = {'int': ctypes.c_int, 'int64_t': ctypes.c_int64, 'size_t': ctypes.c_size_t, 'float': ctypes.c_float}
    for name in ('gccnmf_klnmf_ragged_workspace_bytes', 'gccnmf_klnmf_ragged'):
        m = re.search(r'GCCNMF_API (\w+) %s\(([^)]*)\)' % name, text)
        assert m, name
        params = [p.strip() for p in m.group(2).split(',')]
        restype, argtypes = _lib.SIGNATURES[name]
        assert restype == ctype[m.group(1)]
        assert len(params) == len(argtypes), name
        for p, t in zip(params, argtypes):
            base = p.rsplit(' ', 1)[0].replace('const ', '').strip()
            if '*' in p:
                assert t in (ctypes.c_void_p,), (name, p)
            else:
                assert t == ctype[base], (name, p, t)


def test_refusals_without_a_device(lib):
    """No handle: the call answers before any launch."""
    from gcc_nmf_b200._lib import GCCNMF_OK
    buf = (ctypes.c_float * 64)()
    p = ctypes.addressof(buf)
    V = (ctypes.c_void_p * 2)(p, p)
    ld = (ctypes.c_int64 * 2)(622, 300)
    st = lib.gccnmf_klnmf_ragged(None, V, ld, lengths(622, 300), 2, 513, p, V, 128, 3, 0.0, 1e-16, 1, p, 1 << 30, None)
    assert st != GCCNMF_OK
    assert lib.gccnmf_last_error(None)


@pytest.mark.parametrize('seed', [0, 7])
def test_initial_h_is_a_prefix_of_the_longest_draw(seed):
    """W0 does not depend on T2 and H0(T2) is the first K T2 values drawn after W0: one draw at the longest clip serves all."""
    from gcc_nmf_b200.gccNMFFunctions import _seededInit
    F, K, eps = 513, 128, 1e-16
    W_long, H_long = _seededInit(F, 1874, K, eps, seed)
    for T2 in (1, 90, 622, 1873, 1874):
        W0, H0 = _seededInit(F, T2, K, eps, seed)
        assert np.array_equal(W0, W_long)
        assert np.array_equal(H0, H_long.reshape(-1)[:K * T2].reshape(K, T2)), T2
