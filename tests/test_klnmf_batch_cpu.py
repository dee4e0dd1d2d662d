"""CPU: the batched KL-NMF entry points -- workspace size, bindings, and the refusals made on the host before anything is enqueued."""
import ctypes
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


# tensor-core shapes: ragged F, 2T from 128 to 3744, K in {32, 40, 72, 128, 1024}
TC_SHAPES = [(129, 128, 32), (136, 250, 40), (200, 622, 72), (513, 622, 128), (2049, 600, 128), (513, 3744, 1024)]


def test_workspace_is_b_single_clip_carves(lib):
    for F, T2, K in TC_SHAPES:
        one = lib.gccnmf_klnmf_workspace_bytes(F, T2, K)
        assert one > 0 and one % 256 == 0
        for B in (1, 2, 3, 7, 33, 8191):
            assert lib.gccnmf_klnmf_batched_workspace_bytes(B, F, T2, K) == B * one, (F, T2, K, B)


def test_workspace_of_simt_shapes_holds_a_packed_clip(lib):
    """Off the tensor cores each clip's region also holds a packed copy of its V (the float32 path reads V at pitch T2)."""
    for F, T2, K in [(64, 100, 20), (130, 100, 24), (513, 622, 36)]:
        assert lib.gccnmf_klnmf_batched_workspace_bytes(3, F, T2, K) >= 3 * (lib.gccnmf_klnmf_workspace_bytes(F, T2, K) + 4 * F * T2)


def test_workspace_refuses_bad_sizes(lib):
    for args in [(0, 513, 622, 128), (-1, 513, 622, 128), (8192, 513, 622, 128), (2, 0, 622, 128), (2, 513, -1, 128), (2, 513, 622, 0)]:
        assert lib.gccnmf_klnmf_batched_workspace_bytes(*args) == 0, args


def test_header_prototypes_match_bindings():
    from gcc_nmf_b200 import _lib
    text = open(os.path.join(ROOT, 'include', 'gccnmf_b200.h')).read()
    ctype = {'int': ctypes.c_int, 'int64_t': ctypes.c_int64, 'size_t': ctypes.c_size_t, 'float': ctypes.c_float}
    for name in ('gccnmf_klnmf_batched_workspace_bytes', 'gccnmf_klnmf_batched'):
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
    """Host-side refusals: no handle, then (with no device to create one) every argument check answers before any launch."""
    from gcc_nmf_b200._lib import GCCNMF_OK
    buf = (ctypes.c_float * 64)()
    p = ctypes.addressof(buf)
    st = lib.gccnmf_klnmf_batched(None, p, 622, 513 * 622, 2, 513, 622, p, p, 128, 3, 0.0, 1e-16, 1, p, 256, None)
    assert st != GCCNMF_OK
    assert lib.gccnmf_last_error(None)
