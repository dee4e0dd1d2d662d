"""CPU: stream records of the low-latency engine (gccnmf_llrec_*): record and staging sizes against a restatement of the persistent
regions of the state carve, the header layout, the state sizes against a restatement of the whole carve, the header against the
bindings, and refusals without a device."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _lib():
    from gcc_nmf_b200 import _lib
    try:
        return _lib.load_library()
    except ImportError:
        pytest.skip('library not built')


def _cfg(**kw):
    from gcc_nmf_b200._lib import LLConfig
    c = dict(window_size=256, hop_size=32, hops_per_call=1, num_atoms=64, num_tdoas=16, num_streams=4, inference_iterations=0,
             sparsity_alpha=0.0, epsilon=1e-16)
    c.update(kw)
    return LLConfig(*[c[f] for f, _ in LLConfig._fields_])


def _up(x, a):
    return (x + a - 1) // a * a


def _payload(c, P):
    """The persistent regions of one stream, each 16-aligned: LLStream (24 bytes), the carried maximum (D f64), the input ring
    (2 (Q - 1) hop f32), the output ring(s) (max(P, 1) x 2 N f32) and, with sources, targets and overrides (8 i32 each) and status."""
    N, hop, D = c.window_size, c.hop_size, c.num_tdoas
    R = (-(-N // hop) - 1) * hop
    sizes = [24, 8 * D, 4 * 2 * R, 4 * max(P, 1) * 2 * N] + ([32, 32, 4] if P else [])
    return sum(_up(s, 16) for s in sizes if s)


def _state_bytes(lib, c, P):
    """ll_carve restated: every region 256-aligned, in carve order."""
    S, N, hop, C, K, D = c.num_streams, c.window_size, c.hop_size, c.hops_per_call, c.num_atoms, c.num_tdoas
    F, R, T, inf, Pm = N // 2 + 1, (-(-N // hop) - 1) * hop, S * C, c.inference_iterations > 0, max(P, 1)
    regions = [8, 24 * S, 16, 8 * N, 8 * N, 8 * 2 * F * D, 4 * F * K, 4 * K * F * inf, 4 * K * inf, 4 * 2 * K * inf, 4 * S * 2 * R,
               4 * S * Pm * 2 * N, 8 * S * D, 4 * 2 * S * (R + C * hop), 4 * 4 * F * T, 4 * 2 * F * T * inf, 4 * 2 * F * T, 8 * D * T,
               8 * D * T, 4 * T, 4 * T, 4 * K * T, 4 * K * T, 4 * Pm * (2 if inf else 1) * F * T, 4 * Pm * 4 * F * T, 4 * 2 * K * T * inf,
               4 * Pm * 2 * T * N, lib.gccnmf_wiener_apply_workspace_bytes(F) // 4 * 4, lib.gccnmf_tdoa_argmax_workspace_bytes(F, T, D, K),
               4 * S * 8 * (P > 0), 4 * S * 8 * (P > 0), 4 * S * (P > 0), 4 * T * P, 4 * P * K * T, 4 * P * K * T]
    used = 0
    for r in regions:
        used = _up(used, 256) + r
    return _up(used, 256)


SWEEP = [dict(), dict(window_size=1024, hop_size=64, num_tdoas=128, num_atoms=256, num_streams=1024, hops_per_call=3),
         dict(hop_size=24), dict(hop_size=256), dict(hop_size=100, num_tdoas=4), dict(inference_iterations=5, hops_per_call=7),
         dict(window_size=4096, hop_size=1000, num_tdoas=128, num_streams=4096)]


@pytest.mark.parametrize('kw', SWEEP, ids=[str(i) for i in range(len(SWEEP))])
def test_record_sizes_follow_the_carve(kw):
    lib = _lib()
    for P in (0, 2, 3, 8):
        c = _cfg(**kw)
        assert lib.gccnmf_llrec_record_bytes(ctypes.byref(c), P) == 256 + _up(_payload(c, P), 256), (kw, P)
        for count in (1, 3, 64):
            assert lib.gccnmf_llrec_workspace_bytes(ctypes.byref(c), P, count) == count * _payload(c, P), (kw, P, count)
        # a record depends neither on the number of streams nor on the hops per call
        other = _cfg(**dict(kw, num_streams=1, hops_per_call=2))
        assert lib.gccnmf_llrec_record_bytes(ctypes.byref(other), P) == lib.gccnmf_llrec_record_bytes(ctypes.byref(c), P)


@pytest.mark.parametrize('kw', SWEEP, ids=[str(i) for i in range(len(SWEEP))])
def test_state_sizes_unchanged(kw):
    lib = _lib()
    c = _cfg(**kw)
    assert lib.gccnmf_ll_state_bytes(ctypes.byref(c)) == _state_bytes(lib, c, 0)
    for P in (2, 3, 8):
        assert lib.gccnmf_llsep_state_bytes(ctypes.byref(c), P) == _state_bytes(lib, c, P), P


def test_invalid_sizes():
    lib = _lib()
    c = _cfg()
    for P in (-1, 1, 9):
        assert lib.gccnmf_llrec_record_bytes(ctypes.byref(c), P) == 0, P
        assert lib.gccnmf_llrec_workspace_bytes(ctypes.byref(c), P, 1) == 0, P
    assert lib.gccnmf_llrec_workspace_bytes(ctypes.byref(c), 0, 0) == 0
    assert lib.gccnmf_llrec_record_bytes(None, 0) == 0
    assert lib.gccnmf_llrec_record_bytes(ctypes.byref(_cfg(window_size=1000)), 0) == 0


def test_entry_points_refuse_without_handle():
    lib = _lib()
    c = _cfg()
    assert lib.gccnmf_llrec_save_streams(None, ctypes.byref(c), 0, None, 0, 0, 1, None, 0, None, 0, None) != 0
    assert lib.gccnmf_llrec_load_streams(None, ctypes.byref(c), 2, None, 0, 0, 1, None, 0, None, 0, None) != 0


def test_header_layout():
    from gcc_nmf_b200 import _lib as L
    H = L.RecordHeader
    assert [f for f, _ in H._fields_] == ['magic', 'abi_version', 'kind', 'num_sources', 'payload_bytes', 'synthesis_digest', 'config']
    assert (H.magic.offset, H.abi_version.offset, H.kind.offset, H.num_sources.offset) == (0, 4, 8, 12)
    assert (H.payload_bytes.offset, H.synthesis_digest.offset, H.config.offset) == (16, 24, 32)
    assert ctypes.sizeof(H) == 96 <= L.RECORD_HEADER_BYTES
    assert L.RECORD_MAGIC.to_bytes(4, 'little') == b'GCSR'
    assert ctypes.sizeof(L.LLConfig) <= ctypes.sizeof(H.config.size * ctypes.c_int32)
    header = open(os.path.join(ROOT, 'include', 'gccnmf_b200.h')).read()
    body = re.search(r'typedef struct gccnmf_record_header \{(.*?)\} gccnmf_record_header;', header, re.S).group(1)
    assert re.findall(r'(?:u?int\d+_t)\s+(\w+)(?:\[\d+\])?;', body) == [f for f, _ in H._fields_]
    assert 'int32_t config[16];' in body
    defines = dict(re.findall(r'#define (GCCNMF_RECORD_\w+) (0x[0-9a-f]+u|\d+)', header))
    assert int(defines['GCCNMF_RECORD_MAGIC'].rstrip('u'), 16) == L.RECORD_MAGIC
    assert int(defines['GCCNMF_RECORD_KIND_LL']) == L.RECORD_KIND_LL
    assert int(defines['GCCNMF_RECORD_HEADER_BYTES']) == L.RECORD_HEADER_BYTES


def test_header_agrees_with_bindings():
    from gcc_nmf_b200 import _lib as L
    header = open(os.path.join(ROOT, 'include', 'gccnmf_b200.h')).read()
    declared = set(re.findall(r'GCCNMF_API\s+[\w\s\*]+?\b(gccnmf_llrec_\w+)\s*\(', header))
    bound = {n for n in L.SIGNATURES if n.startswith('gccnmf_llrec_')}
    assert declared == bound == {'gccnmf_llrec_record_bytes', 'gccnmf_llrec_workspace_bytes', 'gccnmf_llrec_save_streams',
                                 'gccnmf_llrec_load_streams'}
    for name in bound:
        decl = re.search(r'GCCNMF_API\s+[\w\s\*]+?\b%s\s*\((.*?)\);' % name, header, re.S).group(1)
        assert len(decl.split(',')) == len(L.SIGNATURES[name][1]), name

