"""CPU: the dictionary bank of the low-latency engine (gccnmf_lldict_*).  State, record and workspace sizes against a restatement of
the carve; the header's declarations, constants and record-header layout against the bindings; refusals that need no device.  The
library's refusals of entries, K_i and shapes on a live state are in tests/test_gpu_ll_dict.py (they need a handle)."""
import ctypes
import os
import re

import numpy as np
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


SWEEP = [dict(), dict(num_tdoas=32, num_streams=5), dict(window_size=1024, hop_size=64, num_tdoas=128, num_atoms=256, num_streams=1024, hops_per_call=3),
         dict(num_atoms=100, hop_size=100, num_tdoas=4), dict(inference_iterations=5, hops_per_call=7, num_atoms=24)]


def _argmax_ws(F, T, D, K):
    """gccnmf_tdoa_argmax's workspace carve at (F, T, D, K), which the grouped argmax of a dictionary bank uses when D >= 32 and
    F >= 32: G's two bf16 planes, W's two planes, |W| sums, E^T, the candidates, C^T, W^T, the list and 4 counters."""
    if not (32 <= D <= 128 and F >= 32):
        return 0
    Fp, cap = (F + 7) & ~7, min(K * T, max(1 << 16, K * T // 8))
    used = 0
    for r in (4 * T * D * Fp, 4 * F * K, 4 * K, 16 * D * Fp, 16 * cap, 8 * T * Fp, 4 * K * Fp, 8 * cap, 16):
        used = _up(used, 256) + r
    return _up(used, 256)


@pytest.mark.parametrize('kw', SWEEP, ids=[str(i) for i in range(len(SWEEP))])
def test_state_record_and_workspace_sizes(kw):
    """The dictionary regions follow the llbank state, each 256-aligned, in slots of Kp = K rounded up to 128: W (F Kp) f32, the two
    bf16 planes (2 F Kp), |W| column sums (Kp), the refinement transpose (Kp Fp) f32, with inference ll_dict_kernel's W^T (Kp F),
    its column sums (Kp) and H0 (2 Kp), rowsum(W) (F), per entry; then the K_i table (Qd), the assignment (S), the sorted streams
    (S) and the entry starts (Qd + 1).  Records are the llbank records.  The workspace holds the payloads, one chunk digest per 1024
    words of the largest dictionary (and H0) and of each table, then the Qd + Qe digests."""
    lib = _lib()
    c = _cfg(**kw)
    S, F, K, D, inf = c.num_streams, c.window_size // 2 + 1, c.num_atoms, c.num_tdoas, c.inference_iterations > 0
    Fp, Kp = (F + 7) & ~7, _up(K, 128)
    for P in (0, 2, 8):
        for Lh in (0, 64):
            for Qe in (1, 8):
                base = lib.gccnmf_llbank_state_bytes(ctypes.byref(c), P, Lh, Qe)
                for Qd in (1, 6, 64):
                    tail = base
                    for r in (4 * Qd * F * Kp, 4 * Qd * F * Kp, 4 * Qd * Kp, 4 * Qd * Kp * Fp, 4 * Qd * Kp * F * inf, 4 * Qd * Kp * inf,
                              8 * Qd * Kp * inf, 4 * Qd * F, 4 * Qd, 4 * S, 4 * S, 4 * (Qd + 1), _argmax_ws(F, S * c.hops_per_call, D, K)):
                        tail = _up(tail, 256) + r
                    assert lib.gccnmf_lldict_state_bytes(ctypes.byref(c), P, Lh, Qd, Qe) == _up(tail, 256), (P, Lh, Qe, Qd)
                    assert lib.gccnmf_lldict_record_bytes(ctypes.byref(c), P, Lh, Qd, Qe) == \
                        lib.gccnmf_llbank_record_bytes(ctypes.byref(c), P, Lh, Qe)
                    cd, ce = -(-(F * K + 2 * K * inf) // 1024), -(-(4 * F * D) // 1024)
                    for count in (1, 3):
                        payloads = lib.gccnmf_llhist_workspace_bytes(ctypes.byref(c), P, Lh, count)
                        assert lib.gccnmf_lldict_workspace_bytes(ctypes.byref(c), P, Lh, Qd, Qe, count) == \
                            _up(payloads, 256) + _up(8 * (cd + Qe * ce), 256) + 8 * (Qd + Qe)


def test_header_agrees_with_bindings():
    from gcc_nmf_b200 import _lib as L
    from gcc_nmf_b200 import lowlatency as ll
    header = open(os.path.join(ROOT, 'include', 'gccnmf_b200.h')).read()
    declared = set(re.findall(r'GCCNMF_API\s+[\w\s\*]+?\b(gccnmf_lldict_\w+)\s*\(', header))
    bound = {n for n in L.SIGNATURES if n.startswith('gccnmf_lldict_')}
    assert declared == bound == {'gccnmf_lldict_' + n for n in (
        'state_bytes', 'init', 'load_dictionary', 'load_steering', 'assign', 'reset_streams', 'set_params', 'set_targets', 'set_window',
        'process', 'graph_create', 'export', 'record_bytes', 'workspace_bytes', 'save_streams', 'load_streams')}
    for name in bound:
        decl = re.search(r'GCCNMF_API\s+[\w\s\*]+?\b%s\s*\((.*?)\);' % name, header, re.S).group(1)
        assert len(decl.split(',')) == len(L.SIGNATURES[name][1]), name
    defines = dict(re.findall(r'#define (GCCNMF_LLDICT_\w+) (\d+)', header))
    assert int(defines['GCCNMF_LLDICT_MAX_DICTIONARIES']) == L.LLDICT_MAX_DICTIONARIES == ll.MAX_DICTIONARIES == 64
    assert int(defines['GCCNMF_LLDICT_EXPORT_DICTIONARY_ASSIGNMENT']) == ll.EXPORT_DICTIONARY_ASSIGNMENT == 27
    assert int(defines['GCCNMF_LLDICT_EXPORT_DICTIONARY_ATOMS']) == ll.EXPORT_DICTIONARY_ATOMS == 28
    # records are gccnmf_llbank_record_header's, whose config.num_atoms the engine rewrites per stream: pin the layout
    fields = [(f, getattr(L.LLBankRecordHeader, f).offset) for f, _ in L.LLBankRecordHeader._fields_]
    assert fields == [('magic', 0), ('abi_version', 4), ('kind', 8), ('num_sources', 12), ('payload_bytes', 16), ('synthesis_digest', 24),
                      ('config', 32), ('dictionary_digest', 96), ('steering_digest', 104)]
    assert ctypes.sizeof(L.LLBankRecordHeader) == 112 <= L.RECORD_HEADER_BYTES
    assert [f for f, _ in L.LLConfig._fields_][3] == 'num_atoms' and ll.ATOMS_OFFSET == 32 + 4 * 3
    struct = re.search(r'typedef struct gccnmf_llbank_record_header \{(.*?)\}', header, re.S).group(1)
    assert re.findall(r'(\w+)(?:\[\d+\])?;', struct) == [f for f, _ in L.LLBankRecordHeader._fields_]


def test_host_refusals():
    lib = _lib()
    c = _cfg()
    for Qd, Qe in ((0, 4), (-1, 4), (65, 4), (2, 0), (2, 65), (2, -1)):
        assert lib.gccnmf_lldict_state_bytes(ctypes.byref(c), 0, 0, Qd, Qe) == 0, (Qd, Qe)
        assert lib.gccnmf_lldict_record_bytes(ctypes.byref(c), 2, 8, Qd, Qe) == 0, (Qd, Qe)
        assert lib.gccnmf_lldict_workspace_bytes(ctypes.byref(c), 0, 0, Qd, Qe, 1) == 0, (Qd, Qe)
    assert lib.gccnmf_lldict_state_bytes(ctypes.byref(c), 1, 0, 2, 4) == 0
    assert lib.gccnmf_lldict_state_bytes(ctypes.byref(c), 0, 1025, 2, 4) == 0
    assert lib.gccnmf_lldict_workspace_bytes(ctypes.byref(c), 0, 0, 2, 4, 0) == 0
    assert lib.gccnmf_lldict_state_bytes(None, 0, 0, 2, 4) == 0
    # (Kmax + F) x 4 bytes of shared memory over the limit with inference
    big = _cfg(num_atoms=60000, inference_iterations=5)
    assert lib.gccnmf_lldict_state_bytes(ctypes.byref(big), 0, 0, 2, 4) == 0
    assert lib.gccnmf_lldict_state_bytes(ctypes.byref(_cfg(num_atoms=60000)), 0, 0, 2, 4) > 0
    d, e = (ctypes.c_int32 * 1)(0), (ctypes.c_int32 * 1)(0)
    assert lib.gccnmf_lldict_assign(None, ctypes.byref(c), 0, 0, 2, 4, None, 0, 0, 1, d, e, None) != 0
    assert lib.gccnmf_lldict_load_dictionary(None, ctypes.byref(c), 0, 0, 2, 4, None, 0, 0, None, 64, None, None) != 0


def test_engine_refuses_dictionary_banks_on_the_host():
    from gcc_nmf_b200 import lowlatency as ll
    W, E = np.ones((129, 64), np.float32), np.ones((129, 8), complex)
    with pytest.raises(ValueError, match='dictionary bank'):
        ll.LowLatencyEngine([W] * 65, E, np.ones(256), np.ones(256), 32)
    with pytest.raises(ValueError, match='dictionary bank'):
        ll.LowLatencyEngine([], E, np.ones(256), np.ones(256), 32)
    with pytest.raises(ValueError, match='all be'):
        ll.LowLatencyEngine([W, np.ones((65, 32), np.float32)], E, np.ones(256), np.ones(256), 32)
    with pytest.raises(ValueError, match='all be'):
        ll.LowLatencyEngine([W, np.ones((129, 0), np.float32)], E, np.ones(256), np.ones(256), 32)
