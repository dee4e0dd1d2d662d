"""CPU: the steering bank of the low-latency engine (gccnmf_llbank_*).  State, record and workspace sizes against a restatement of
the carve (Qe = 0 giving the llhist sizes for every (P, Lh)); the header's declarations against the bindings; the numpy content
digest of a complex128 table against a plain loop; and refusals that need no device."""
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


SWEEP = [dict(), dict(window_size=1024, hop_size=64, num_tdoas=128, num_atoms=256, num_streams=1024, hops_per_call=3),
         dict(hop_size=100, num_tdoas=4), dict(inference_iterations=5, hops_per_call=7)]


@pytest.mark.parametrize('kw', SWEEP, ids=[str(i) for i in range(len(SWEEP))])
def test_state_record_and_workspace_sizes(kw):
    """Qe = 0 is llhist; Qe >= 1 grows E to Qe tables in place and appends the transposed tables (Qe, D, Fp) complex128, the
    assignment (S), the sorted streams (S) and the entry starts (Qe + 1), each 256-aligned.  Records keep the llhist payload; the
    workspace adds one digest per 1024-word chunk of the dictionary and of each table, then the 1 + Qe item digests."""
    lib = _lib()
    c = _cfg(**kw)
    S, F, K, D, inf = c.num_streams, c.window_size // 2 + 1, c.num_atoms, c.num_tdoas, c.inference_iterations > 0
    Fp = (F + 7) & ~7
    for P in (0, 2, 8):
        for Lh in (0, 5, 64):
            base = lib.gccnmf_llhist_state_bytes(ctypes.byref(c), P, Lh)
            rec = lib.gccnmf_llhist_record_bytes(ctypes.byref(c), P, Lh)
            assert lib.gccnmf_llbank_state_bytes(ctypes.byref(c), P, Lh, 0) == base
            assert lib.gccnmf_llbank_record_bytes(ctypes.byref(c), P, Lh, 0) == rec
            for count in (1, 3):
                assert lib.gccnmf_llbank_workspace_bytes(ctypes.byref(c), P, Lh, 0, count) == \
                    lib.gccnmf_llhist_workspace_bytes(ctypes.byref(c), P, Lh, count)
            for Qe in (1, 8, 64):
                # E's region grows from 1 to Qe tables; everything after it moves by the growth (rounded to 256)
                grow = _up(16 * F * D * Qe, 256) - _up(16 * F * D, 256)
                tail = _up(base, 256)
                for r in (16 * Qe * D * Fp, 4 * S, 4 * S, 4 * (Qe + 1)):
                    tail = _up(tail, 256) + r
                want = _up(tail + grow, 256)
                assert lib.gccnmf_llbank_state_bytes(ctypes.byref(c), P, Lh, Qe) == want, (P, Lh, Qe)
                assert lib.gccnmf_llbank_record_bytes(ctypes.byref(c), P, Lh, Qe) == rec
                cd, ce = -(-(F * K + 2 * K * inf) // 1024), -(-(4 * F * D) // 1024)
                for count in (1, 3):
                    payloads = lib.gccnmf_llhist_workspace_bytes(ctypes.byref(c), P, Lh, count)
                    assert lib.gccnmf_llbank_workspace_bytes(ctypes.byref(c), P, Lh, Qe, count) == \
                        _up(payloads, 256) + _up(8 * (cd + Qe * ce), 256) + 8 * (1 + Qe)


def test_header_agrees_with_bindings():
    from gcc_nmf_b200 import _lib as L
    from gcc_nmf_b200 import lowlatency as ll
    header = open(os.path.join(ROOT, 'include', 'gccnmf_b200.h')).read()
    declared = set(re.findall(r'GCCNMF_API\s+[\w\s\*]+?\b(gccnmf_llbank_\w+)\s*\(', header))
    bound = {n for n in L.SIGNATURES if n.startswith('gccnmf_llbank_')}
    assert declared == bound == {'gccnmf_llbank_' + n for n in (
        'state_bytes', 'init', 'load_steering', 'assign', 'reset_streams', 'set_params', 'set_targets', 'set_window', 'process',
        'graph_create', 'export', 'record_bytes', 'workspace_bytes', 'save_streams', 'load_streams')}
    for name in bound:
        decl = re.search(r'GCCNMF_API\s+[\w\s\*]+?\b%s\s*\((.*?)\);' % name, header, re.S).group(1)
        assert len(decl.split(',')) == len(L.SIGNATURES[name][1]), name
    defines = dict(re.findall(r'#define (GCCNMF_(?:LLBANK|RECORD_KIND)_\w+) (\d+)', header))
    assert int(defines['GCCNMF_LLBANK_MAX_STEERINGS']) == L.LLBANK_MAX_STEERINGS == ll.MAX_STEERINGS == 64
    assert int(defines['GCCNMF_LLBANK_EXPORT_ASSIGNMENT']) == ll.EXPORT_ASSIGNMENT == 26
    assert int(defines['GCCNMF_RECORD_KIND_LLBANK']) == L.RECORD_KIND_LLBANK
    assert len({L.RECORD_KIND_LL, L.RECORD_KIND_RT, L.RECORD_KIND_LLBANK}) == 3
    # the bank header is gccnmf_record_header's fields, then the two digests; it fits the 256 header bytes
    assert [f for f, _ in L.LLBankRecordHeader._fields_[:len(L.RecordHeader._fields_)]] == [f for f, _ in L.RecordHeader._fields_]
    assert L.LLBankRecordHeader.dictionary_digest.offset == ctypes.sizeof(L.RecordHeader)
    assert ctypes.sizeof(L.LLBankRecordHeader) <= L.RECORD_HEADER_BYTES


def _plain_digest(table):
    """The chunked FNV-1a 64 of include/gccnmf_b200.h over the table's bytes as 32-bit words, one word at a time."""
    words = [int(w) for w in np.ascontiguousarray(table).reshape(-1).view(np.uint32)]
    M = (1 << 64) - 1

    def fnv(h, ws):
        for w in ws:
            h = ((h ^ w) * 0x100000001b3) & M
        return h
    chunks = [fnv(0xcbf29ce484222325, words[i:i + 1024]) for i in range(0, len(words), 1024)]
    fold = [len(words) & 0xFFFFFFFF, len(words) >> 32]
    for c in chunks:
        fold += [c & 0xFFFFFFFF, c >> 32]
    return fnv(0xcbf29ce484222325, fold)


@pytest.mark.parametrize('F,D', [(129, 16), (33, 4), (513, 8)])
def test_content_digest_of_a_steering_table(F, D):
    from gcc_nmf_b200 import gccNMFFunctions as fn
    from gcc_nmf_b200.records import content_digest
    E = fn.getExpJOmegaTau(fn.getFrequenciesInHz(16000, F), fn.getTDOAsInSeconds(0.1, D))
    assert E.dtype == np.complex128 and E.shape == (F, D)
    d = content_digest(E)
    assert d == _plain_digest(E)
    assert d == content_digest(E.view(np.float64))                      # the bytes as stored on the device
    E2 = E.copy()
    E2[F // 2, D - 1] = np.nextafter(E2[F // 2, D - 1].real, 2.0) + 1j * E2[F // 2, D - 1].imag
    assert content_digest(E2) != d


def test_host_refusals():
    lib = _lib()
    c = _cfg()
    for Qe in (-1, 65, 1000):
        assert lib.gccnmf_llbank_state_bytes(ctypes.byref(c), 0, 0, Qe) == 0, Qe
        assert lib.gccnmf_llbank_record_bytes(ctypes.byref(c), 2, 8, Qe) == 0, Qe
        assert lib.gccnmf_llbank_workspace_bytes(ctypes.byref(c), 0, 0, Qe, 1) == 0, Qe
    assert lib.gccnmf_llbank_state_bytes(ctypes.byref(c), 1, 0, 4) == 0
    assert lib.gccnmf_llbank_state_bytes(ctypes.byref(c), 0, 1025, 4) == 0
    assert lib.gccnmf_llbank_workspace_bytes(ctypes.byref(c), 0, 0, 4, 0) == 0
    assert lib.gccnmf_llbank_state_bytes(None, 0, 0, 4) == 0
    e = (ctypes.c_int32 * 1)(0)
    assert lib.gccnmf_llbank_assign(None, ctypes.byref(c), 0, 0, 4, None, 0, 0, 1, e, None) != 0
    assert lib.gccnmf_llbank_load_steering(None, ctypes.byref(c), 0, 0, 4, None, 0, 0, None, None) != 0
    assert lib.gccnmf_llbank_save_streams(None, ctypes.byref(c), 0, 0, 4, None, 0, 0, 1, None, 0, None, 0, None) != 0


def test_engine_refuses_banks_on_the_host():
    from gcc_nmf_b200 import lowlatency as ll
    W, E = np.ones((129, 64), np.float32), np.ones((129, 8), complex)
    with pytest.raises(ValueError, match='steering bank'):
        ll.LowLatencyEngine(W, [E] * 65, np.ones(256), np.ones(256), 32)
    with pytest.raises(ValueError, match='all be'):
        ll.LowLatencyEngine(W, [E, np.ones((65, 8), complex)], np.ones(256), np.ones(256), 32)
