"""CPU: stream records of the real-time engines (gccnmf_rtrec_*): record and workspace sizes against a restatement of the persistent
regions of rt_carve and of the digest workspace, their independence of S, Qd, Qe and K_max, the gccnmf_rtrec_header layout and its
prefix shared with gccnmf_record_header, the numpy content digest against a plain word loop, the bound symbols and refusals
without a device."""
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
    from gcc_nmf_b200._lib import RtConfig
    c = dict(window_size=512, hop_size=128, block_size=128, windows_per_block=1, num_atoms=64, num_tdoas=64, history_length=128,
             inference_iterations=0, sparsity_alpha=0.0, epsilon=1e-16)
    c.update(kw)
    return RtConfig(*[c[f] for f, _ in RtConfig._fields_])


def _up(x, a):
    return (x + a - 1) // a * a


def _payload(c, P):
    """The persistent regions of one slot, each 16-aligned: RtDev (11 words), the history (D x history f64), the input ring and
    max(P, 1) output rings (2 x 8 B f32 each) and, with sources, the targets (8 i32) and the status (1 i32)."""
    ring = 4 * 2 * 8 * c.block_size
    sizes = [44, 8 * c.num_tdoas * c.history_length, ring] + [ring] * max(P, 1) + ([32, 4] if P else [])
    return sum(_up(s, 16) for s in sizes)


def _record(c, P):
    return 256 + _up(_payload(c, P), 256)


def _workspace(c, P, Qd, Qe, count):
    """count records, then one 8-byte digest per 1024-word chunk of every item (the windows, max(Qd, 1) dictionaries sized at K_max
    with H0 under inference, max(Qe, 1) steering tables (D, Fp) complex64), one 8-byte digest and one K_i per item."""
    N, K, D = c.window_size, c.num_atoms, c.num_tdoas
    F = N // 2 + 1
    Fp = _up(F, 4)
    nd, ne = max(Qd, 1), max(Qe, 1)
    chunks = -(-2 * N // 1024) + nd * -(-(F * K + 2 * K * (c.inference_iterations > 0)) // 1024) + ne * -(-2 * D * Fp // 1024)
    items = 1 + nd + ne
    return _up(count * _record(c, P), 256) + _up(8 * chunks, 256) + _up(8 * items, 256) + _up(4 * items, 256)


SWEEP = [dict(), dict(window_size=1024, hop_size=256, block_size=256, num_atoms=1024, num_tdoas=128, history_length=5),
         dict(windows_per_block=3, hop_size=64, block_size=192, num_atoms=77, num_tdoas=17, history_length=1, inference_iterations=5),
         dict(window_size=2048, hop_size=512, block_size=1024, windows_per_block=2, num_atoms=4096, num_tdoas=3, inference_iterations=10),
         dict(window_size=64, hop_size=16, block_size=16, num_atoms=1, num_tdoas=1, history_length=300)]
BANKS = [(0, 0), (1, 1), (3, 2), (64, 64)]


@pytest.mark.parametrize('kw', SWEEP, ids=[str(i) for i in range(len(SWEEP))])
def test_record_sizes_follow_the_carve(kw):
    lib = _lib()
    c = _cfg(**kw)
    for P in (0, 2, 3, 8):
        assert lib.gccnmf_rtrec_record_bytes(ctypes.byref(c), P) == _record(c, P), (kw, P)
        for Qd, Qe in BANKS:
            for S, count in ((1, 1), (64, 3), (4096, 64)):
                got = lib.gccnmf_rtrec_workspace_bytes(ctypes.byref(c), S, P, Qd, Qe, count)
                assert got == _workspace(c, P, Qd, Qe, count), (kw, P, Qd, Qe, count)


@pytest.mark.parametrize('kw', SWEEP, ids=[str(i) for i in range(len(SWEEP))])
def test_record_independent_of_slots_bank_and_kmax(kw):
    lib = _lib()
    c = _cfg(**kw)
    for P in (0, 2, 8):
        want = lib.gccnmf_rtrec_record_bytes(ctypes.byref(c), P)
        for K in (1, 33, 4096):
            assert lib.gccnmf_rtrec_record_bytes(ctypes.byref(_cfg(**dict(kw, num_atoms=K))), P) == want
        rb = [lib.gccnmf_rtrec_workspace_bytes(ctypes.byref(c), S, P, Qd, Qe, 2) - lib.gccnmf_rtrec_workspace_bytes(ctypes.byref(c), S, P, Qd, Qe, 1)
              for S in (1, 7, 4096) for Qd, Qe in BANKS]
        assert all(_up(2 * want, 256) - _up(want, 256) == r for r in rb)
        # the staging of the records does not depend on S: only the bank and K_max size the digest part
        assert len({lib.gccnmf_rtrec_workspace_bytes(ctypes.byref(c), S, P, 3, 2, 5) for S in (1, 7, 4096)}) == 1


def test_configs2_record_size():
    """configs[2] (512-FFT, hop 128, B 128, nT 1, D 64, history 128): about 82 KB, 64 KiB of it the history."""
    lib = _lib()
    c = _cfg()
    assert lib.gccnmf_rtrec_record_bytes(ctypes.byref(c), 0) == 256 + _up(48 + 65536 + 8192 + 8192, 256) == 82432


def test_invalid_sizes():
    lib = _lib()
    c = _cfg()
    for P in (-1, 1, 9):
        assert lib.gccnmf_rtrec_record_bytes(ctypes.byref(c), P) == 0, P
        assert lib.gccnmf_rtrec_workspace_bytes(ctypes.byref(c), 4, P, 0, 0, 1) == 0, P
    for Qd, Qe in ((1, 0), (0, 1), (65, 1), (1, 65), (-1, -1)):
        assert lib.gccnmf_rtrec_workspace_bytes(ctypes.byref(c), 4, 0, Qd, Qe, 1) == 0, (Qd, Qe)
    for S in (0, 4097):
        assert lib.gccnmf_rtrec_workspace_bytes(ctypes.byref(c), S, 0, 0, 0, 1) == 0, S
    assert lib.gccnmf_rtrec_workspace_bytes(ctypes.byref(c), 4, 0, 0, 0, 0) == 0
    assert lib.gccnmf_rtrec_record_bytes(None, 0) == 0
    assert lib.gccnmf_rtrec_workspace_bytes(None, 1, 0, 0, 0, 1) == 0
    assert lib.gccnmf_rtrec_record_bytes(ctypes.byref(_cfg(window_size=1000)), 0) == 0
    assert lib.gccnmf_rtrec_record_bytes(ctypes.byref(_cfg(num_tdoas=129)), 0) == 0


def test_entry_points_refuse_without_handle():
    lib = _lib()
    c = _cfg()
    assert lib.gccnmf_rtrec_save_slots(None, ctypes.byref(c), 1, 0, 0, 0, None, 0, 0, 1, None, 0, None, 0, None) != 0
    assert lib.gccnmf_rtrec_load_slots(None, ctypes.byref(c), 4, 2, 3, 2, None, 0, 0, 1, None, 0, None, 0, None) != 0


def test_header_layout():
    from gcc_nmf_b200 import _lib as L
    H, R = L.RtRecordHeader, L.RecordHeader
    assert [f for f, _ in H._fields_] == ['magic', 'abi_version', 'kind', 'num_sources', 'payload_bytes', 'windows_digest', 'dictionary_digest',
                                          'steering_digest', 'dictionary_atoms', 'reserved', 'config']
    # the first 24 bytes are gccnmf_record_header's
    for f in ('magic', 'abi_version', 'kind', 'num_sources', 'payload_bytes'):
        assert (getattr(H, f).offset, getattr(H, f).size) == (getattr(R, f).offset, getattr(R, f).size), f
    assert (H.windows_digest.offset, H.dictionary_digest.offset, H.steering_digest.offset) == (24, 32, 40)
    assert (H.dictionary_atoms.offset, H.reserved.offset, H.config.offset) == (48, 52, 56)
    assert ctypes.sizeof(H) == 120 <= L.RECORD_HEADER_BYTES
    assert ctypes.sizeof(L.RtConfig) <= ctypes.sizeof(H.config.size * ctypes.c_int32)
    assert L.RECORD_KIND_RT != L.RECORD_KIND_LL
    header = open(os.path.join(ROOT, 'include', 'gccnmf_b200.h')).read()
    body = re.search(r'typedef struct gccnmf_rtrec_header \{(.*?)\} gccnmf_rtrec_header;', header, re.S).group(1)
    assert re.findall(r'(?:u?int\d+_t)\s+(\w+)(?:\[\d+\])?;', body) == [f for f, _ in H._fields_]
    assert 'int32_t config[16];' in body
    defines = dict(re.findall(r'#define (GCCNMF_RECORD_KIND_RT|GCCNMF_RTREC_\w+) (0x[0-9a-f]+ull|\d+)', header))
    assert int(defines['GCCNMF_RECORD_KIND_RT']) == L.RECORD_KIND_RT
    assert int(defines['GCCNMF_RTREC_DIGEST_CHUNK_WORDS']) == L.RTREC_DIGEST_CHUNK_WORDS == 1024
    assert int(defines['GCCNMF_RTREC_DIGEST_BASIS'].rstrip('ul'), 16) == 0xcbf29ce484222325
    assert int(defines['GCCNMF_RTREC_DIGEST_PRIME'].rstrip('ul'), 16) == 0x100000001b3


def test_header_agrees_with_bindings():
    from gcc_nmf_b200 import _lib as L
    header = open(os.path.join(ROOT, 'include', 'gccnmf_b200.h')).read()
    declared = set(re.findall(r'GCCNMF_API\s+[\w\s\*]+?\b(gccnmf_rtrec_\w+)\s*\(', header))
    bound = {n for n in L.SIGNATURES if n.startswith('gccnmf_rtrec_')}
    assert declared == bound == {'gccnmf_rtrec_record_bytes', 'gccnmf_rtrec_workspace_bytes', 'gccnmf_rtrec_save_slots',
                                 'gccnmf_rtrec_load_slots'}
    for name in bound:
        decl = re.search(r'GCCNMF_API\s+[\w\s\*]+?\b%s\s*\((.*?)\);' % name, header, re.S).group(1)
        assert len(decl.split(',')) == len(L.SIGNATURES[name][1]), name


def _fnv(words):
    h = 0xcbf29ce484222325
    for w in words:
        h = ((h ^ int(w)) * 0x100000001b3) & 0xFFFFFFFFFFFFFFFF
    return h


def _digest_loop(words):
    """The digest of include/gccnmf_b200.h, one word at a time."""
    n = len(words)
    fold = [n & 0xFFFFFFFF, n >> 32]
    for j in range(0, n, 1024):
        c = _fnv(words[j:j + 1024])
        fold += [c & 0xFFFFFFFF, c >> 32]
    return _fnv(fold)


@pytest.mark.parametrize('n', [1, 2, 1023, 1024, 1025, 2047, 2048, 2049, 3 * 1024 + 7])
def test_numpy_digest_against_word_loop(n):
    from gcc_nmf_b200.records import content_digest
    rng = np.random.RandomState(n)
    x = rng.standard_normal(n).astype(np.float32)
    words = x.view(np.uint32).tolist()
    assert content_digest(x) == _digest_loop(words)
    # split anywhere, the concatenation is what is hashed
    k = n // 3
    assert content_digest(x[:k], x[k:]) == _digest_loop(words)
    # complex64 is two words per element
    z = rng.standard_normal(n).astype(np.float32).view(np.complex64) if n % 2 == 0 else None
    if z is not None:
        assert content_digest(z) == _digest_loop(z.view(np.uint32).tolist())


def test_digest_sees_every_word():
    from gcc_nmf_b200.records import content_digest
    x = np.arange(2500, dtype=np.float32)
    base = content_digest(x)
    for i in (0, 1023, 1024, 2499):
        y = x.copy()
        y[i] += 1
        assert content_digest(y) != base, i
    assert content_digest(x[:2048]) != content_digest(x[:2048], np.zeros(0, np.float32), np.zeros(1, np.float32))


def test_steering_digest_includes_the_pad():
    from gcc_nmf_b200.realtime import slotrecords
    rng = np.random.RandomState(0)
    F, D = 257, 5
    E = (rng.standard_normal((F, D)) + 1j * rng.standard_normal((F, D))).astype(np.complex64)
    ET = np.zeros((D, 260), np.complex64)
    ET[:, :F] = E.T
    assert slotrecords.steering_digest(E) == _digest_loop(ET.view(np.uint32).ravel().tolist())


def test_mirrors_round_trip(tmp_path):
    from gcc_nmf_b200.realtime import slotrecords
    from gcc_nmf_b200 import records
    from gcc_nmf_b200._lib import RECORD_KIND_RT, RECORD_MAGIC, RtRecordHeader
    import torch
    params = [dict(targetTDOAIndex=None, epsilon=0.25, beta=1.5, noiseFloor=0.01, mode=0, separationEnabled=False, localizationEnabled=True,
                   localizationWindowSize=3, active=False),
              dict(targetTDOAIndex=12.5, epsilon=2.0, beta=1.0, noiseFloor=0.0, mode=1, separationEnabled=True, localizationEnabled=False,
                   localizationWindowSize=6, active=True)]
    data = np.zeros((2, 512), np.uint8)
    head = RtRecordHeader(magic=RECORD_MAGIC, kind=RECORD_KIND_RT)
    data[:, :ctypes.sizeof(head)] = np.frombuffer(bytes(head), np.uint8)
    rec = records.StreamRecord(RECORD_KIND_RT, 0, torch.from_numpy(data), slotrecords.params_to_mirrors(params))
    assert isinstance(rec.header(1), RtRecordHeader) and rec.header(1).kind == RECORD_KIND_RT
    rec.save(str(tmp_path / 'r.npz'))
    # records.load pins its buffer, which needs a device: read the file as it does
    with np.load(str(tmp_path / 'r.npz')) as z:
        assert int(z['kind']) == RECORD_KIND_RT and np.array_equal(z['data'], data)
        back = {k[len('mirror_'):]: z[k].copy() for k in z.files if k.startswith('mirror_')}
    assert [slotrecords.mirrors_to_params(back, i) for i in range(2)] == params
    for k, v in rec.mirrors.items():
        assert back[k].dtype == v.dtype and np.array_equal(back[k], v, equal_nan=True), k
