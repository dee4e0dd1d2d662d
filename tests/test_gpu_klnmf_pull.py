"""GPU, one device: the pull exchange of the frame-sharded KL-NMF loop (gccnmf_klnmf_step_pull, csrc/klnmf_tma.cu) run at
world = 1, through distributed.klnmf_sharded_pull, in every form: one-shot (form 0) and two-shot (form 1), each with the numerator
packed by tma_pack_numer_kernel or written straight into the exchange buffer by the cluster-reduced contraction (direct), and the
exchange inside the W update (form 2).

At world 1 one zeroed device buffer serves as bases[0].  Every kernel of every form runs -- the pack with its peer signal,
tma_reduce_pull_kernel, tma_apply_w_kernel<kApplyPull> / <kApplyPullOwner>, tma_apply_w_exchange_kernel, G2's epilogue writing
the exchange row-sum slots and G4's cluster-reduced contraction writing the numerator and signalling from its last CTA -- and each
wait is met by work earlier in the same stream.  To keep it so, every (form, direct, option set) gets a fresh zeroed buffer, a
buffer is never shared between forms (form 2 never advances counter 0, form 0 never counter 1), epoch is the number of iterations
already run on the buffer, the test never writes counters or flags, and direct and form 2 are only asked for where
gccnmf_klnmf_pull_supported offers them.

Bit-identical to h.klnmf wherever the additions happen in the same order, which at world 1 holds for:
  - every direct form and form 2: the numerator is the contraction's own sum (one cluster-reduced slab, or the k-split slabs summed
    in split order, as the single-GPU W update sums them), and the W update reads the row-sum slots in the same 8 strided groups;
    the slots between the plan's count and max_rowsum_slots(layout_T2) are zero, and x + 0 = x;
  - the two-shot slice reduction: at world 1 it is acc = v[0], a copy;
  - packed forms with at most 8 row-sum slots: the pack adds the slots in sequence, 0 + s0 + s1 + ..., and the W update adds its
    8 strided groups in group order -- with one slot per group that is the same sequence (test_building_blocks_on_tensor_cores
    relies on the same fact).  With more than 8 slots the orders differ, so those runs are held to the float64 bars only.
Every run is also held to the float64 iteration of tests/test_gpu_klnmf.py, element by element, with its bars."""
import contextlib
import ctypes
import types

import numpy as np
import pytest

from test_gpu_klnmf import BOUNDS, DEFAULT_OPTIONS, Records, check, expected_ctas, make_inputs, options, reference, run, sm_count, tile_plan  # noqa: F401

pytestmark = pytest.mark.gpu

PULL_BIT, DIRECT_BIT, FORM2_BIT = 1, 2, 4      # gccnmf_klnmf_pull_supported

# (F, T2, K): what each shape reaches
SHAPES = [
    (200, 622, 72),      # numerator k-splits >= 2, at most 8 row-sum slots
    (136, 2500, 40),     # more than 8 row-sum slots, K < 128
    (263, 1001, 200),    # SIMT tail rows, K % 128 != 0
    (513, 468, 1024),    # an 8-way frame shard of configs[1]: the W update's 136 tiles, form 2's residency condition.  On a
                         # 132-SM H100 only the packed forms run here (136 tiles > one resident wave, and the numerator's 3-CTA
                         # clusters do not all fit): test_refusals_launch_nothing checks that direct and form 2 are refused
]
WORST = {}
COVERED = set()


@pytest.fixture(scope='module')
def h():
    from gcc_nmf_b200._lib import default_handle
    hd = default_handle()
    yield hd
    for name, value in DEFAULT_OPTIONS.items():
        hd.set_option(name, value)


# ------------------------------------------------------------------------------------------------ buffer layout
def max_rowsum_slots(T2):
    return -(-T2 // 128)


def pull_layout(h, F, layout_T2, K):
    """Offsets (floats) of the exchange buffer, as tests/test_cabi_cpu.py::test_pull_exchange_buffer_layout pins its size:
    numerator + packed row sums x 2 parities | row-sum slots x 2 | slice-owner buffer | 64 floats of counters | one flag per tile."""
    fk, rs = F * K, max_rowsum_slots(layout_T2) * K
    L = types.SimpleNamespace(numer=(0, fk + K), rowsum=(2 * (fk + K), 2 * (fk + K) + rs))
    L.reduced = L.rowsum[1] + rs
    L.counters = L.reduced + fk
    L.flags = L.counters + 64
    L.tiles = -(-F // 32) * -(-K // 128)
    L.total = L.flags + -(-L.tiles // 64) * 64
    assert L.total == h.lib.gccnmf_klnmf_pull_buffer_floats(F, layout_T2, K)
    return L


def new_exchange(h, F, layout_T2, K, form, direct):
    """World-1 stand-in for distributed.PullExchange: one fresh zeroed buffer as bases[0]."""
    import torch
    buf = torch.zeros(h.lib.gccnmf_klnmf_pull_buffer_floats(F, layout_T2, K), dtype=torch.float32, device=h.device)
    return types.SimpleNamespace(buffer=buf, bases=(ctypes.c_void_p * 1)(buf.data_ptr()), rank=0, world=1, layout_T2=layout_T2,
                                 two_shot=form, direct=bool(direct), epoch=0)


def run_pull(h, px, V, W0, H0, iters, alpha=0.0, eps=1e-16, records=None, fill=None):
    """distributed.klnmf_sharded_pull on copies of the inputs -> (W, H) numpy; fill: byte written over the cached workspace first."""
    import torch
    from gcc_nmf_b200 import distributed
    F, T2 = V.shape
    K = W0.shape[1]
    Vd, W, H = h.to_device(V), h.to_device(W0.copy()), h.to_device(H0.copy())
    if fill is not None:
        h._klnmf_ws(F, T2, K).fill_(fill)
    with records if records is not None else contextlib.nullcontext():
        distributed.klnmf_sharded_pull(h, px, Vd, W, H, iters, alpha, eps)
    torch.cuda.synchronize()
    return W.cpu().numpy(), H.cpu().numpy()


def assert_buffer_state(h, px, F, T2, K, n, slots):
    """Counters, flags, row-sum slots and the slice-owner buffer after n iterations on this buffer."""
    import torch
    L = pull_layout(h, F, px.layout_T2, K)
    u32 = px.buffer.view(torch.int32).cpu().numpy()
    buf = px.buffer.cpu().numpy()
    form, direct = px.two_shot, px.direct
    counters, flags = u32[L.counters:L.counters + 2], u32[L.flags:L.total]
    if form == 2:
        assert list(counters) == [0, 0], counters
        assert (flags[:L.tiles] == n).all() and (flags[L.tiles:] == 0).all(), (n, np.unique(flags[:L.tiles]))
    else:
        assert list(counters) == [n, n if form == 1 else 0], (form, n, counters)
        assert (flags == 0).all()
    rs = buf[L.rowsum[0]:L.reduced].reshape(2, max_rowsum_slots(px.layout_T2), K)
    if direct or form == 2:
        assert (rs[:, slots:] == 0).all(), 'row-sum slots past the plan\'s %d written' % slots
        for parity in range(min(n, 2)):
            assert (rs[parity, :slots] > 0).all(), ('row-sum slots of parity %d not written' % parity)
    else:
        assert (rs == 0).all(), 'a packed form wrote the row-sum slot region'
    reduced = buf[L.reduced:L.counters]
    if form == 1:     # acc = v[0]: the slice sum of the last iteration is a copy of its numerator
        last = L.numer[(n - 1) & 1]
        assert np.array_equal(reduced, buf[last:last + F * K])
    else:
        assert (reduced == 0).all()


# ------------------------------------------------------------------------------------------------ cases
def case(form, direct, opts=None, alpha=0.0, eps=1e-16, tag=''):
    return types.SimpleNamespace(form=form, direct=bool(direct), opts=dict(opts or {}), alpha=alpha, eps=eps, tag=tag)


def case_name(c):
    return 'form %d %s%s%s' % (c.form, 'direct' if c.direct else 'packed' if c.form < 2 else '',
                               ''.join(' %s=%d' % kv for kv in sorted(c.opts.items())), (' ' + c.tag) if c.tag else '')


def shape_cases(h, sm, shape, extras=True):
    """Every form this card offers at `shape`: direct, packed from k-split slabs (w_cluster_reduce 0), packed from the
    contraction's single slab (pull_force_pack 1 for form 0, direct = 0 for form 1) and form 2 from either."""
    F, T2, K = shape
    bits = h.lib.gccnmf_klnmf_pull_supported(h.h, F, T2, K)
    assert bits & PULL_BIT, (shape, bits)
    splits = tile_plan(h, sm, F, T2, K)[3]
    out = []
    for form in (0, 1):
        if bits & DIRECT_BIT:
            out.append(case(form, True))
        if splits >= 2:
            out.append(case(form, False, dict(w_cluster_reduce=0)))
        out.append(case(form, False, dict(pull_force_pack=1) if form == 0 else {}))
    if bits & FORM2_BIT:
        out.append(case(2, False))
        if splits >= 2:
            out.append(case(2, False, dict(w_cluster_reduce=0)))
    if extras and shape == SHAPES[0] and bits & DIRECT_BIT:
        out.append(case(1, True, dict(nmf_pdl=0)))
    if extras and shape == SHAPES[2]:
        out.append(case(0, bool(bits & DIRECT_BIT), alpha=0.3, eps=0.25))
    return out


def numerator_source(h, sm, shape, c):
    """How the numerator reaches the exchange: 'direct', 'k-split slabs', 'cluster-reduced slab' or 'one slab' (no k-splits)."""
    F, T2, K = shape
    if c.direct:
        return 'direct'
    if tile_plan(h, sm, F, T2, K)[3] < 2:
        return 'one slab'
    if c.opts.get('w_cluster_reduce', 1) == 0:
        return 'k-split slabs'
    with options(h, pull_force_pack=0):
        clustered = h.lib.gccnmf_klnmf_pull_supported(h.h, F, T2, K) & DIRECT_BIT
    return 'cluster-reduced slab' if clustered else 'k-split slabs'


def bit_exact(c, slots):
    return c.direct or c.form == 2 or slots <= 8


_SINGLE = {}


def single_gpu(h, shape, iters, c, V, W0, H0):
    """h.klnmf with the case's library options (pull_force_pack does not concern it), cached."""
    opts = {k: v for k, v in c.opts.items() if k != 'pull_force_pack'}
    key = (shape, iters, tuple(sorted(opts.items())), c.alpha, c.eps)
    if key not in _SINGLE:
        with options(h, **opts):
            _SINGLE[key] = run(h, V, W0, H0, iters, c.alpha, c.eps)
    return _SINGLE[key]


def assert_records(h, sm, rec, shape, iters, c):
    """Per iteration: 2 G1 + G2 + G4 plane-GEMM CTA records (epilogue stamp set), then one record per launch of the exchange --
    pack P (stamps 0 and 7 only), slice reduction and W update S (stamps 0, 1, 2, 7), exchange inside the W update X (0 .. 3, 7)."""
    g1, g2, g4 = expected_ctas(h, sm, *shape)
    gemm = 2 * g1 + g2 + g4
    tail = {(0, True): 'S', (0, False): 'PS', (1, True): 'SS', (1, False): 'PSS', (2, False): 'X'}[c.form, c.direct]
    n = gemm + len(tail)
    assert rec.count == iters * n, ('records', rec.count, iters, (g1, g2, g4), tail)
    s = rec.buf[:rec.count * 8].cpu().numpy().reshape(-1, 8)
    for i in range(iters):
        blk = s[i * n:(i + 1) * n]
        assert (blk[:gemm, 6] != 0).all(), ('a plane-GEMM record without its epilogue stamp', i)
        extra = blk[gemm:]
        assert (extra[:, 0] != 0).all() and (extra[:, 7] != 0).all() and (extra[:, 6] == 0).all(), (i, extra)
        kinds = ''.join('P' if r[1] == 0 else 'X' if r[3] != 0 else 'S' for r in extra)
        assert kinds == tail, ('launch sequence of iteration %d' % i, kinds, tail)


def check_case(h, sm, shape, c, iters, layout_T2=None):
    """One case on a fresh buffer: records, bits or float64 bars, buffer state.  Returns (W, H)."""
    F, T2, K = shape
    layout_T2 = layout_T2 or T2
    slots = tile_plan(h, sm, F, T2, K)[4]
    V, W0, H0 = make_inputs(F, T2, K, 1)
    with options(h, **c.opts):
        bits = h.lib.gccnmf_klnmf_pull_supported(h.h, F, T2, K)
        assert not c.direct or bits & DIRECT_BIT, (shape, case_name(c), bits)
        assert c.form != 2 or bits & FORM2_BIT, (shape, case_name(c), bits)
        px = new_exchange(h, F, layout_T2, K, c.form, c.direct)
        rec = Records(h)
        W, H = run_pull(h, px, V, W0, H0, iters, c.alpha, c.eps, records=rec)
    what = (shape, case_name(c), 'iters', iters, 'layout_T2', layout_T2)
    assert px.epoch == iters
    assert_records(h, sm, rec, shape, iters, c)
    assert_buffer_state(h, px, F, T2, K, iters, slots)
    errs = check(iters, what, W, H, reference(F, T2, K, 1, iters, c.alpha, c.eps))
    for m, e in errs.items():
        if e > WORST.get((iters, m), (0.0, None))[0]:
            WORST[iters, m] = (e, what)
    Ws, Hs = single_gpu(h, shape, iters, c, V, W0, H0)
    if bit_exact(c, slots):
        assert np.array_equal(W, Ws) and np.array_equal(H, Hs), ('not bit-identical to h.klnmf', what)
    COVERED.add((c.form, numerator_source(h, sm, shape, c), 'slots > 8' if slots > 8 else 'slots <= 8',
                 'uneven' if layout_T2 != T2 else 'even'))
    return W, H


# ------------------------------------------------------------------------------------------------ tests
@pytest.mark.parametrize('shape', SHAPES, ids=lambda s: '%dx%dx%d' % s)
def test_pull_forms_match_single_gpu_and_float64(h, sm_count, shape):
    """Every form and numerator source at 1 and 3 iterations: the kernels of the form ran, the buffer holds what the form leaves,
    W and H are held to float64 element by element and, where the additions are in the same order, to h.klnmf bit for bit."""
    for c in shape_cases(h, sm_count, shape):
        for iters in (1, 3):
            check_case(h, sm_count, shape, c, iters)


def test_epoch_continues_on_the_other_parity_half(h, sm_count):
    """3 iterations, then 2 more on the same buffer (epoch 3: the second run starts on the other parity half and waits for
    arrivals 4 and 5) give the bits of 2 iterations from the first run's output on a fresh buffer; the counters end at 5."""
    shape = SHAPES[0]
    F, T2, K = shape
    slots = tile_plan(h, sm_count, F, T2, K)[4]
    V, W0, H0 = make_inputs(F, T2, K, 1)
    for c in shape_cases(h, sm_count, shape, extras=False):
        with options(h, **c.opts):
            px = new_exchange(h, F, T2, K, c.form, c.direct)
            W3, H3 = run_pull(h, px, V, W0, H0, 3)
            W5, H5 = run_pull(h, px, V, W3, H3, 2)
            assert px.epoch == 5
            Wf, Hf = run_pull(h, new_exchange(h, F, T2, K, c.form, c.direct), V, W3, H3, 2)
        assert np.array_equal(W5, Wf) and np.array_equal(H5, Hf), case_name(c)
        assert_buffer_state(h, px, F, T2, K, 5, slots)


@pytest.mark.parametrize('shape', SHAPES[:2], ids=lambda s: '%dx%dx%d' % s)
def test_uneven_shard_layout(h, sm_count, shape):
    """The shorter rank of an uneven split lays its buffer out for the longest shard: layout_T2 > T2 with more row-sum slots
    than T2 needs.  The extra slots stay zero and the bits are those of layout_T2 = T2."""
    F, T2, K = shape
    layout_T2 = T2 + 256
    assert max_rowsum_slots(layout_T2) > max_rowsum_slots(T2)
    for c in shape_cases(h, sm_count, shape, extras=False):
        W, H = check_case(h, sm_count, shape, c, 3, layout_T2)
        We, He = check_case(h, sm_count, shape, c, 3)
        assert np.array_equal(W, We) and np.array_equal(H, He), case_name(c)


def test_uninitialised_workspace_is_never_read(h, sm_count):
    """0xFF over the whole cached KL-NMF workspace before klnmf_begin gives the bits of a zeroed one: nothing reads what the
    iteration did not write, and prepare zeroes the completion counters of the pack, the slice reduction and the direct
    contraction (the last CTA of each would otherwise never be the one to signal)."""
    shape = SHAPES[0]
    F, T2, K = shape
    V, W0, H0 = make_inputs(F, T2, K, 5)
    for c in shape_cases(h, sm_count, shape, extras=False):
        with options(h, **c.opts):
            Wz, Hz = run_pull(h, new_exchange(h, F, T2, K, c.form, c.direct), V, W0, H0, 3, fill=0)
            Wn, Hn = run_pull(h, new_exchange(h, F, T2, K, c.form, c.direct), V, W0, H0, 3, fill=0xFF)
        assert np.isfinite(Wz).all() and np.isfinite(Hz).all()
        assert np.array_equal(Wz, Wn) and np.array_equal(Hz, Hn), case_name(c)


def test_refusals_launch_nothing(h, sm_count):
    """Bad arguments and forms the card or shape cannot run fail with their status before anything is enqueued."""
    import torch
    from gcc_nmf_b200._lib import GCCNMF_ERR_INVALID_ARGUMENT as INVALID, GCCNMF_ERR_UNSUPPORTED as UNSUPPORTED
    F, T2, K = SHAPES[0]
    assert h.lib.gccnmf_klnmf_pull_supported(h.h, F, T2, K) & DIRECT_BIT

    def call(shape=SHAPES[0], world=1, rank=0, bases='buffer', layout_T2=None, form=0, direct=0, iteration=0, epoch=0):
        F, T2, K = shape
        V, W0, H0 = make_inputs(F, T2, K, 1)
        Vd, W, H = h.to_device(V), h.to_device(W0), h.to_device(H0)
        buf = torch.zeros(h.lib.gccnmf_klnmf_pull_buffer_floats(F, max(T2, layout_T2 or T2), K), dtype=torch.float32, device=h.device)
        if bases == 'buffer':
            bases = (ctypes.c_void_p * 9)(*([buf.data_ptr()] * 9))
        ws = h._klnmf_ws(F, T2, K)
        torch.cuda.synchronize()
        before = h.launches
        st = h.lib.gccnmf_klnmf_step_pull(h.h, Vd.data_ptr(), F, T2, W.data_ptr(), H.data_ptr(), K, 0.0, 1e-16, iteration, epoch, rank, world,
                                          bases, layout_T2 or T2, form, direct, ws.data_ptr(), ws.numel(), h.stream)
        torch.cuda.synchronize()
        assert h.launches == before, 'a refused call launched'
        return st

    assert call(layout_T2=T2 - 8) == INVALID
    assert call(world=0) == INVALID
    assert call(world=9) == INVALID
    assert call(world=1, rank=1) == INVALID
    assert call(world=2, rank=-1) == INVALID
    assert call(bases=(ctypes.c_void_p * 1)(None)) == INVALID
    assert call(bases=None) == INVALID
    assert call(iteration=-1) == INVALID
    assert call(epoch=-1) == INVALID
    for form in (0, 1):
        with options(h, pull_force_pack=1):
            assert not h.lib.gccnmf_klnmf_pull_supported(h.h, F, T2, K) & DIRECT_BIT
            assert call(form=form, direct=1) == UNSUPPORTED
        with options(h, w_cluster_reduce=0):
            assert not h.lib.gccnmf_klnmf_pull_supported(h.h, F, T2, K) & DIRECT_BIT
            assert call(form=form, direct=1) == UNSUPPORTED
    for shape in SHAPES:                                  # forms the card's residency does not offer at a shape
        bits = h.lib.gccnmf_klnmf_pull_supported(h.h, *shape)
        if not bits & DIRECT_BIT:
            assert call(shape=shape, form=0, direct=1) == UNSUPPORTED, shape
        if not bits & FORM2_BIT:
            assert call(shape=shape, form=2) == UNSUPPORTED, shape
    simt = (F, T2, 68)                                    # K % 8 != 0: the SIMT path
    assert h.lib.gccnmf_klnmf_pull_supported(h.h, *simt) == 0
    assert call(shape=simt) == UNSUPPORTED
    with options(h, force_simt_nmf=1):
        assert h.lib.gccnmf_klnmf_pull_supported(h.h, F, T2, K) == 0
        for form in (0, 1, 2):
            assert call(form=form) == UNSUPPORTED
    # the handle is left usable: a run after the refusals still matches h.klnmf
    check_case(h, sm_count, SHAPES[0], case(0, True), 1)


def test_case_list_reaches_every_form(h, sm_count):
    """The cases above reach, on this card: every form direct (form 2: from the contraction's own result), packed from k-split
    slabs and packed from a cluster-reduced slab; at most 8 and more than 8 row-sum slots; an uneven layout.  A form the card's
    plan or residency does not offer at these shapes fails here -- then the shapes have to change."""
    reach = set()
    for shape in SHAPES:
        F, T2, K = shape
        slots = tile_plan(h, sm_count, F, T2, K)[4]
        for c in shape_cases(h, sm_count, shape):
            reach.add((c.form, numerator_source(h, sm_count, shape, c)))
            reach.add(('slots', slots > 8))
    for shape in SHAPES[:2]:
        reach |= {('uneven', c.form, c.direct) for c in shape_cases(h, sm_count, shape, extras=False)}
    want = {(f, 'direct') for f in (0, 1)} | {(f, s) for f in (0, 1, 2) for s in ('k-split slabs', 'cluster-reduced slab')}
    want |= {('slots', False), ('slots', True)} | {('uneven', 0, True), ('uneven', 1, True), ('uneven', 2, False), ('uneven', 0, False)}
    assert want <= reach, ('not offered on %d SMs' % sm_count, sorted(want - reach, key=str))


def test_report(h, sm_count, capsys):
    """The worst normalised error against float64 over the pull-exchange runs (runs last)."""
    with capsys.disabled():
        print('\npull exchange offered on %d SMs (1 pull, 2 direct, 4 form 2): %s' % (sm_count, ', '.join(
            '%dx%dx%d: %d' % (s + (h.lib.gccnmf_klnmf_pull_supported(h.h, *s),)) for s in SHAPES)))
        print('pull exchange, forms reached: %s' % '; '.join(sorted('form %d %s, %s, %s' % k for k in COVERED)))
        print('pull exchange, element-wise error against float64, worst per group (bound):')
        for key in sorted(WORST, key=str):
            e, what = WORST[key]
            print('  %-8s %.3e (%.1e)  at %s' % ('%s %s' % key, e, BOUNDS[key], what))
