"""GPU: the KL-NMF loop (csrc/klnmf.cu, csrc/klnmf_tma.cu on the plane GEMM of csrc/tma_gemm*.cuh) against a float64 run of the
same iterations, ELEMENT BY ELEMENT, at shapes and tile plans chosen to reach every path of the tensor-core loop: SIMT tail rows
(1, 7 and 8 of them), partial m tiles, half k-blocks and partial 32-atom blocks (K % 32 != 0, K < 128), odd T2 and padded Fp,
every W.H tile width, every H-update width, the W-update numerator with and without k-splits, the fixed-dictionary loop, the
building blocks of the sharded loop and the options the library accepts.

Error measure: |gpu - ref| / (|ref| + 2^-10 max |ref| over the atom), per atom (W column, H row), so one wrong row, column, tile
or atom fails however large the matrix.  Every tensor-core run arms gccnmf_debug_timing and checks that the launches ran the
CTA counts its plan implies (8 stamps per plane-GEMM CTA, one record per W update)."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# Bound per group (iterations, fixed dictionary, recorded spectrogram) and matrix: 4 x the worst normalised error measured over all
# shapes, plans and both paths on one H100 80GB HBM3 at its 700 W power limit (DESIGN.md 4.1), rounded up.
BOUNDS = {
    (1, 'W'): 1.4e-5, (1, 'H'): 6.1e-5,         # measured 3.4e-6, 1.5e-5
    (3, 'W'): 2.1e-5, (3, 'H'): 3.3e-5,         # measured 5.3e-6, 8.1e-6
    ('fixed', 'H'): 2.5e-5,                     # measured 6.1e-6
    ('real', 'W'): 2.9e-5, ('real', 'H'): 6.2e-5,   # measured 7.2e-6, 1.5e-5
}
WORST = {}
COVERED = set()

# (F, T2, K): what each shape reaches on the tensor-core path
TC_SHAPES = [
    (129, 128, 32),      # minimum T2 and K, one SIMT tail row, one m tile
    (136, 250, 40),      # 8 tail rows, K % 32 = 8 (half k-block, partial atom block), K < 128
    (200, 622, 72),      # tail of 72 rows > 8: a partial m tile instead of SIMT rows; T2 % 8 = 6
    (263, 1001, 200),    # 7 tail rows, F % 8 = 7 (Fp pad), odd T2, K % 128 = 72
    (384, 130, 1000),    # F % 128 = 0, K % 16 = 8
    (2049, 600, 128),    # 16 m tiles + 1 tail row, Fp = 2056
]
# the (alpha, eps) and fixed-dictionary cases: tail rows, partial m tile, partial atom block
EDGE_SHAPES = [(136, 250, 40), (200, 622, 72), (263, 1001, 200)]
WH_WIDTHS = (104, 112, 120, 128, 256)


@pytest.fixture(scope='module')
def h():
    from gcc_nmf_b200._lib import default_handle
    hd = default_handle()
    yield hd
    for name, value in DEFAULT_OPTIONS.items():
        hd.set_option(name, value)


DEFAULT_OPTIONS = {'force_simt_nmf': 0, 'nmf_pdl': 1, 'wh_tile': 0, 'gemm_cluster': -1, 'gemm_pair': -1, 'gemm_preload': 1,
                   'gemm_streaming': 0, 'l2_persist': 0, 'w_cluster_reduce': 1, 'wh_split2': 0, 'pull_force_pack': 0}


class options(object):
    """set_option for the duration of a with-block, back to the library defaults after it."""
    def __init__(self, h, **kw):
        self.h, self.kw = h, kw

    def __enter__(self):
        for k, v in self.kw.items():
            self.h.set_option(k, v)

    def __exit__(self, *exc):
        for k in self.kw:
            self.h.set_option(k, DEFAULT_OPTIONS[k])


@pytest.fixture(scope='module')
def sm_count(h):
    import torch
    props = torch.cuda.get_device_properties(h.device)
    try:
        power = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', str(h.device.index)],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = 'unknown'
    print('\n%s, %d SMs, power limit %s' % (props.name, props.multi_processor_count, power or 'unknown'))
    return props.multi_processor_count


# ------------------------------------------------------------------------------------------------ references and measures
def make_inputs(F, T2, K, seed):
    from oracle import gccnmf_oracle as orc
    rng = np.random.default_rng(seed)
    V = (rng.random((F, T2)) ** 3 + 1e-3).astype(np.float32)
    W0, H0 = orc.initKLNMF(F, T2, K)
    return V, W0, H0


def klnmf64(V, W0, H0, snapshots, alpha=0.0, eps=1e-16, update_W=True):
    """float64 iterations from the float32 inputs: {iterations: (W, H)} for every count in `snapshots`."""
    from oracle import gccnmf_oracle as orc
    V, W, H = V.astype(np.float64), W0.astype(np.float64), H0.astype(np.float64)
    out = {}
    denom = W.sum(0)[:, None] + alpha + eps
    for it in range(1, max(snapshots) + 1):
        with np.errstate(divide='ignore', invalid='ignore'):
            if update_W:
                orc.klnmfIteration(V, W, H, alpha, eps)     # float64 in, float64 arithmetic
            else:
                H *= W.T @ (V / (W @ H)) / denom             # gccNMFFunctions.py:76 with a fixed dictionary
        if it in snapshots:
            out[it] = (W.copy(), H.copy())
    return out


_REFS = {}


def reference(F, T2, K, seed, iters, alpha=0.0, eps=1e-16, update_W=True):
    """Cached per (shape, seed, alpha, eps, update_W); 1 and 3 iterations come from one run."""
    key = (F, T2, K, seed, alpha, eps, update_W)
    if key not in _REFS:
        V, W0, H0 = make_inputs(F, T2, K, seed)
        _REFS[key] = klnmf64(V, W0, H0, (1, 3), alpha, eps, update_W)
    return _REFS[key][iters]


def atom_error(gpu, ref, axis):
    """max |gpu - ref| / (|ref| + 2^-10 max |ref| of the atom); axis = the axis an atom runs along (0 for W columns, 1 for H rows)."""
    ref = np.asarray(ref, np.float64)
    floor = 2.0 ** -10 * np.abs(ref).max(axis=axis, keepdims=True)
    return float((np.abs(gpu.astype(np.float64) - ref) / (np.abs(ref) + floor)).max())


def check(group, what, W, H, ref):
    """Holds W and / or H to the group's bound and keeps the worst value seen."""
    errs = {}
    if W is not None:
        errs['W'] = atom_error(W, ref[0], 0)
    errs['H'] = atom_error(H, ref[1], 1)
    for m, e in errs.items():
        key = (group, m)
        if e > WORST.get(key, (0.0, None))[0]:
            WORST[key] = (e, what)
    for m, e in errs.items():
        assert np.isfinite(e) and e <= BOUNDS[group, m], (what, m, e, BOUNDS[group, m])
    return errs


# ------------------------------------------------------------------------------------------------ plans and records
def tile_plan(h, sm, F, T2, K):
    out = (ctypes.c_int * 8)()
    assert h.lib.gccnmf_klnmf_tile_plan(sm, F, T2, K, out) == 0
    return list(out)


def launch_m_tiles(M, bn, simt_tail):
    """m tiles of a plane-GEMM launch (launch_plane_gemm): SIMT tail rows when 1 .. 8 rows are left and the m tiles of an n tile
    can share its columns (at most 128 each)."""
    tail = M % 128
    if simt_tail and 0 < tail <= 8 and M > 128 and (M // 128) * 128 >= bn:
        return M // 128
    return -(-M // 128)


def expected_ctas(h, sm, F, T2, K, wh_tile=0, split2=False):
    """(G1 = G3, G2, G4) CTAs of one iteration as the launches compute them from the plan."""
    p = tile_plan(h, sm, F, T2, K)
    if split2:
        g1 = 2 * launch_m_tiles(F, 208, True) * -(-T2 // 208)
    else:
        bn = wh_tile or p[0]
        g1 = launch_m_tiles(F, bn, True) * -(-T2 // bn)
    g2 = launch_m_tiles(K, p[1], False) * -(-T2 // p[1])
    g4 = launch_m_tiles(K, p[2], False) * -(-F // p[2]) * p[3]
    return g1, g2, g4


class Records(object):
    """Arms gccnmf_debug_timing around a block; .count = plane-GEMM CTA records + W-update records, .w_updates = positions of the
    W-update records (the only records without an epilogue stamp)."""
    def __init__(self, h):
        import torch
        self.h = h
        self.buf = torch.zeros(1 << 21, dtype=torch.int64, device=h.device)

    def __enter__(self):
        self.buf.zero_()
        self.h.lib.gccnmf_debug_timing(self.h.h, self.buf.data_ptr(), 1)
        return self

    def __exit__(self, *exc):
        import torch
        torch.cuda.synchronize()
        used = self.h.lib.gccnmf_debug_timing(self.h.h, None, 1)
        s = self.buf[:used].cpu().numpy().reshape(-1, 8)
        self.count = len(s)
        self.w_updates = list(np.nonzero(s[:, 6] == 0)[0])


def assert_ran(rec, per_iteration, iters, update_W=True):
    """The records of `iters` iterations: G1, G2 (+ G3, G4, W update with update_W) CTAs per iteration, in launch order."""
    g1, g2, g4 = per_iteration
    n = 2 * g1 + g2 + g4 + 1 if update_W else g1 + g2
    assert rec.count == iters * n, ('CTA records', rec.count, iters, per_iteration)
    assert rec.w_updates == ([i * n + n - 1 for i in range(iters)] if update_W else []), rec.w_updates


def run(h, V, W0, H0, iters, alpha=0.0, eps=1e-16, update_W=True, fill=None, records=None):
    """h.klnmf on copies of the inputs -> (W, H) numpy; fill: byte written over the whole cached workspace first."""
    import torch
    F, T2 = V.shape
    K = W0.shape[1]
    Vd, W, H = h.to_device(V), h.to_device(W0.copy()), h.to_device(H0.copy())
    if fill is not None:
        h._klnmf_ws(F, T2, K).fill_(fill)
    if records is not None:
        with records:
            h.klnmf(Vd, W, H, iters, alpha, eps, update_W)
    else:
        h.klnmf(Vd, W, H, iters, alpha, eps, update_W)
    torch.cuda.synchronize()
    return W.cpu().numpy(), H.cpu().numpy()


def run_checked(h, sm, shape, iters, seed=1, alpha=0.0, eps=1e-16, update_W=True, wh_tile=0, split2=False):
    """Tensor-core run with its plan asserted from the records."""
    F, T2, K = shape
    assert h.klnmf_uses_tensor_cores(F, T2, K), shape
    V, W0, H0 = make_inputs(F, T2, K, seed)
    rec = Records(h)
    W, H = run(h, V, W0, H0, iters, alpha, eps, update_W, records=rec)
    assert_ran(rec, expected_ctas(h, sm, F, T2, K, wh_tile, split2), iters, update_W)
    p = tile_plan(h, sm, F, T2, K)
    COVERED.update([('G1/G3', 'split2 208' if split2 else str(wh_tile or p[0])), ('G2', str(p[1]))])
    if update_W:
        COVERED.add(('G4 splits', '1' if p[3] == 1 else '>= 2'))
    return W, H


# ------------------------------------------------------------------------------------------------ tile plans x shapes
@pytest.mark.parametrize('shape', TC_SHAPES, ids=lambda s: '%dx%dx%d' % s)
def test_wh_tile_widths_match_float64(h, sm_count, shape):
    """Every W.H tile width (G1 / G3) and the planned one, at 1 and 3 iterations, against float64 element by element."""
    F, T2, K = shape
    p = tile_plan(h, sm_count, F, T2, K)
    # the planner's CTA counts are the ones the launches run
    assert tuple(p[5:8]) == expected_ctas(h, sm_count, F, T2, K), (shape, p)
    for iters in (1, 3):
        ref = reference(F, T2, K, 1, iters)
        for wh in (0,) + WH_WIDTHS:
            with options(h, wh_tile=wh):
                W, H = run_checked(h, sm_count, shape, iters, wh_tile=wh)
            check(iters, (shape, 'wh_tile', wh or p[0]), W, H, ref)


def search_plans(h, sm, F=128, K=1024, T2_max=8192):
    """Smallest T2 (multiple of 8) at which the planner picks each H-update width and the W-update numerator with and without
    k-splits, for this card's SM count."""
    want = {('G2', w) for w in (128, 176, 208, 240, 256)} | {('G4 splits', 1), ('G4 splits', 2)}
    found = {}
    for T2 in range(128, T2_max + 1, 8):
        p = tile_plan(h, sm, F, T2, K)
        for key in (('G2', p[1]), ('G4 splits', min(p[3], 2))):
            if key in want and key not in found:
                found[key] = T2
        if len(found) == len(want):
            break
    return want, found


def test_h_update_widths_and_numerator_splits_match_float64(h, sm_count):
    """G2 (H update) at every width in {128, 176, 208, 240, 256} and G4 (W-update numerator) with one and with >= 2 k-splits, on
    shapes the host planner picks for this card: K = 1024 (8 m tiles), F = 128, T2 searched upwards."""
    F, K = 128, 1024
    want, found = search_plans(h, sm_count, F, K)
    assert set(found) == want, ('plans the search did not reach on %d SMs' % sm_count, sorted(want - set(found)))
    print('\nplans covered on %d SMs: %s' % (sm_count, ', '.join('%s %d at T2 = %d' % (k[0], k[1], v) for k, v in sorted(found.items()))))
    for key, T2 in sorted(found.items(), key=lambda kv: kv[1]):
        shape = (F, T2, K)
        for iters in (1, 3):
            W, H = run_checked(h, sm_count, shape, iters, seed=2)
            check(iters, (shape, key), W, H, reference(F, T2, K, 2, iters))


def test_planner_counts_the_launched_m_tiles(h, sm_count):
    """F = 129 .. 136 with 256-column W.H tiles: the launch runs two m tiles (no SIMT tail: one 128-row tile cannot share 256
    columns), and the planner must count the same CTAs.  wh_tile forces the width where the planner does not pick it."""
    F, T2, K = 129, 17000, 32
    ref = reference(F, T2, K, 3, 1)
    with options(h, wh_tile=256):
        W, H = run_checked(h, sm_count, (F, T2, K), 1, seed=3, wh_tile=256)
    check(1, ((F, T2, K), 'wh_tile', 256), W, H, ref)
    for T2 in range(16000, 36000, 500):
        p = tile_plan(h, sm_count, F, T2, K)
        assert p[5] == launch_m_tiles(F, p[0], True) * -(-T2 // p[0]), (T2, p)


def test_wh_split2_matches_float64(h, sm_count):
    """wh_split2: the W.H contractions as 128 x 208 tiles whose two contraction halves a (1, 1, 2) cluster sums before the ratio
    epilogue -- another summation order, so it is held to the float64 bound.  Where the split grid fits in one wave (2 x tiles <=
    SMs, K >= 128) the records must show the split form ran (2 CTAs per tile)."""
    ran = 0
    for shape in [s for s in TC_SHAPES if s[2] >= 128]:
        F, T2, K = shape
        split2 = 2 * launch_m_tiles(F, 208, True) * -(-T2 // 208) <= sm_count
        for iters in (1, 3):
            with options(h, wh_split2=1):
                W, H = run_checked(h, sm_count, shape, iters, split2=split2)
            check(iters, (shape, 'wh_split2'), W, H, reference(F, T2, K, 1, iters))
        ran += split2
    assert ran >= 2


def test_alpha_eps_and_fixed_dictionary_match_float64(h, sm_count):
    """(alpha, eps) = (0.3, 0.25): eps is large enough that its place in the gauge, (c + nrm alpha) + nrm eps, shows.  The
    fixed-dictionary loop (update_W = False: colsum(W) computed once, colsum_state 1) through h.klnmf and through
    gccNMFFunctions.inferCoefficientsKLNMF, against the float64 H-only update."""
    import gcc_nmf_b200.gccNMFFunctions as fn
    for shape in EDGE_SHAPES:
        F, T2, K = shape
        for iters in (1, 3):
            W, H = run_checked(h, sm_count, shape, iters, alpha=0.3, eps=0.25)
            check(iters, (shape, 'alpha 0.3 eps 0.25'), W, H, reference(F, T2, K, 1, iters, 0.3, 0.25))
        for alpha, eps in ((0.0, 1e-16), (0.3, 0.25)):
            W, H = run_checked(h, sm_count, shape, 3, alpha=alpha, eps=eps, update_W=False)
            V, W0, _ = make_inputs(F, T2, K, 1)
            assert np.array_equal(W, W0)                      # the dictionary is left as it was
            check('fixed', (shape, 'update_W=0', alpha, eps), None, H, reference(F, T2, K, 1, 3, alpha, eps, False))
    # inferCoefficientsKLNMF: seeded H init, unit-norm dictionary
    F, T2, K = EDGE_SHAPES[-1]
    V, W0, _ = make_inputs(F, T2, K, 4)
    Wd = (W0 / np.linalg.norm(W0, axis=0)).astype(np.float32)
    np.random.seed(0)
    H0 = (np.random.random((K, T2)).astype(np.float32) + 1e-16).astype(np.float32)
    rec = Records(h)
    with rec:
        H = fn.inferCoefficientsKLNMF(V, Wd, 3, 0.3, 1e-16, 0)
    assert_ran(rec, expected_ctas(h, sm_count, F, T2, K), 3, update_W=False)
    check('fixed', ((F, T2, K), 'inferCoefficientsKLNMF'), None, H, klnmf64(V, Wd, H0, (3,), 0.3, 1e-16, False)[3])


SIMT_SHAPES = [(300, 700, 100), (257, 100, 64), (263, 1001, 200)]     # K % 8 != 0; T2 < 128; force_simt_nmf at a tensor-core shape


@pytest.mark.parametrize('shape', SIMT_SHAPES, ids=lambda s: '%dx%dx%d' % s)
def test_simt_path_matches_float64(h, shape):
    """The float32 SIMT path (shapes the plane GEMM does not cover, or force_simt_nmf) against the same float64 runs and bars."""
    F, T2, K = shape
    forced = shape == SIMT_SHAPES[-1]
    with options(h, force_simt_nmf=1 if forced else 0):
        assert not h.klnmf_uses_tensor_cores(F, T2, K)
        assert h.lib.gccnmf_klnmf_uses_tensor_cores(h.h, F, T2, K) == 0
        V, W0, H0 = make_inputs(F, T2, K, 1)
        for alpha, eps in ((0.0, 1e-16), (0.3, 0.25)):
            for iters in (1, 3):
                rec = Records(h)
                W, H = run(h, V, W0, H0, iters, alpha, eps, records=rec)
                assert rec.count == 0                          # no plane GEMM ran
                check(iters, (shape, 'simt', alpha, eps), W, H, reference(F, T2, K, 1, iters, alpha, eps))
            _, H = run(h, V, W0, H0, 3, alpha, eps, update_W=False)
            check('fixed', (shape, 'simt update_W=0', alpha, eps), None, H, reference(F, T2, K, 1, 3, alpha, eps, False))


# ------------------------------------------------------------------------------------------------ options
# Options that change only the schedule, caching or operand routing -- never which products are summed in which order -- give
# bit-identical results:
#   nmf_pdl           programmatic dependent launch: every kernel waits for the prior grids before it touches global memory
#   gemm_cluster      CN x CM clusters: a CTA gets slices of its operand tiles from its peers by TMA multicast; it still runs the
#                     same MMAs over the same k-blocks of its own tile, and the SIMT tail columns do not depend on the cluster
#   gemm_pair         a 1 x 2 cluster sharing the B tile: the same as gemm_cluster 12
#   gemm_preload      the ratio epilogue's V^T columns are loaded while the main loop runs instead of after it
#   gemm_streaming    st.global.cs instead of st.global for the k-split slabs of the numerator (a cache hint)
#   l2_persist        an L2 access-policy window over G^T (a cache hint)
#   w_cluster_reduce  the numerator's k-splits summed through distributed shared memory (tma_gemm.cuh: the tile of split 0, then
#                     + split 1, + split 2, ...) or written as slabs and summed by tma_apply_w_kernel (slab 0, then + slab 1, ...):
#                     the same additions in the same order
NEUTRAL = [('nmf_pdl', 0), ('gemm_cluster', 11), ('gemm_cluster', 12), ('gemm_cluster', 21), ('gemm_cluster', 22),
           ('gemm_pair', 0), ('gemm_pair', 1), ('gemm_preload', 0), ('gemm_streaming', 1), ('l2_persist', 1), ('l2_persist', 2),
           ('w_cluster_reduce', 0), (('w_cluster_reduce', 0), ('gemm_streaming', 1))]


@pytest.mark.parametrize('shape', [(200, 622, 72), (2049, 600, 128)], ids=lambda s: '%dx%dx%d' % s)
def test_schedule_options_are_bit_identical(h, sm_count, shape):
    """Each option above against the default run, 3 iterations, with the default run held to the float64 bound."""
    import torch
    F, T2, K = shape
    assert tile_plan(h, sm_count, F, T2, K)[3] >= 2           # the numerator has k-splits: w_cluster_reduce and the slabs matter
    W0_, H0_ = run_checked(h, sm_count, shape, 3)
    check(3, (shape, 'defaults'), W0_, H0_, reference(F, T2, K, 1, 3))
    for opt in NEUTRAL:
        kw = dict(opt) if isinstance(opt[0], tuple) else dict([opt])
        with options(h, **kw):
            W, H = run_checked(h, sm_count, shape, 3)
        assert torch.equal(torch.from_numpy(W), torch.from_numpy(W0_)) and torch.equal(torch.from_numpy(H), torch.from_numpy(H0_)), kw


# ------------------------------------------------------------------------------------------------ building blocks
def run_blocks(h, V, W0, H0, iters, records=None):
    """klnmf_begin / klnmf_step_numer / klnmf_step_apply / klnmf_end, the blocks of the frame-sharded loop, on one GPU."""
    import torch
    F, T2 = V.shape
    K = W0.shape[1]
    Vd, W, H = h.to_device(V), h.to_device(W0.copy()), h.to_device(H0.copy())
    numer = torch.empty(F * K + K, dtype=torch.float32, device=h.device)
    with records:
        h.klnmf_begin(Vd, W, H)
        for it in range(iters):
            h.klnmf_step_numer(Vd, W, H, it, numer)
            h.klnmf_step_apply(W, H, numer)
        h.klnmf_end(W, H, iters)
    return W.cpu().numpy(), H.cpu().numpy()


@pytest.mark.parametrize('w_cluster_reduce', [1, 0])
@pytest.mark.parametrize('shape', [(200, 622, 72), (136, 2500, 40)], ids=lambda s: '%dx%dx%d' % s)
def test_building_blocks_on_tensor_cores(h, sm_count, shape, w_cluster_reduce):
    """Up to 8 row-sum slots the numerator pack adds the slots in the order the fused W update does (8 strided groups of one
    slot): bit-identical to h.klnmf.  With more slots the two orders differ: both are held to the float64 bound."""
    import torch
    F, T2, K = shape
    p = tile_plan(h, sm_count, F, T2, K)
    slots = p[4]
    V, W0, H0 = make_inputs(F, T2, K, 1)
    ref = reference(F, T2, K, 1, 3)
    with options(h, w_cluster_reduce=w_cluster_reduce):
        Wf, Hf = run_checked(h, sm_count, shape, 3)
        rec = Records(h)
        Wb, Hb = run_blocks(h, V, W0, H0, 3, rec)
    g1, g2, g4 = expected_ctas(h, sm_count, F, T2, K)
    assert rec.count == 3 * (2 * g1 + g2 + g4 + 2)         # + one numerator pack and one W update record per iteration
    check(3, (shape, 'fused', 'w_cluster_reduce', w_cluster_reduce), Wf, Hf, ref)
    check(3, (shape, 'building blocks', 'w_cluster_reduce', w_cluster_reduce), Wb, Hb, ref)
    if slots <= 8:
        assert torch.equal(torch.from_numpy(Wb), torch.from_numpy(Wf)) and torch.equal(torch.from_numpy(Hb), torch.from_numpy(Hf))
    else:
        assert shape == (136, 2500, 40)


# ------------------------------------------------------------------------------------------------ workspace, scale, NaN
@pytest.mark.parametrize('shape', [(263, 1001, 200), (136, 250, 40), (200, 622, 72)], ids=lambda s: '%dx%dx%d' % s)
def test_uninitialised_workspace_is_never_read(h, sm_count, shape):
    """0xFF bytes (NaN in float32 and in bf16) over the whole cached workspace before each call give the bits of a call on a
    zeroed workspace: nothing reads padding, row-sum slots, slabs or partials the call did not write.  Both paths, update_W on
    and off, and the numerator's k-split slabs (w_cluster_reduce 0) where it has splits."""
    F, T2, K = shape
    V, W0, H0 = make_inputs(F, T2, K, 5)
    variants = [dict(force_simt_nmf=0), dict(force_simt_nmf=1)]
    if tile_plan(h, sm_count, F, T2, K)[3] >= 2:
        variants.append(dict(force_simt_nmf=0, w_cluster_reduce=0))
    for kw in variants:
        with options(h, **kw):
            assert h.klnmf_uses_tensor_cores(F, T2, K) == (kw['force_simt_nmf'] == 0)
            for update_W in (True, False):
                Wz, Hz = run(h, V, W0, H0, 3, update_W=update_W, fill=0)
                Wn, Hn = run(h, V, W0, H0, 3, update_W=update_W, fill=0xFF)
                assert np.isfinite(Hz).all() and np.isfinite(Wz).all()
                assert np.array_equal(Wz, Wn) and np.array_equal(Hz, Hn), (kw, update_W)


@pytest.mark.parametrize('shape', [(263, 1001, 200), (136, 250, 40)], ids=lambda s: '%dx%dx%d' % s)
def test_power_of_two_scale_of_V(h, shape):
    """V 2^+-40: W comes out bit-identical and H exactly 2^+-40 H.  The hi/lo split, the three products, __fdividef, float32
    accumulation and IEEE division all commute with a power-of-two scale when nothing is denormal; a hidden additive constant or
    a flush to zero would not."""
    F, T2, K = shape
    V, W0, H0 = make_inputs(F, T2, K, 6)
    for simt in (0, 1):
        with options(h, force_simt_nmf=simt):
            for alpha, eps in ((0.0, 1e-16), (0.3, 0.25)):
                W, H = run(h, V, W0, H0, 3, alpha, eps)
                for e in (40, -40):
                    s = np.float32(2.0 ** e)
                    Ws, Hs = run(h, V * s, W0, H0, 3, alpha, eps)
                    assert np.array_equal(Ws, W), (simt, e, alpha)
                    assert np.array_equal(Hs, H * s), (simt, e, alpha)


def test_silent_frame_propagates_nan_like_float64(h, sm_count):
    """One V column of zeros: the H update zeroes that column of H, the second ratio is 0 / 0, and NaN propagates as in numpy --
    after one iteration with a W update everything is NaN; with a fixed dictionary only the silent column.  The GPU's NaN
    pattern must be the float64 reference's, on both paths; the finite values are held to the bound."""
    F, T2, K = 263, 1001, 200
    V, W0, H0 = make_inputs(F, T2, K, 7)
    V[:, 17] = 0
    ref1 = klnmf64(V, W0, H0, (1,))[1]
    ref3 = klnmf64(V, W0, H0, (3,), update_W=False)[3]
    assert np.isnan(ref1[0]).all() and np.isnan(ref3[1][:, 17]).all() and not np.isnan(np.delete(ref3[1], 17, axis=1)).any()
    for simt in (0, 1):
        with options(h, force_simt_nmf=simt):
            assert h.klnmf_uses_tensor_cores(F, T2, K) == (simt == 0)
            W, H = run(h, V, W0, H0, 1)
            assert np.array_equal(np.isnan(W), np.isnan(ref1[0])) and np.array_equal(np.isnan(H), np.isnan(ref1[1])), simt
            _, H = run(h, V, W0, H0, 3, update_W=False)
            assert np.array_equal(np.isnan(H), np.isnan(ref3[1])), simt
            check('fixed', ('silent frame', 'simt' if simt else 'tc'), None, np.delete(H, 17, axis=1), (None, np.delete(ref3[1], 17, axis=1)))


def test_real_spectrogram_matches_float64(h, sm_count):
    """The shipped recording's magnitude spectrogram (1024-point STFT, F = 513, both channels: T2 = 622), for its dynamic range
    (7 decades), K = 200 (partial m tile of atoms, partial 32-atom block), on both paths."""
    from oracle import gccnmf_oracle as orc
    from gcc_nmf_b200 import wavio
    x, _ = wavio.wavread(os.path.join(ROOT, 'tests', 'golden', 'dev1_female3_liverec_130ms_1m_mix.wav'))
    V = np.concatenate(np.abs(orc.computeComplexMixtureSpectrogram(x, 1024, 512)), axis=-1).astype(np.float32)
    F, T2 = V.shape
    K = 200
    W0, H0 = orc.initKLNMF(F, T2, K)
    refs = klnmf64(V, W0, H0, (3,))
    for simt in (0, 1):
        with options(h, force_simt_nmf=simt):
            rec = Records(h)
            W, H = run(h, V, W0, H0, 3, records=rec)
        if not simt:
            assert_ran(rec, expected_ctas(h, sm_count, F, T2, K), 3)
        check('real', ('recording', 'simt' if simt else 'tc'), W, H, refs[3])


def test_report(h, sm_count, capsys):
    """The worst normalised error of each group against its bound (runs last)."""
    with capsys.disabled():
        print('\nKL-NMF tensor-core plans run and checked: %s' % '; '.join(
            '%s %s' % (k, ', '.join(sorted(v for c, v in COVERED if c == k))) for k in ('G1/G3', 'G2', 'G4 splits')))
        print('KL-NMF element-wise error against float64, worst per group (bound):')
        for key in sorted(WORST, key=str):
            e, what = WORST[key]
            print('  %-14s %.3e (%.1e)  at %s' % ('%s %s' % key, e, BOUNDS[key], what))
