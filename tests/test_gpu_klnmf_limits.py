"""GPU: gccnmf_klnmf_batched and gccnmf_klnmf_ragged at the limits of their contract.  B = 8191 equal clips whose numerator runs 8
k-splits (grid z = 65528) and 8191 ragged clips, each with a workspace past 2^32 bytes: every clip's W and H held to a float64 run
of the same iterations element by element, and sampled clips -- the first, the last, those whose workspace region starts past 2^31
and 2^32 bytes, every clip at a first-round step of the tile search, and a seeded sample -- bit for bit against gccnmf_klnmf on the
clip alone.  Then ragged calls whose tile lists hold 31, 32, 33, 1023, 1024 and 1025 clips, B = 8192 refused and B = 8191
accepted, and 2000 ragged clips mixing the tensor-core and SIMT paths.  Each case estimates its footprint first and skips when the
device has not that much free memory; the report prints the sizes, the search rounds, the worst float64 errors, the peak memory
and the wall times."""
import ctypes
import time

import numpy as np
import pytest

from test_gpu_klnmf import BOUNDS, DEFAULT_OPTIONS, tile_plan
from test_klnmf_limits_cpu import (MAX_CLIPS, LONG_T2, CONTRACTIONS, describe, first_step, klnmf64_batched, launch_plan, limit_lengths,
                                   plane_launches, rounds_needed)
from test_klnmf_ragged_cpu import TABLE_EXTRA, TABLE_PER_CLIP, lengths

pytestmark = pytest.mark.gpu

GiB = 1 << 30
MARGIN = 4 * GiB            # left free for the allocator's rounding, the float64 chunks and whoever else shares the device
REF_CHUNK = 256             # clips per float64 reference chunk
REPORT = []
WORST = {}
T_START = time.perf_counter()


@pytest.fixture(scope='module')
def h():
    from gcc_nmf_b200._lib import default_handle
    hd = default_handle()
    yield hd
    for name, value in DEFAULT_OPTIONS.items():
        hd.set_option(name, value)


@pytest.fixture(scope='module')
def sm_count(h):
    import torch
    return torch.cuda.get_device_properties(h.device).multi_processor_count


@pytest.fixture
def fresh(h):
    """Peak-memory counter from zero; after the test, the cached batched / ragged workspaces go back to the device."""
    import torch
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats(h.device)
    yield
    for key in ('klnmf_batched', 'klnmf_ragged'):
        h._workspaces.pop(key, None)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def need(h, nbytes, what):
    import torch
    free, _ = torch.cuda.mem_get_info(h.device)
    if free < nbytes + MARGIN:
        pytest.skip('%s needs about %.1f GiB + %.0f GiB margin, %.1f GiB free' % (what, nbytes / GiB, MARGIN / GiB, free / GiB))


def peak(h):
    import torch
    return torch.cuda.max_memory_allocated(h.device)


def rand(h, shape, seed, lo, cube=False):
    """Seeded device uniforms: x^3 + lo (a spectrogram-like spread) or x + lo."""
    import torch
    g = torch.Generator(device=h.device)
    g.manual_seed(seed)
    x = torch.rand(shape, generator=g, device=h.device, dtype=torch.float32)
    return (x.pow_(3) if cube else x).add_(lo)


# ------------------------------------------------------------------------------------------------ float64 and solo checks
def clip_errors(gpu, ref, axis):
    """Per clip: max |gpu - ref| / (|ref| + 2^-10 max |ref| of the atom) (test_gpu_klnmf.atom_error over a leading clip axis)."""
    floor = 2.0 ** -10 * ref.abs().amax(dim=axis, keepdim=True)
    return ((gpu.double() - ref).abs() / (ref.abs() + floor)).flatten(1).amax(1)


def hold_to_float64(what, clips, V, W0, H0, W, H, iters, alpha, eps, update_W):
    """Clips (index list) whose V, W0, H0, W, H stack along dim 0 (one shape): each against klnmf64_batched on float64 device
    tensors, REF_CHUNK clips at a time, to BOUNDS; keeps the worst error per group."""
    import torch
    group = iters if update_W else 'fixed'
    for s in range(0, len(clips), REF_CHUNK):
        sl = slice(s, s + REF_CHUNK)
        Wr, Hr = klnmf64_batched(V[sl].double(), W0[sl].double(), H0[sl].double(), iters, alpha, eps, update_W)
        errs = {'H': clip_errors(H[sl], Hr, 2)}
        if update_W:
            errs['W'] = clip_errors(W[sl], Wr, 1)
        else:
            assert torch.equal(W[sl], W0[sl]), (what, 'the dictionary changed')
        del Wr, Hr
        for m, e in errs.items():
            e = e.cpu().numpy()
            worst = int(np.argmax(np.where(np.isfinite(e), e, np.inf)))
            key = (group, m)
            if e[worst] > WORST.get(key, (0.0, None))[0]:
                WORST[key] = (float(e[worst]), (what, 'clip', clips[s + worst]))
            assert np.isfinite(e).all() and (e <= BOUNDS[key]).all(), (what, m, clips[s + worst], float(e[worst]), BOUNDS[key])


def solo(h, V, W0, H0, iters, alpha, eps, update_W):
    W, H = W0.clone(), H0.clone()
    h.klnmf(V.contiguous(), W, H, iters, alpha, eps, update_W=update_W)
    return W, H


def assert_solo_equal(h, what, picks, get, iters, alpha, eps, update_W):
    """For each picked clip b, get(b) = (V, W0, H0, W, H): the call's W and H NaN-equal to gccnmf_klnmf on the clip alone (one
    synchronisation for all of them)."""
    import torch
    same = []
    for b in picks:
        V, W0, H0, W, H = get(b)
        Ws, Hs = solo(h, V, W0, H0, iters, alpha, eps, update_W)
        same.append(((W == Ws) | (torch.isnan(W) & torch.isnan(Ws))).all() & ((H == Hs) | (torch.isnan(H) & torch.isnan(Hs))).all())
    ok = torch.stack(same).cpu().numpy()
    assert ok.all(), (what, 'clips that differ from their solo run', [b for b, o in zip(picks, ok) if not o][:16])


def past(offsets, limit):
    """The clip whose workspace region holds byte `limit` and the first whose region starts at or past it."""
    i = int(np.searchsorted(offsets, limit, side='right'))
    return [c for c in (i - 1, i) if 0 <= c < len(offsets)]


def ragged_launch_count(launches, iters, update_W):
    """gccnmf_klnmf_tma_ragged's launches (DESIGN.md 4.4.1): prepare V, split W, prepare H; per iteration G1 (one launch per W.H
    width), the column sums once, G2 (one per width), and with a W update G3, G4 and the W update; then the H finish and the W
    finish."""
    g1, g2 = len(launches['G1/G3']), len(launches['G2'])
    if update_W:
        return 3 + 1 + iters * (plane_launches(launches) + 1) + 2
    return 3 + 1 + iters * (g1 + g2) + 1


# ------------------------------------------------------------------------------------------------ B = 8191, equal lengths
def test_batched_8191_clips_eight_splits(h, sm_count, fresh):
    """F 129, 2T 1024, K 32: the solo plan's numerator runs 8 k-splits, so its batched launch has grid z = 8191 x 8 = 65528."""
    import torch
    lib, B, F, T2, K = h.lib, MAX_CLIPS, 129, 1024, 32
    iters, alpha, eps = 3, 0.1, 1e-16
    p = tile_plan(h, sm_count, F, T2, K)
    assert p[3] == 8 and B * p[3] == 65528, p
    assert h.klnmf_uses_tensor_cores(F, T2, K)
    ws = lib.gccnmf_klnmf_batched_workspace_bytes(B, F, T2, K)
    clip_bytes = ws // B
    assert ws == B * clip_bytes and ws > 1 << 32, ws
    data = 4 * B * (F * T2 + 2 * F * K + 2 * K * T2)
    ref = 8 * REF_CHUNK * (3 * F * T2 + 2 * K * T2 + 2 * F * K)
    need(h, ws + data + ref + 2 * 4 * B * K * T2, 'batched B = 8191')
    V = rand(h, (B, F, T2), 101, 1e-3, cube=True)
    W0 = rand(h, (B, F, K), 102, 0.1)
    H0 = rand(h, (B, K, T2), 103, 0.1)
    offsets = np.arange(B, dtype=np.int64) * clip_bytes
    rng = np.random.default_rng(8191)
    picks = sorted({0, 1, B - 1, *past(offsets, 1 << 31), *past(offsets, 1 << 32)} | set(int(b) for b in rng.choice(B, 64, replace=False)))
    assert any(offsets[b] >= 1 << 32 for b in picks)
    for update_W in (True, False):
        W, H = W0.clone(), H0.clone()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        h.klnmf_batched(V, W, H, iters, alpha, eps, update_W=update_W)
        torch.cuda.synchronize()
        t_call = time.perf_counter() - t0
        t0 = time.perf_counter()
        hold_to_float64(('batched 8191', update_W), list(range(B)), V, W0, H0, W, H, iters, alpha, eps, update_W)
        t_ref = time.perf_counter() - t0
        t0 = time.perf_counter()
        assert_solo_equal(h, ('batched 8191', update_W), picks, lambda b: (V[b], W0[b], H0[b], W[b], H[b]), iters, alpha, eps, update_W)
        t_solo = time.perf_counter() - t0
        del W, H
        REPORT.append('batched  B %d  F %d 2T %d K %d  G4 splits %d (grid z %d)  update_W %d  workspace %d B (%.2f x 2^32)  call %.2f s, '
                      'float64 %.2f s, %d solo clips %.2f s' % (B, F, T2, K, p[3], B * p[3], update_W, ws, ws / 2.0 ** 32, t_call, t_ref,
                                                                 len(picks), t_solo))
    REPORT.append('batched  peak memory %.2f GiB' % (peak(h) / GiB))


# ------------------------------------------------------------------------------------------------ B = 8191, ragged
def ragged_inputs(h, F, K, T2s, seed):
    """V as column ranges of one (F, sum 2T) device matrix (read in place), W0 (B, F, K), H0 as contiguous (K, 2T) pieces of one
    buffer; -> Vs, W0, H0 buffer, H0 views."""
    B, total = len(T2s), int(sum(T2s))
    M = rand(h, (F, total), seed, 1e-3, cube=True)
    offs = [int(o) for o in np.concatenate([[0], np.cumsum(T2s)])]
    Vs = [M[:, offs[b]:offs[b + 1]] for b in range(B)]
    W0 = rand(h, (B, F, K), seed + 1, 0.1)
    H0 = rand(h, (K * total,), seed + 2, 0.1)
    return Vs, W0, H0, views(H0, K, T2s)


def views(flat, K, T2s):
    offs = [int(o) for o in np.concatenate([[0], np.cumsum(T2s)]) * K]
    return [flat[offs[b]:offs[b + 1]].view(K, t) for b, t in enumerate(T2s)]


def run_ragged(h, Vs, W0, H0flat, K, T2s, iters, alpha, eps, update_W):
    W, Hflat = W0.clone(), H0flat.clone()
    Hs = views(Hflat, K, T2s)
    before = h.launches
    h.klnmf_ragged(Vs, W, Hs, iters, alpha, eps, update_W=update_W)
    return W, Hs, h.launches - before


def ragged_float64(what, T2s, Vs, W0, H0s, W, Hs, iters, alpha, eps, update_W):
    """Every clip against float64, the clips of each length stacked."""
    import torch
    for t in sorted(set(T2s)):
        idx = [b for b, x in enumerate(T2s) if x == t]
        for s in range(0, len(idx), REF_CHUNK):
            c = idx[s:s + REF_CHUNK]
            st = lambda xs: torch.stack([xs[b] for b in c])
            hold_to_float64(what + ('2T %d' % t,), c, st(Vs), W0[c], st(H0s), W[c], st(Hs), iters, alpha, eps, update_W)


def search_boundaries(launches):
    """Clips at the first-round steps of each launch's tile search: the entries lane x step and the ones just before them."""
    out = set()
    for ls in launches.values():
        for l in ls:
            n, step = len(l['clips']), first_step(len(l['clips']))
            for j in range(0, n, step):
                out.update(l['clips'][k] for k in (j - 1, j) if 0 <= k < n)
            out.add(l['clips'][-1])
    return out


def test_ragged_8191_clips_three_search_rounds(h, sm_count, fresh):
    """F 200, K 32, 8158 clips of 2T 128 .. 640 and 33 of 2T 6872 spread among them: on 132 SMs the W.H contractions launch an
    8158-clip and a 33-clip group, G2 and G4 one 8191-clip group; three search rounds, first steps that do not divide their ranges,
    clips of one CTA and of many.  The launch count is the ragged formula's."""
    import torch
    lib, F, K = h.lib, 200, 32
    iters, alpha, eps = 3, 0.1, 1e-16
    T2s = limit_lengths()
    B = len(T2s)
    launches = launch_plan(lib, sm_count, F, T2s, K)
    d = describe(launches)
    sizes = [n for c in CONTRACTIONS for n in d[c][0]]
    assert max(r for _, r in d.values()) == 3 and any(n > 1024 and first_step(n) * 32 != n for n in sizes), d
    if sm_count == 132:
        assert d['G1/G3'] == ([B - 33, 33], 3) and d['G2'] == ([B], 3) and d['G4'] == ([B], 3), d
    ctas = {t: tile_plan(h, sm_count, F, t, K)[5:8] for t in set(T2s)}
    assert min(c[1] for c in ctas.values()) == 1 and max(c[0] for c in ctas.values()) > 100, ctas
    assert all(h.klnmf_uses_tensor_cores(F, t, K) for t in set(T2s))
    ws = lib.gccnmf_klnmf_ragged_workspace_bytes(B, F, lengths(*T2s), K)
    regions = {t: lib.gccnmf_klnmf_batched_workspace_bytes(1, F, t, K) for t in set(T2s)}
    offsets = TABLE_PER_CLIP * B + TABLE_EXTRA + np.concatenate([[0], np.cumsum([regions[t] for t in T2s])[:-1]])
    assert ws == TABLE_PER_CLIP * B + TABLE_EXTRA + sum(regions[t] for t in T2s) and ws > 1 << 32, ws
    total = int(sum(T2s))
    data = 4 * (F * total + 2 * B * F * K + 2 * K * total)
    ref = 8 * REF_CHUNK * (3 * F * LONG_T2 + 2 * K * LONG_T2 + 2 * F * K)
    need(h, ws + data + ref + 4 * 2 * K * total, 'ragged B = 8191')
    Vs, W0, H0flat, H0s = ragged_inputs(h, F, K, T2s, 201)
    rng = np.random.default_rng(8192)
    picks = sorted({0, 1, B - 1, *past(offsets, 1 << 31), *past(offsets, 1 << 32)} | search_boundaries(launches) |
                   set(int(b) for b in rng.choice(B, 64, replace=False)))
    assert any(offsets[b] >= 1 << 32 for b in picks) and any(T2s[b] == LONG_T2 for b in picks)
    for update_W in (True, False):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        W, Hs, got = run_ragged(h, Vs, W0, H0flat, K, T2s, iters, alpha, eps, update_W)
        torch.cuda.synchronize()
        t_call = time.perf_counter() - t0
        assert got == ragged_launch_count(launches, iters, update_W), (got, update_W)
        t0 = time.perf_counter()
        ragged_float64(('ragged 8191', update_W), T2s, Vs, W0, H0s, W, Hs, iters, alpha, eps, update_W)
        t_ref = time.perf_counter() - t0
        t0 = time.perf_counter()
        assert_solo_equal(h, ('ragged 8191', update_W), picks, lambda b: (Vs[b], W0[b], H0s[b], W[b], Hs[b]), iters, alpha, eps, update_W)
        t_solo = time.perf_counter() - t0
        del W, Hs
        REPORT.append('ragged   B %d  F %d K %d 2T %d .. %d  update_W %d  workspace %d B (%.2f x 2^32)  launches %d  call %.2f s, float64 '
                      '%.2f s, %d solo clips %.2f s' % (B, F, K, min(T2s), max(T2s), update_W, ws, ws / 2.0 ** 32, got, t_call, t_ref,
                                                         len(picks), t_solo))
    for c in CONTRACTIONS:
        REPORT.append('ragged   %-6s groups (width: clips) %s, search rounds %d' % (
            c, ', '.join('%d: %d' % (l['bn'], len(l['clips'])) for l in launches[c]), d[c][1]))
    REPORT.append('ragged   peak memory %.2f GiB' % (peak(h) / GiB))


# ------------------------------------------------------------------------------------------------ search edges at small B
EDGE_T2 = (128, 160, 250, 384, 130, 520)


@pytest.mark.parametrize('B', [31, 32, 33, 1023, 1024, 1025])
def test_search_edges_bit_for_bit(h, sm_count, fresh, B):
    """One width group per contraction holding exactly B clips (one search round up to 32, two up to 1024, three at 1025): every
    clip NaN-equal to its solo run."""
    F, K, iters, alpha, eps = 129, 32, 2, 0.1, 1e-16
    T2s = [EDGE_T2[b % len(EDGE_T2)] for b in range(B)]
    launches = launch_plan(h.lib, sm_count, F, T2s, K)
    assert describe(launches) == {c: ([B], rounds_needed(B)) for c in CONTRACTIONS}, describe(launches)
    Vs, W0, H0flat, H0s = ragged_inputs(h, F, K, T2s, 300 + B)
    W, Hs, got = run_ragged(h, Vs, W0, H0flat, K, T2s, iters, alpha, eps, True)
    assert got == ragged_launch_count(launches, iters, True)
    assert_solo_equal(h, ('search edge', B), list(range(B)), lambda b: (Vs[b], W0[b], H0s[b], W[b], Hs[b]), iters, alpha, eps, True)
    REPORT.append('edges    B %4d: one group of %d clips per contraction, %d search rounds, every clip bit-identical to its solo run'
                  % (B, B, rounds_needed(B)))


# ------------------------------------------------------------------------------------------------ refusals at the edge
def test_refusals_at_the_limit(h):
    """B = 8192 is refused by both entries before anything is enqueued, and both size queries answer 0; B = 8191 is accepted (zero
    iterations: the call checks everything and enqueues nothing, so no buffer behind the pointers is read)."""
    import torch
    from gcc_nmf_b200._lib import GCCNMF_OK
    lib, F, T2, K = h.lib, 129, 128, 32
    buf = torch.empty(1 << 20, dtype=torch.float32, device=h.device)
    p = buf.data_ptr()
    for B in (MAX_CLIPS, MAX_CLIPS + 1):
        nb = lib.gccnmf_klnmf_batched_workspace_bytes(B, F, T2, K)
        nr = lib.gccnmf_klnmf_ragged_workspace_bytes(B, F, lengths(*([T2] * B)), K)
        if B > MAX_CLIPS:
            assert nb == 0 and nr == 0
            nb = nr = 1 << 40
        else:
            assert nb > 0 and nr > 0
        ptrs = (ctypes.c_void_p * B)(*([p] * B))
        for it in ((3, 0) if B > MAX_CLIPS else (0,)):
            before = h.launches
            sb = lib.gccnmf_klnmf_batched(h.h, p, T2, F * T2, B, F, T2, p, p, K, it, 0.0, 1e-16, 1, p, nb, h.stream)
            sr = lib.gccnmf_klnmf_ragged(h.h, ptrs, (ctypes.c_int64 * B)(*([T2] * B)), lengths(*([T2] * B)), B, F, p, ptrs, K, it, 0.0,
                                         1e-16, 1, p, nr, h.stream)
            assert h.launches == before, (B, it)
            if B > MAX_CLIPS:
                assert sb != GCCNMF_OK and sr != GCCNMF_OK and b'8191' in lib.gccnmf_last_error(h.h), (B, it)
            elif it == 0:
                assert sb == GCCNMF_OK and sr == GCCNMF_OK, (sb, sr)
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ mixed fallbacks at scale
MIXED_T2 = (128, 64, 200, 100, 300, 127, 500, 250, 96, 622)


def test_ragged_2000_clips_tensor_core_and_simt(h, sm_count, fresh):
    """2000 clips, 2 in 5 with 2T < 128 (the float32 SIMT loop, one clip at a time on its own region): every SIMT clip and a
    sample of the tensor-core clips NaN-equal to their solo runs, and the call's launches = the SIMT clips' solo launches + the
    ragged loop's (DESIGN.md 4.4.1) over the tensor-core clips."""
    import torch
    F, K, iters, alpha, eps = 129, 32, 3, 0.1, 1e-16
    B = 2000
    T2s = [MIXED_T2[b % len(MIXED_T2)] for b in range(B)]
    tc = [b for b, t in enumerate(T2s) if h.klnmf_uses_tensor_cores(F, t, K)]
    simt = [b for b in range(B) if b not in set(tc)]
    assert len(simt) == 2 * B // 5 and all(T2s[b] < 128 for b in simt)
    Vs, W0, H0flat, H0s = ragged_inputs(h, F, K, T2s, 400)
    launches = launch_plan(h.lib, sm_count, F, [T2s[b] for b in tc], K)
    for update_W in (True, False):
        W, Hs, got = run_ragged(h, Vs, W0, H0flat, K, T2s, iters, alpha, eps, update_W)
        solo_launches = {}
        for t in sorted(set(T2s[b] for b in simt)):
            b = T2s.index(t)
            before = h.launches
            solo(h, Vs[b], W0[b], H0s[b], iters, alpha, eps, update_W)
            solo_launches[t] = h.launches - before
        want = sum(solo_launches[T2s[b]] for b in simt) + ragged_launch_count(launches, iters, update_W)
        assert got == want, (got, want, solo_launches, update_W)
        rng = np.random.default_rng(2000)
        picks = simt + sorted({tc[0], tc[-1]} | set(int(b) for b in rng.choice(tc, 96, replace=False)))
        assert_solo_equal(h, ('mixed 2000', update_W), picks, lambda b: (Vs[b], W0[b], H0s[b], W[b], Hs[b]), iters, alpha, eps, update_W)
        torch.cuda.synchronize()
        REPORT.append('mixed    B %d (%d SIMT, %d tensor-core)  update_W %d  launches %d = %d SIMT solo + %d ragged; %d clips bit-identical '
                      'to solo' % (B, len(simt), len(tc), update_W, got, got - ragged_launch_count(launches, iters, update_W),
                                   ragged_launch_count(launches, iters, update_W), len(picks)))


# ------------------------------------------------------------------------------------------------ report
def test_report(h, sm_count, capsys):
    """Sizes, search rounds, worst float64 error per group against its bound, peak memory and wall times (runs last)."""
    import torch
    with capsys.disabled():
        print('\n%s, %d SMs' % (torch.cuda.get_device_properties(h.device).name, sm_count))
        for line in REPORT:
            print('  ' + line)
        print('  wall time of the file up to the report: %.1f s' % (time.perf_counter() - T_START))
        print('  element-wise error against float64, worst per group (bound):')
        for key in sorted(WORST, key=str):
            e, what = WORST[key]
            print('    %-10s %.3e (%.1e)  at %s' % ('%s %s' % key, e, BOUNDS[key], what))
