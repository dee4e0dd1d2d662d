"""CPU: what the batched and ragged KL-NMF entries do at B = 8191, pinned without a device -- a float64 KL-NMF iteration batched over
clips (the reference that holds thousands of clips to float64 in seconds) against the per-clip float64 reference; a host mirror of
the ragged launch plan (each contraction's clips stably sorted by tile width, one launch per width, CTAs numbered along it) from
gccnmf_klnmf_tile_plan; and a mirror of ragged_find (csrc/tma_gemm.cuh), the 32-way warp search a ragged CTA runs to find its clip,
against a linear scan for every CTA of every launch, at group sizes 1 .. 8191 and at the layout of the GPU test's 8191-clip call."""
import ctypes

import numpy as np
import pytest

MAX_CLIPS = 8191                    # 65535 // 8: a batched contraction's grid z is clips x k-splits (at most 8)
H100_SMS = 132


@pytest.fixture(scope='module')
def lib():
    import __graft_entry__ as entry
    entry.build()
    from gcc_nmf_b200 import _lib
    return _lib.load_library()


# ------------------------------------------------------------------------------------------------ float64 reference over clips
def klnmf64_batched(V, W0, H0, iters, alpha=0.0, eps=1e-16, update_W=True):
    """float64 KL-NMF of a stack of clips: V (B, F, T2), W0 (B, F, K), H0 (B, K, T2) -> (W, H) after `iters` iterations, clip b as
    klnmf64 (test_gpu_klnmf.py) computes it alone: gccNMFFunctions.py:76-81 with matmul over the leading clip axis.  Written with
    the operators numpy arrays and torch tensors share, so the same function runs on float64 device tensors; the caller passes
    float64 arrays."""
    W, H = W0 * 1, H0 * 1
    tr = lambda x: x.swapaxes(-1, -2)
    denom = W.sum(-2)[..., :, None] + alpha + eps
    for _ in range(iters):
        if update_W:
            H = H * ((tr(W) @ (V / (W @ H))) / (W.sum(-2)[..., :, None] + alpha + eps))
            W = W * (((V / (W @ H)) @ tr(H)) / H.sum(-1)[..., None, :])
            norms = (W ** 2).sum(-2) ** 0.5
            W = W / norms[..., None, :]
            H = H * norms[..., :, None]
        else:
            H = H * ((tr(W) @ (V / (W @ H))) / denom)
    return W, H


def batched_inputs(B, F, T2, K, seed):
    rng = np.random.default_rng(seed)
    V = (rng.random((B, F, T2)) ** 3 + 1e-3).astype(np.float32)
    W0 = (rng.random((B, F, K)) + 0.1).astype(np.float32)
    H0 = (rng.random((B, K, T2)) + 0.1).astype(np.float32)
    return V, W0, H0


@pytest.mark.parametrize('shape', [(129, 128, 32), (136, 250, 40), (200, 622, 72), (17, 33, 5)], ids=lambda s: '%dx%dx%d' % s)
@pytest.mark.parametrize('update_W', [True, False])
def test_batched_float64_matches_per_clip_float64(shape, update_W):
    """Clip by clip the same values as the per-clip float64 reference (a few units in the last place of float64 at most: the two
    associate nothing differently, but BLAS may block a stacked product differently from a single one)."""
    from test_gpu_klnmf import klnmf64
    F, T2, K = shape
    V, W0, H0 = batched_inputs(3, F, T2, K, seed=F)
    for alpha, eps in ((0.0, 1e-16), (0.3, 0.25)):
        W, H = klnmf64_batched(V.astype(np.float64), W0.astype(np.float64), H0.astype(np.float64), 3, alpha, eps, update_W)
        for b in range(3):
            Wr, Hr = klnmf64(V[b], W0[b], H0[b], (3,), alpha, eps, update_W)[3]
            np.testing.assert_allclose(W[b], Wr, rtol=1e-12, atol=0)
            np.testing.assert_allclose(H[b], Hr, rtol=1e-12, atol=0)


def test_batched_float64_runs_on_torch_tensors():
    import torch
    V, W0, H0 = batched_inputs(2, 129, 128, 32, seed=1)
    d = lambda x: torch.from_numpy(x.astype(np.float64))
    for update_W in (True, False):
        Wn, Hn = klnmf64_batched(V.astype(np.float64), W0.astype(np.float64), H0.astype(np.float64), 3, 0.1, 1e-16, update_W)
        Wt, Ht = klnmf64_batched(d(V), d(W0), d(H0), 3, 0.1, 1e-16, update_W)
        np.testing.assert_allclose(Wt.numpy(), Wn, rtol=1e-12, atol=0)
        np.testing.assert_allclose(Ht.numpy(), Hn, rtol=1e-12, atol=0)


# ------------------------------------------------------------------------------------------------ the ragged launch plan
CONTRACTIONS = ('G1/G3', 'G2', 'G4')


def tile_plans(lib, sm, F, T2s, K):
    """gccnmf_klnmf_tile_plan of each distinct length: {T2: [W.H width, G2 width, G4 width, G4 splits, slots, G1 CTAs, G2 CTAs, G4 CTAs]}."""
    plans = {}
    for t in sorted(set(T2s)):
        out = (ctypes.c_int * 8)()
        assert lib.gccnmf_klnmf_tile_plan(sm, F, t, K, out) == 0, (F, t, K)
        plans[t] = list(out)
    return plans


def launch_plan(lib, sm, F, T2s, K):
    """Host mirror of gccnmf_klnmf_tma_ragged's launch plan: per contraction, the clips stably sorted by their solo plan's tile width,
    one launch per run of equal widths, each clip's first CTA numbered from 0 along its launch.
    -> {contraction: [dict(bn, clips (clip indices in tile-list order), cta_begin (np.int64), ctas)]}"""
    plans = tile_plans(lib, sm, F, T2s, K)
    out = {}
    for c, name in enumerate(CONTRACTIONS):
        width = [plans[t][c] for t in T2s]
        ctas = [plans[t][5 + c] for t in T2s]             # the clip's CTAs in that contraction (G4: x k-splits)
        order = sorted(range(len(T2s)), key=lambda i: width[i])        # (sorted is stable)
        launches = []
        for i in order:
            if not launches or launches[-1]['bn'] != width[i]:
                launches.append(dict(bn=width[i], clips=[], cta_begin=[], ctas=0))
            l = launches[-1]
            l['clips'].append(i)
            l['cta_begin'].append(l['ctas'])
            l['ctas'] += ctas[i]
        for l in launches:
            l['cta_begin'] = np.asarray(l['cta_begin'], dtype=np.int64)
        out[name] = launches
    return out


def plane_launches(launches):
    """Plane-GEMM launches per iteration: G1 and G3 launch each W.H width, G2 and G4 each of theirs."""
    return 2 * len(launches['G1/G3']) + len(launches['G2']) + len(launches['G4'])


def ragged_find(cta_begin, ctas):
    """ragged_find (csrc/tma_gemm.cuh) for every CTA 0 .. ctas - 1 of a launch at once: lane l of the warp tests entry lo + l step,
    the highest lane whose entry starts at or before the CTA moves lo there, and the range shrinks to one step.
    -> (entry index, rounds of loads) per CTA."""
    count = len(cta_begin)
    me = np.arange(ctas, dtype=np.int64)
    lo = np.zeros(ctas, dtype=np.int64)
    hi = np.full(ctas, count, dtype=np.int64)
    rounds = np.zeros(ctas, dtype=np.int64)
    lanes = np.arange(32, dtype=np.int64)
    while True:
        live = hi - lo > 1
        if not live.any():
            return lo, rounds
        step = (hi - lo + 31) // 32
        i = lo[:, None] + lanes[None, :] * step[:, None]
        le = (i < hi[:, None]) & (cta_begin[np.minimum(i, count - 1)] <= me[:, None])
        assert le[live, 0].all()                                        # lane 0 always qualifies
        top = 31 - np.argmax(le[:, ::-1], axis=1)                       # 31 - __clz(ballot)
        lo = np.where(live, lo + top * step, lo)
        hi = np.where(live, np.minimum(hi, lo + step), hi)
        rounds += live


def check_search(cta_begin, ctas):
    """The mirror against a linear scan (the last entry whose first CTA is at or before the CTA) for every CTA; -> max rounds."""
    got, rounds = ragged_find(cta_begin, ctas)
    want = np.searchsorted(cta_begin, np.arange(ctas), side='right') - 1
    assert np.array_equal(got, want), (len(cta_begin), np.nonzero(got != want)[0][:8])
    return int(rounds.max())


def rounds_needed(n):
    """Rounds of the 32-way search over n entries for its worst CTA: 0 for one entry, then one more per factor of 32."""
    r, span = 0, 1
    while span < n:
        span *= 32
        r += 1
    return r


def first_step(n):
    return (n + 31) // 32


GROUP_SIZES = sorted(set(list(range(1, 70)) + [127, 128, 129, 255, 256, 257, 993, 1000, 1023, 1024, 1025, 1026, 1055, 1056, 1057, 2047,
                                               2048, 2049, 4095, 4096, 4097, 8158, 8159, 8160, 8161, 8190, 8191] +
                         list(np.random.default_rng(0).integers(70, 8192, 40))))


@pytest.mark.parametrize('layout', ['one', 'many', 'mixed'])
def test_ragged_find_matches_a_linear_scan(layout):
    """Every CTA of launches whose tile lists hold 1 .. 8191 entries (every size up to 69, each side of every power of 32 and of
    8191, and a seeded sample): clips of one CTA each, of many, and a seeded mix of 1 .. 40 CTAs."""
    rng = np.random.default_rng({'one': 1, 'many': 2, 'mixed': 3}[layout])
    for n in GROUP_SIZES:
        n = int(n)
        per = {'one': np.ones(n, np.int64), 'many': np.full(n, 17, np.int64), 'mixed': rng.integers(1, 41, n)}[layout]
        begin = np.concatenate([[0], np.cumsum(per)[:-1]])
        assert check_search(begin, int(per.sum())) == rounds_needed(n), n


def test_search_rounds_and_steps():
    """One round up to 32 entries, two up to 1024, three up to 8191; and the sizes the GPU tests pick are the ones they claim."""
    assert [rounds_needed(n) for n in (1, 2, 31, 32, 33, 1023, 1024, 1025, 8191)] == [0, 1, 1, 1, 2, 2, 2, 3, 3]
    assert first_step(8191) * 32 != 8191 and first_step(8158) * 32 != 8158 and first_step(1025) * 32 != 1025
    assert first_step(1024) * 32 == 1024


# ------------------------------------------------------------------------------------------------ the layouts of the GPU tests
LONG_T2 = 6872              # at F 200, K 32 on 132 SMs: the shortest 2T whose W.H contraction takes 120-column tiles (others: 104)
SHORT_T2 = (128, 136, 200, 256, 330, 417, 512, 640)


def limit_lengths(B=MAX_CLIPS, long_clips=33, seed=0):
    """2T of the 8191-clip ragged call (F 200, K 32): `long_clips` clips of LONG_T2 spread through the call at seeded positions, the
    others cycling through SHORT_T2 (128: one CTA in G2; 640: five)."""
    rng = np.random.default_rng(seed)
    T2s = [SHORT_T2[b % len(SHORT_T2)] for b in range(B)]
    for b in rng.choice(np.arange(1, B - 1), long_clips, replace=False):
        T2s[int(b)] = LONG_T2
    return T2s


def describe(launches):
    """Per contraction: the tile-list sizes of its launches and the most search rounds any of them needs."""
    return {c: ([len(l['clips']) for l in ls], max(rounds_needed(len(l['clips'])) for l in ls)) for c, ls in launches.items()}


def test_limit_layout_reaches_three_rounds(lib):
    """The GPU test's 8191-clip ragged layout on an H100's 132 SMs: the W.H contractions launch a 8158-clip group (three rounds; its
    first step, 255, does not divide it) and a 33-clip group (two rounds) whose clips the stable sort moves past the others; G2 and G4
    launch all 8191 (three rounds, first step 256 does not divide 8191); some clips own one CTA, others many.  Every CTA of every
    launch finds its clip in the mirror of the search."""
    F, K = 200, 32
    T2s = limit_lengths()
    launches = launch_plan(lib, H100_SMS, F, T2s, K)
    d = describe(launches)
    assert d['G1/G3'] == ([MAX_CLIPS - 33, 33], 3) and d['G2'] == ([MAX_CLIPS], 3) and d['G4'] == ([MAX_CLIPS], 3), d
    assert [l['bn'] for l in launches['G1/G3']] == [104, 120]
    assert launches['G1/G3'][1]['clips'] == sorted(b for b, t in enumerate(T2s) if t == LONG_T2)
    plans = tile_plans(lib, H100_SMS, F, T2s, K)
    assert plans[128][6] == 1 and plans[LONG_T2][6] > 1 and plans[LONG_T2][5] > 100
    for c, ls in launches.items():
        for l in ls:
            assert check_search(l['cta_begin'], l['ctas']) == rounds_needed(len(l['clips'])), c
    assert plane_launches(launches) == 6                 # G1 and G3 twice each, G2 and G4 once


def test_launch_plan_of_mixed_plans(lib):
    """Lengths whose solo plans differ in every width (F 513, K 1024): the mirror's groups are the distinct widths, each group's clips
    in call order, and its CTA total the sum of the planner's CTA counts."""
    F, K = 513, 1024
    T2s = [3744, 250, 1250, 622, 3000, 130, 1874, 938, 2500]
    launches = launch_plan(lib, H100_SMS, F, T2s, K)
    plans = tile_plans(lib, H100_SMS, F, T2s, K)
    for c, name in enumerate(CONTRACTIONS):
        ls = launches[name]
        assert [l['bn'] for l in ls] == sorted({plans[t][c] for t in T2s})
        for l in ls:
            assert l['clips'] == sorted(l['clips']) and all(plans[T2s[i]][c] == l['bn'] for i in l['clips'])
            assert l['ctas'] == sum(plans[T2s[i]][5 + c] for i in l['clips'])
            check_search(l['cta_begin'], l['ctas'])
    assert plane_launches(launches) > 5


def test_workspace_past_4_gib_at_the_limit(lib):
    """The 8191-clip cases' workspaces pass 2^32 bytes; B = 8192 is refused by both size queries."""
    from test_klnmf_ragged_cpu import lengths
    assert lib.gccnmf_klnmf_batched_workspace_bytes(MAX_CLIPS, 129, 1024, 32) > 1 << 32
    assert lib.gccnmf_klnmf_batched_workspace_bytes(MAX_CLIPS + 1, 129, 1024, 32) == 0
    T2s = limit_lengths()
    assert lib.gccnmf_klnmf_ragged_workspace_bytes(MAX_CLIPS, 200, lengths(*T2s), 32) > 1 << 32
    assert lib.gccnmf_klnmf_ragged_workspace_bytes(MAX_CLIPS + 1, 200, lengths(*(T2s + [128])), 32) == 0
    out = (ctypes.c_int * 8)()
    assert lib.gccnmf_klnmf_tile_plan(H100_SMS, 129, 1024, 32, out) == 0 and out[3] == 8 and MAX_CLIPS * out[3] == 65528
