"""GPU: the all-TDOA argmax on the tensor cores (gccnmf_tdoa_argmax, csrc/gcc_tc.cu) against the float64 kernel
(gccnmf_tdoa_gccnmf) and float64 numpy.

gccnmf_tdoa_argmax finds a provisional argmax with the bf16 hi / lo plane GEMM, flags every (atom, frame) whose best-minus-second
margin is below margin_factor(F) * sum_f |W|, and recomputes the flagged decisions in float64.  Its contract is that every decision
equals the float64 kernel's, on every input.  These tests hold it to that at every supported TDOA count, with both GEMM forms
(persistent, one CTA per tile) and both refinement kernels (candidates, all TDOAs), on ragged m and n tiles, on near-ties only the
refinement can resolve, on NaN, zero and exact-tie inputs, past the capacity of the refinement list, and they measure the error
budget the margin is built from.  Each test asserts that the tensor-core path ran (workspace > 256 bytes) and, where it relies on
the refinement, that decisions were refined.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import gccnmf_oracle as orc  # noqa: E402  (the checker)

SR = 16000
MIC_SEP = 0.2          # metres: 588 us of TDOA range


@pytest.fixture(scope='module')
def h():
    from gcc_nmf_b200._lib import default_handle
    hd = default_handle()
    yield hd
    hd.set_option('argmax_persistent', 1)
    hd.set_option('argmax_refine_shared', 1)
    hd.set_option('force_simt_nmf', 0)


def set_path(h, persistent, refine_shared):
    h.set_option('force_simt_nmf', 0)
    h.set_option('argmax_persistent', persistent)
    h.set_option('argmax_refine_shared', refine_shared)


def tdoas(D, mic_sep=MIC_SEP):
    return orc.getTDOAsInSeconds(mic_sep, D)


def steering(F, D, mic_sep=MIC_SEP):
    return np.ascontiguousarray(orc.getExpJOmegaTau(orc.getFrequenciesInHz(SR, F), tdoas(D, mic_sep)))


def dictionary(rng, F, K):
    """Non-negative atoms of unit L2 norm, like a learnt KL-NMF dictionary."""
    W = rng.random((F, K)) ** 3
    W /= np.sqrt((W ** 2).sum(axis=0))
    return W.astype(np.float32)


def source_at(F, tau):
    """Coherence of a source at TDOA tau (Re(C E[:, d]) peaks where tdoa[d] = tau), complex128."""
    return np.exp(2j * np.pi * orc.getFrequenciesInHz(SR, F)[:, None] * np.atleast_1d(tau)[None, :])


def midpoints(D, pairs, mic_sep=MIC_SEP):
    """TDOAs half-way between hypotheses d and d + 1 for every d in `pairs`."""
    t = tdoas(D, mic_sep)
    d = np.asarray(pairs)
    return 0.5 * (t[d] + t[d + 1])


def mixed_coherence(rng, F, T, D, near_tie_frames=8):
    """PHAT coherence (unit modulus, complex64) of two sources at fixed TDOAs with per-frame gains over random-phase noise, plus a
    few frames of a single source half-way between two hypotheses (near-ties that only the refinement resolves)."""
    t = tdoas(D)
    taus = rng.uniform(t[0], t[-1], 2)
    X = 0.7 * np.exp(2j * np.pi * rng.random((F, T)))
    for tau in taus:
        X += rng.random(T)[None, :] * 2.0 * source_at(F, tau)
    C = X / np.abs(X)
    frames = rng.choice(T, near_tie_frames, replace=False)
    C[:, frames] = source_at(F, midpoints(D, rng.integers(0, D - 1, near_tie_frames)))
    return C.astype(np.complex64)


def tc_argmax(h, coh, E, W):
    """gccnmf_tdoa_argmax into an output pre-filled with -1, so that a decision the kernels never write cannot pass.
    Returns (argmax (K, T) int32 cuda, refined count)."""
    import torch
    F, T = coh.shape
    D, K = E.shape[1], W.shape[1]
    nbytes = h.lib.gccnmf_tdoa_argmax_workspace_bytes(F, T, D, K)
    assert nbytes > 256, 'the tensor-core path does not take this shape'
    argmax = torch.full((K, T), -1, dtype=torch.int32, device=h.device)
    refined = torch.full((1,), -1, dtype=torch.int32, device=h.device)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=h.device)
    h.check(h.lib.gccnmf_tdoa_argmax(h.h, coh.data_ptr(), F, T, E.data_ptr(), D, W.data_ptr(), K, argmax.data_ptr(), refined.data_ptr(),
                                     ws.data_ptr(), ws.numel(), h.stream))
    torch.cuda.synchronize()
    return argmax, int(refined.item())


def float64_argmax(h, coh, E, W):
    _, argmax = h.tdoa_gccnmf(coh, E, W, want_values=False, want_argmax=True)
    return argmax


def numpy_argmax(coh, E, W, frames):
    return np.argmax(orc.getGCCNMFAllTDOAs(coh[:, frames], E, W), axis=1)


def check_numpy(argmax, coh, E, W, frames):
    """argmax[:, frames] == numpy's argmax wherever numpy's best and second values are more than 1e-12 sum_f |W| apart (NaN
    decisions included).  Closer decisions are ordered by the summation order, and numpy's BLAS order is not the float64
    kernel's; those are held to the float64 kernel.  Returns the fraction of decisions compared."""
    v = orc.getGCCNMFAllTDOAs(coh[:, frames], E, W)                     # (K, D, frames)
    top2 = np.sort(v, axis=1)[:, -2:]
    gap = (top2[:, 1] - top2[:, 0]) / np.maximum(np.abs(W).astype(np.float64).sum(axis=0), 1e-300)[:, None]
    compared = ~(gap <= 1e-12)
    a = argmax.cpu().numpy()[:, frames]
    assert np.array_equal(a[compared], np.argmax(v, axis=1)[compared])
    return compared.mean()


def check(h, coh, E, W, frames, label=''):
    """Tensor-core argmax == float64 kernel on every decision, and == numpy on `frames` (check_numpy); returns the refined count."""
    import torch
    cd, Ed, Wd = h.to_device(coh), h.to_device(E), h.to_device(W)
    argmax, refined = tc_argmax(h, cd, Ed, Wd)
    argmax64 = float64_argmax(h, cd, Ed, Wd)
    bad = (argmax != argmax64).sum().item()
    assert torch.equal(argmax, argmax64), '%s: %d of %d decisions differ from the float64 kernel (%d refined)' % (label, bad, argmax.numel(), refined)
    assert check_numpy(argmax, coh, E, W, frames) > 0.8, label
    return refined


# ------------------------------------------------------------------------------------ 1. shapes x options
# (F, T, K) per TDOA count: every D has a ragged last m tile (K = 72 or 200) and a K that is a multiple of 128, and T D % 256 != 0
# everywhere (a ragged last n tile: 256 / D frames per tile, fewer in the last); F = 33 (the smallest covered F plus one), 513,
# 1025 and 2049 (n_fft 4096).
SHAPES = {
    8: [(33, 97, 72), (2049, 70, 128)],
    16: [(513, 41, 200), (1025, 50, 256)],
    32: [(2049, 37, 128), (33, 30, 200)],
    64: [(1025, 45, 200), (513, 37, 128)],
    128: [(513, 23, 72), (2049, 19, 256)],
}


@pytest.mark.parametrize('refine_shared', [1, 0])
@pytest.mark.parametrize('persistent', [1, 0])
@pytest.mark.parametrize('D', [8, 16, 32, 64, 128])
def test_argmax_shapes_and_options_match_float64(h, D, persistent, refine_shared):
    """Every TDOA count x GEMM form (persistent kernel for D >= 32, or plane GEMM + whole-tile epilogue) x refinement kernel
    (candidates, or all TDOAs: shared-memory E for D <= 64, one warp per pair for D = 128), ragged m and n tiles, F up to 2049."""
    for F, T, K in SHAPES[D]:
        assert K % 128 == 0 or K in (72, 200)
        assert (T * D) % 256 != 0
        rng = np.random.default_rng([D, F, T, K])
        coh = mixed_coherence(rng, F, T, D)
        E = steering(F, D)
        W = dictionary(rng, F, K)
        set_path(h, persistent, refine_shared)
        frames = np.r_[0:3, T - 3:T]                             # the first frames and the last (ragged) n tile's
        refined = check(h, coh, E, W, frames, label='D=%d F=%d T=%d K=%d persistent=%d refine_shared=%d' % (D, F, T, K, persistent, refine_shared))
        print('D=%d F=%d T=%d K=%d persistent=%d refine_shared=%d: %d of %d refined' % (D, F, T, K, persistent, refine_shared, refined, K * T))
        assert 0 < refined <= h.lib.gccnmf_tdoa_argmax_refine_capacity(K, T)


# ------------------------------------------------------------------------------------ 2. constructed near-ties
@pytest.mark.parametrize('refine_shared', [1, 0])
@pytest.mark.parametrize('D', [8, 16, 32, 64, 128])
def test_argmax_near_ties_are_resolved_by_refinement(h, D, refine_shared):
    """Every frame is a source half-way between two neighbouring hypotheses, rounded to complex64: the two columns differ by 1e-11
    to 1e-9 of sum_f W (the complex64 rounding breaks the symmetry), far below what the 3-product GEMM resolves and far above
    float64 order noise, and either one can be the larger, so only the float64 refinement gives the right answer.  A 2 cm spacing
    keeps every steering phase difference below pi, so the two neighbours are the top two.  Every neighbouring pair, those in the
    upper candidate words of D = 128 included, is the tie of some frame."""
    F, K, mic_sep = 513, 200, 0.02
    T = max(2 * (D - 1), 64) + 3                                # T D >= 256 and not a multiple of 256
    rng = np.random.default_rng(100 + D)
    coh = source_at(F, midpoints(D, np.arange(T) % (D - 1), mic_sep)).astype(np.complex64)
    E = steering(F, D, mic_sep)
    W = dictionary(rng, F, K)
    set_path(h, 1, refine_shared)
    refined = check(h, coh, E, W, np.arange(T), label='near-ties D=%d refine_shared=%d' % (D, refine_shared))
    print('near-ties D=%d refine_shared=%d: %d of %d refined' % (D, refine_shared, refined, K * T))
    assert refined == K * T <= h.lib.gccnmf_tdoa_argmax_refine_capacity(K, T)


# ------------------------------------------------------------------------------------ 3. NaN, zero and exact-tie inputs
@pytest.mark.parametrize('refine_shared', [1, 0])
@pytest.mark.parametrize('D', [8, 16, 32, 64, 128])
def test_argmax_special_values(h, D, refine_shared):
    """numpy's argmax rules: NaN is the maximum (and the first NaN wins), the first of equal maxima wins.
      - all-zero frames: the PHAT coherence is 0/0 = NaN in every bin -> index 0;
      - one NaN bin in a frame: every TDOA's value is NaN -> index 0;
      - an all-zero atom: every value is 0, an exact tie -> index 0;
      - two identical columns of E (1 and D - 2) with sources at tdoa[1]: an exact tie -> index 1;
      - polarity-inverted mono at a 1 cm spacing: every value is negative and the two end TDOAs tie exactly -> index 0."""
    import torch
    F, T, K = 513, 64, 128
    rng = np.random.default_rng(200 + D)
    E = steering(F, D)
    E[:, D - 2] = E[:, 1]
    X = (rng.standard_normal((2, F, T)) + 1j * rng.standard_normal((2, F, T))).astype(np.complex64)
    zero_frames, nan_bin_frame = [3, T - 1], 10
    X[:, :, zero_frames] = 0
    coh, _, _ = h.phat_angspec(h.to_device(X), None, want_angular=False, want_mean=False)
    coh = coh.cpu().numpy()
    assert np.isnan(coh[:, zero_frames]).all()
    coh[100, nan_bin_frame] = np.nan
    tie_frames = np.arange(20, 40)
    coh[:, tie_frames] = source_at(F, np.full(len(tie_frames), tdoas(D)[1])).astype(np.complex64)
    W = dictionary(rng, F, K)
    zero_atom = 5
    W[:, zero_atom] = 0
    set_path(h, 1, refine_shared)
    cd, Ed, Wd = h.to_device(coh), h.to_device(E), h.to_device(W)
    argmax, refined = tc_argmax(h, cd, Ed, Wd)
    argmax64 = float64_argmax(h, cd, Ed, Wd)
    assert torch.equal(argmax, argmax64), (argmax != argmax64).sum().item()
    a = argmax.cpu().numpy()
    assert (a[:, zero_frames] == 0).all() and (a[:, nan_bin_frame] == 0).all() and (a[zero_atom] == 0).all()
    others = np.arange(K) != zero_atom
    assert (a[others][:, tie_frames] == 1).all()
    frames = np.r_[zero_frames, nan_bin_frame, tie_frames[:4], 0:2]
    ref = numpy_argmax(coh, E, W, frames)
    assert (ref[:, :3] == 0).all() and (ref[others, 3:7] == 1).all() and (ref[zero_atom] == 0).all()      # numpy's rules, as stated
    assert check_numpy(argmax, coh, E, W, frames) > 0.5           # 4 of the 9 frames are exact ties, compared above
    print('special values D=%d refine_shared=%d: %d of %d refined' % (D, refine_shared, refined, K * T))
    assert refined >= K * (len(zero_frames) + 1 + len(tie_frames))      # NaN frames and exact ties are always refined
    assert refined <= h.lib.gccnmf_tdoa_argmax_refine_capacity(K, T)

    # negative maxima: C = -1 and steering phases below pi / 2, so every value is negative; the maximum is at the two ends, tied
    E1 = steering(F, D, mic_sep=0.01)
    neg = np.full((F, T), -1, np.complex64)
    cd = h.to_device(neg)
    E1d = h.to_device(E1)
    argmax, refined = tc_argmax(h, cd, E1d, Wd)
    argmax64 = float64_argmax(h, cd, E1d, Wd)
    assert torch.equal(argmax, argmax64), (argmax != argmax64).sum().item()
    assert (argmax.cpu().numpy() == 0).all()
    assert (numpy_argmax(neg, E1, W, np.arange(2)) == 0).all()
    assert refined == K * T


# ------------------------------------------------------------------------------------ 4. mono input, below capacity
def mono_coherence(h, rng, F, T):
    """PHAT coherence of two identical channels: real, 1 to float32 rounding, in every bin."""
    X = (rng.standard_normal((F, T)) + 1j * rng.standard_normal((F, T))).astype(np.complex64)
    coh, _, _ = h.phat_angspec(h.to_device(np.stack([X, X])), None, want_angular=False, want_mean=False)
    return coh


@pytest.mark.parametrize('refine_shared', [1, 0])
@pytest.mark.parametrize('D', [16, 64, 128])
def test_argmax_mono_input_every_decision_refined(h, D, refine_shared):
    """Identical channels: every TDOA value is sum_f W cos(2 pi f tau), so the two central TDOAs of a symmetric grid tie to float64
    rounding (the grid is symmetric only to rounding) in every decision.  All of them are refined, and the refinement must order
    them exactly as the float64 kernel does: one fma chain over the bins in order."""
    import torch
    F, T, K = 513, 500, 128                                     # K T = 64 000 <= the list's capacity of 65 536
    rng = np.random.default_rng(300 + D)
    coh = mono_coherence(h, rng, F, T)
    E = h.to_device(steering(F, D))
    W = h.to_device(dictionary(rng, F, K))
    set_path(h, 1, refine_shared)
    argmax, refined = tc_argmax(h, coh, E, W)
    argmax64 = float64_argmax(h, coh, E, W)
    print('mono D=%d refine_shared=%d: %d of %d refined, %d decisions differ' % (D, refine_shared, refined, K * T,
                                                                                (argmax != argmax64).sum().item()))
    assert refined > K * T // 2
    assert refined <= h.lib.gccnmf_tdoa_argmax_refine_capacity(K, T)
    assert torch.equal(argmax, argmax64)


# ------------------------------------------------------------------------------------ 5. refinement-list overflow, end to end
def test_argmax_overflow_falls_back_to_float64_end_to_end(h):
    """Mono input with K T = 131 072 > the list's capacity of 65 536: nearly every decision is a near-tie, the list overflows,
    and every host caller must fall back to the float64 kernel; the fused one-call flow must report it in status bit 2."""
    import torch
    import gcc_nmf_b200.gccNMFFunctions as fn
    from gcc_nmf_b200.pipeline import GCCNMFPipeline
    from gcc_nmf_b200.synth import synthetic_stereo
    N, hop, D, K, I = 1024, 256, 64, 128, 5
    T = 1024
    x = synthetic_stereo(2.0 + (N + hop * (T - 1)) / SR, seed=5)[:, :N + hop * (T - 1)]
    x = np.ascontiguousarray(np.stack([x[0], x[0]]))            # mono: identical channels
    set_path(h, 1, 1)
    pipe = GCCNMFPipeline(SR, N, hop, D, 0.1, K, I, handle=h)
    try:
        r = pipe.enhance(h.to_device(x))
    except ValueError as e:
        pytest.fail('peak picking found no target on the mono input: %s' % e)
    assert len(r['targetTDOAIndexes']) == 1
    coh, W = r['coherence'], r['W']
    assert tuple(coh.shape) == (N // 2 + 1, T)
    capacity = h.lib.gccnmf_tdoa_argmax_refine_capacity(K, T)
    assert capacity == 65536 and r['refinedDecisions'] > capacity
    argmax64 = float64_argmax(h, coh, pipe.E, W)
    assert torch.equal(r['argMaxGCCNMF'], argmax64)
    _, refined = tc_argmax(h, coh, pipe.E, W)
    print('overflow: %d of %d decisions flagged, capacity %d' % (refined, K * T, capacity))
    assert refined > capacity
    host = fn.getGCCNMFArgMaxTDOA(coh.cpu().numpy(), pipe.frequenciesInHz, 0.1, D, W.cpu().numpy())
    assert np.array_equal(host, argmax64.cpu().numpy())
    fused = pipe.run_fused(h.to_device(x), 0)
    torch.cuda.synchronize()
    assert int(fused['status'].item()) == 4                       # bit 2 only: the target was found
    with pytest.raises(RuntimeError):
        pipe.raise_on_status(fused['status'])


# ------------------------------------------------------------------------------------ 6. the error budget behind the margin
@pytest.mark.parametrize('F', [513, 1025, 2049])
def test_argmax_gemm_error_within_margin_budget(h, F):
    """The per-value error budget margin_factor(F) is built from (csrc/gcc_tc.cu, margin_factor): 3 x 2^-18 for the bf16 hi / lo
    products, 2^-24 for G's float32 rounding and 2^-24 per accumulation over 3 F / 16 accumulations, relative to
    sum_f |W| max |G|, with 25 % slack; the margin is twice that.  Worst case for the accumulator: coherent data, W >= 0 and
    G in [0.5, 1].  This is a proxy: it runs the plane GEMM in the argmax GEMM's configuration (A = W MN-major, B = G K-major,
    256-column tiles, i.e. plane_gemm_kernel<256, 32, true, false>), and the persistent argmax kernel states that it does the
    same arithmetic."""
    import torch
    K, N = 256, 512
    g = torch.Generator(device='cpu').manual_seed(F)
    W = torch.rand(F, K, generator=g) ** 3
    W /= W.norm(dim=0)
    G = 0.5 + 0.5 * torch.rand(N, F, generator=g)
    Wd, Gd = W.to(h.device), G.to(h.device)
    DT = h.gemm_planes(Wd, Gd, a_mn_major=True, b_mn_major=False, tile_n=256)
    torch.cuda.synchronize()
    ref = Gd.double() @ Wd.double()                                            # (N, K)
    scale = Wd.double().abs().sum(0)[None, :] * Gd.double().abs().max()
    measured = ((DT[0].double() - ref).abs() / scale).max().item()
    budget = 1.25 * (3 / 2 ** 18 + (1 + 3 * F / 16) / 2 ** 24)
    print('margin budget F=%d: max error %.3e of sum|W| max|G| = %.3f of the per-value budget %.3e' % (F, measured, measured / budget, budget))
    assert measured <= budget
