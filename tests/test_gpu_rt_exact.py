"""GPU: the real-time block path (csrc/rt.cu) stage by stage against the bit-exact host model of oracle/rt_exact.py.

Each block runs through a RealtimeEngine (input / output rings on the device, one graph launch) and through a twin engine fed by
oracle.OverlapAddProcessorOracle (the reference's rings on the host, the twin's processFrames in between).  The two must agree
bit for bit on the output block and on every export item, which pins the ring cut, the overlap-add and the emit.  Every stage is
then checked against the model from the device's output of the stage before it:
  X         float64 rfft of the float32 windowed frame     max |dX| <= 2e-7 max |X|; >= 98 % of the float32 parts of a run bit-equal
  gccPHAT, inferred H, per-atom TDOA argmax, atom mask (boxcar), GCC-PHAT history, its index, target TDOA     bit-exact
  atom mask (window mode)      <= 4 + 2 x float64 ulps, x = (dist / eps)^beta (CUDA exp, and pow's error times exp's condition)
  Y         <= 1 float32 ulp of the float64 filter (the float64 sums may be contracted to DFMA)
  frames    float64 irfft(Y) . window, relative to the stereo frame's peak (SYNTHESIS_BAR, 4x the worst measured on the H100)
The multi-stream cases check the wide atoms tile and the slot-grouped inference / filter kernels against the model directly."""
import math

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import gccnmf_oracle as orc  # noqa: E402
from oracle import rt_exact as rx  # noqa: E402

F32 = np.float32
SR, MIC_SEP = 16000, 0.1
SYNTHESIS_BAR = 2e-6
STATS = {'x_bit_equal': [], 'x_err': 0.0, 'y_bit_equal': [], 'y_ulps': 0.0, 'synthesis_err': 0.0, 'mask_ulps': 0.0}


# ------------------------------------------------------------------------------------------------ inputs
def _steering(N, D, mirrored=False):
    """expJOmegaTau (F, D) complex64 of GCCNMFProcessor.buildConstants; mirrored: column D-1-d = conj(column d), i.e.
    tau[D-1-d] = -tau[d] exactly."""
    from gcc_nmf_b200 import gccNMFFunctions as fn
    freq = np.linspace(0, SR / 2, N // 2 + 1).astype(F32)
    maxT = MIC_SEP / fn.SPEED_OF_SOUND_IN_METRES_PER_SECOND
    tdoas = np.linspace(-maxT, maxT, D).astype(F32)
    E = np.exp(np.outer(freq, -(2j * np.pi) * tdoas)).astype(np.complex64)
    if mirrored:
        for d in range(D // 2):
            E[:, D - 1 - d] = np.conj(E[:, d])
        if D % 2:
            E[:, D // 2] = 1
    return E


def _dictionary(F, K, seed):
    return ((np.random.default_rng(seed).random((F, K)) ** 3) + 1e-3).astype(F32)


def _audio(B, blocks, seed):
    """(blocks, 2, B) float32 synthetic two-source mixture."""
    from gcc_nmf_b200.synth import synthetic_stereo
    n = blocks * B
    x = synthetic_stereo(n / float(SR) + 0.01, seed=seed)[:, :n]
    return np.ascontiguousarray(x.reshape(2, blocks, B).transpose(1, 0, 2))


def _windows(N, kind, hop):
    from gcc_nmf_b200.online import getAsymmetricAnalysisWindow, getAsymmetricSynthesisWindow
    if kind == 'asym':
        return getAsymmetricAnalysisWindow(N, 2 * hop, 0).astype(F32), getAsymmetricSynthesisWindow(N, 2 * hop, 0).astype(F32)
    w = np.sqrt(np.hamming(N).astype(F32))
    return w, w


PARAMS = dict(targetTDOAIndex=None, epsilon=2.0, beta=1.0, noiseFloor=0.0, mode=1, separationEnabled=True, localizationEnabled=True,
              localizationWindowSize=6)


# ------------------------------------------------------------------------------------------------ host selection (rt.cu)
def _sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def atoms_form(K, D, pairs, sm):
    """rt_enqueue_atoms: <8, 8> once ceil(K / 128) ceil(pairs / (128 / Dp)) CTAs reach the SM count, else <Dp / 16, 1>."""
    Dp = 32 if D <= 32 else 64 if D <= 64 else 128
    big = -(-K // 128) * -(-pairs // (128 // Dp))
    return ((8, 8) if big >= sm else (Dp // 16, 1)), 128 // Dp


def slots_grouped(ctas_x, S, SG, sm):
    """rt_group_slots."""
    return SG > 1 and S > 1 and ctas_x * -(-S // SG) >= 4 * sm


# ------------------------------------------------------------------------------------------------ stage checks
def _check_stages(c, p, ex, frames_in, frames_out, prev, atoms, H0):
    """Every stage of one block against the model, each from the device's output of the stage before."""
    W, E, wa, ws = c['W'], c['E'], c['wa'], c['ws']
    X = ex[3]
    Xm = rx.analysis(frames_in, wa)
    peak = float(np.abs(Xm).max())
    err = float(np.abs(X.astype(np.complex128) - Xm).max())
    assert err <= 2e-7 * peak, (err, peak)
    STATS['x_err'] = max(STATS['x_err'], err / peak if peak else 0.0)
    c['x_equal'] = c.get('x_equal', 0) + int(np.sum(X.view(F32) == Xm.view(F32)))
    c['x_parts'] = c.get('x_parts', 0) + X.size * 2
    G = rx.real_gcc(X, E)
    assert np.array_equal(ex[0], rx.gccphat(G), equal_nan=True)
    if c['inf']:
        H = rx.infer(X, W, H0, c['inf'], c['alpha'], c['eps'])
        assert np.array_equal(ex[6], H, equal_nan=True), np.nanmax(rx.ulps32(ex[6], H))
    if atoms:
        C = rx.atoms(G, W)
        am = rx.argmax_over_tdoa(C)
        bad = np.argwhere(ex[5] != am)
        assert bad.size == 0, (len(bad), bad[:4].tolist())
        c.setdefault('C', []).append(C)
    m = rx.atom_mask(ex[5], prev['target'], p['epsilon'], p['beta'], p['noiseFloor'], p['mode'])
    if p['mode'] == 0:
        assert np.array_equal(ex[2], m)
    else:
        u = rx.ulps64(ex[2], m)
        STATS['mask_ulps'] = max(STATS['mask_ulps'], float(u.max()))
        assert np.all(u <= rx.atom_mask_ulp_bound(ex[5], prev['target'], p['epsilon'], p['beta'])), float(u.max())
    Ym = rx.filter_spectrum(X, W, ex[2], ex[6] if c['inf'] else None, p['separationEnabled'])
    u = rx.ulps32(ex[4], Ym)
    assert float(u.max()) <= 1, float(u.max())
    STATS['y_ulps'] = max(STATS['y_ulps'], float(u.max()))
    STATS['y_bit_equal'].append(float(np.mean(ex[4] == Ym.astype(np.complex64))))
    fm = rx.synthesis(ex[4], ws)
    assert np.array_equal(np.isnan(frames_out), np.isnan(fm))
    # per frame over both channels: rt_synthesis inverts the stereo pair as ONE complex transform (left + i right), so its
    # rounding error scales with the louder channel (a near-silent channel beside a loud one has a large error of its own)
    fpk = np.nanmax(np.abs(fm), axis=(0, 1), initial=0.0)
    ferr = np.nanmax(np.abs(frames_out - fm), axis=(0, 1), initial=0.0)
    rel = float(np.max(np.where(fpk > 0, ferr / np.where(fpk > 0, fpk, 1), ferr)))
    STATS['synthesis_err'] = max(STATS['synthesis_err'], rel)
    assert rel <= SYNTHESIS_BAR, rel
    h, i, t = rx.localize(prev['hist'], prev['index'], ex[0], p['localizationWindowSize'], p['localizationEnabled'], prev['target'])
    assert np.array_equal(ex[7], h, equal_nan=True)
    assert int(ex[8][0]) == i and ex[1][0] == t, (int(ex[8][0]), i, float(ex[1][0]), float(t))


def _case(N, hop, B, nT, K, D, inf=0, alpha=0.0, eps=1e-16, hist=128, window='hamming', mirrored=False, seed=0):
    wa, ws = _windows(N, window, hop)
    return dict(N=N, hop=hop, B=B, nT=nT, K=K, D=D, inf=inf, alpha=alpha, eps=eps, hist=hist, wa=wa, ws=ws,
                W=_dictionary(N // 2 + 1, K, seed), E=_steering(N, D, mirrored))


def _engine(c):
    from gcc_nmf_b200.realtime.engine import RealtimeEngine
    return RealtimeEngine(c['W'], c['E'], c['wa'], c['ws'], c['hop'], c['B'], c['nT'], historyLength=c['hist'], numInferenceIterations=c['inf'],
                          sparsityAlpha=c['alpha'], epsilon=c['eps'])


def _run(c, x, params, atoms_blocks, check=True, x_bit_equal=0.98):
    """x (blocks, 2, B); params {block: set_params keywords} (merged into PARAMS); atoms_blocks: blocks whose per-atom argmax is
    modelled (the fmaf chains are the expensive part of the model).  Returns the device output blocks and last exports."""
    eng, twin = _engine(c), _engine(c)
    ola = orc.OverlapAddProcessorOracle(2, c['N'], c['hop'], c['B'], c['nT'])
    H0 = rx.seeded_H0(c['K'], c['eps']) if c['inf'] else None
    p = dict(PARAMS)
    out = np.zeros_like(x)
    for b in range(x.shape[0]):
        if b in params:
            p.update(params[b])
            eng.set_params(**p)
            twin.set_params(**p)
            p['targetTDOAIndex'] = None
        prev = dict(hist=eng.export(7), index=int(eng.export(8)[0]), target=F32(eng.export(1)[0]))
        out[b] = eng.process_block(x[b])
        cut = {}

        def frames_fn(windowed):
            cut['in'] = windowed.copy()
            cut['out'] = twin.process_frames(windowed).copy()
            return cut['out']
        ref = ola.processFrames(x[b], frames_fn)
        assert np.array_equal(out[b], ref, equal_nan=True), ('block', b)
        ex = {i: eng.export(i) for i in range(9)}
        for i in range(9):
            assert np.array_equal(ex[i], twin.export(i), equal_nan=True), ('export', i, 'block', b)
        if check:
            _check_stages(c, p, ex, cut['in'], cut['out'], prev, b in atoms_blocks, H0)
    if check:
        _assert_x_bit_equal(c, x_bit_equal)
    return out, ex


def _assert_x_bit_equal(c, bar=0.98):
    eq = c['x_equal'] / float(c['x_parts'])
    STATS['x_bit_equal'].append(eq)
    assert eq >= bar, eq


# ------------------------------------------------------------------------------------------------ §3 single engine
CASES = {
    # name: (case, per-block parameters, modelled argmax blocks, intended atoms tile)
    'configs2': (dict(N=512, hop=128, B=128, nT=1, K=1024, D=64, inf=10), {0: dict(targetTDOAIndex=30.0, epsilon=5.0, beta=2.0)}, (9, 19), (4, 1)),
    'configs4': (dict(N=1024, hop=64, B=512, nT=8, K=256, D=128, window='asym'), {0: dict(targetTDOAIndex=60.0, epsilon=8.0)}, (17,), (8, 1)),
    'smallest': (dict(N=64, hop=16, B=48, nT=3, K=1, D=1, inf=2), {0: dict(targetTDOAIndex=0.0)}, tuple(range(20)), (2, 1)),
    'largest_fft': (dict(N=2048, hop=512, B=1024, nT=2, K=17, D=33), {0: dict(targetTDOAIndex=16.0, epsilon=4.0, mode=0)}, (3, 9, 19), (4, 1)),
    'ragged': (dict(N=256, hop=64, B=400, nT=5, K=200, D=65, inf=3, alpha=0.3, eps=0.25), {0: dict(targetTDOAIndex=20.0, epsilon=6.0)},
               (9, 19), (8, 1)),
    'nT6': (dict(N=256, hop=32, B=224, nT=6, K=64, D=32, inf=1), {0: dict(targetTDOAIndex=12.0)}, (9, 19), (2, 1)),
    'nT7': (dict(N=256, hop=32, B=64, nT=7, K=64, D=32, inf=1), {0: dict(targetTDOAIndex=12.0, mode=0, epsilon=3.0)}, (9, 19), (2, 1)),
    'history': (dict(N=256, hop=64, B=256, nT=4, K=64, D=20, hist=5),
                {0: dict(targetTDOAIndex=7.0, noiseFloor=0.1, beta=2.0, epsilon=3.0, localizationWindowSize=3),
                 8: dict(separationEnabled=False, localizationWindowSize=200), 13: dict(separationEnabled=True)}, (5, 10, 19), (2, 1)),
}


@pytest.mark.parametrize('name', list(CASES))
def test_block_stages_match_model(name):
    spec, params, atoms_blocks, form = CASES[name]
    c = _case(**spec, seed=len(name))
    N, hop, B, nT = c['N'], c['hop'], c['B'], c['nT']
    assert atoms_form(c['K'], c['D'], nT, _sm_count())[0] == form
    L = 8 * B
    w_first = L - N - (nT - 1) * hop
    if name == 'nT6':
        assert w_first > L - 3 * B                     # p_first = L - 3 B: the emit range starts before the first window
    if name == 'nT7':
        assert w_first < L - 3 * B                     # p_first = w_first
    if name == 'history':
        assert c['hist'] % nT != 0                     # the history ring wraps inside a block
    x = _audio(B, 20, seed=len(name))
    _run(c, x, params, atoms_blocks)
    print('%s: X bit-equal min %.4f, Y bit-equal min %.4f, worst Y %.2f ulp, worst synthesis %.2e of the frame peak, mask %.1f ulp'
          % (name, min(STATS['x_bit_equal']), min(STATS['y_bit_equal']), STATS['y_ulps'], STATS['synthesis_err'], STATS['mask_ulps']))


# ------------------------------------------------------------------------------------------------ constructed inputs
@pytest.mark.parametrize('D', [32, 64, 128])
def test_mirrored_tdoa_ties_go_to_the_lower_index(D):
    """Mono input (left = right) and mirrored TDOAs: Im(coherence) = 0 and cos is even, so rows d and D-1-d of realGCC are equal
    bit for bit and every atom ties between them, across thread row groups.  The lower index must win."""
    c = _case(N=256, hop=64, B=128, nT=2, K=96, D=D, mirrored=True, seed=D)
    x = _audio(c['B'], 10, seed=D)
    x[:, 1] = x[:, 0]
    _run(c, x, {0: dict(targetTDOAIndex=D / 3.0)}, (8, 9))
    ties = 0
    for C in c['C']:
        am = np.argmax(C, axis=1)                                         # (nT, K), model values
        mirror = np.take_along_axis(C, (D - 1 - am)[:, None, :], axis=1)[:, 0]
        best = np.take_along_axis(C, am[:, None, :], axis=1)[:, 0]
        assert np.array_equal(best, mirror) and np.all(am < D - 1 - am)   # the ties exist, and the model takes the lower index
        ties += am.size
    assert ties == 2 * c['nT'] * c['K']


def test_digital_silence_nan_pattern():
    """Zeros at the start, in the middle and in one channel: NaN coherence, argmax 0 for every atom, NaN gccPHAT columns in the
    history and, with inference, NaN in the Wiener filter and the output ring.  Every NaN must be where the model puts it."""
    c = _case(N=256, hop=64, B=256, nT=4, K=64, D=32, inf=2, seed=3)
    x = _audio(c['B'], 24, seed=3)
    x[0:4] = 0
    x[9:14] = 0
    x[17:22, 1] = 0
    # rt_analysis transforms the stereo pair as one complex FFT, so a near-silent channel beside a loud one carries the loud
    # one's float64 rounding: its float32 X parts round differently more often (92 % bit-equal on the H100); max |dX| still holds
    out, _ = _run(c, x, {0: dict(targetTDOAIndex=10.0, localizationWindowSize=3)}, (2, 11, 19), x_bit_equal=0.9)
    assert np.isnan(out).any() and not np.isnan(out).all()
    sil = c['C'][1]
    assert np.isnan(sil).all()


def test_power_of_two_scaling_is_exact():
    """x 2^20 and x 2^-20: gccPHAT, atom mask, argmax and target bit-identical; X, Y, H and the output blocks scale exactly."""
    c = _case(N=256, hop=64, B=128, nT=2, K=64, D=32, inf=3, seed=5)
    x = _audio(c['B'], 12, seed=5)
    params = {0: dict(targetTDOAIndex=11.0)}
    base, e0 = _run(c, x, params, (), check=False)
    for k in (20, -20):
        s = F32(2.0 ** k)
        out, e = _run(c, x * s, params, (), check=False)
        for i in (0, 1, 2, 5, 7, 8):
            assert np.array_equal(e[i], e0[i], equal_nan=True), (k, i)
        for i in (3, 4, 6):
            assert np.array_equal(e[i], e0[i] * s), (k, i)
        assert np.array_equal(out, base * s), k


def test_localization_window_below_one_is_rejected():
    from gcc_nmf_b200 import _lib
    from gcc_nmf_b200.realtime.multistream import MultiStreamRealtimeEngine
    c = _case(N=256, hop=64, B=128, nT=2, K=16, D=8)
    eng = _engine(c)
    for w in (0, -1):
        with pytest.raises(_lib.ParameterError, match='localization_window'):
            eng.set_params(localizationWindowSize=w)
    eng.set_params(localizationWindowSize=1)
    m = MultiStreamRealtimeEngine(c['W'], c['E'], c['wa'], c['ws'], c['hop'], c['B'], c['nT'], 3)
    with pytest.raises(_lib.ParameterError, match='slot 1: localization_window'):
        m.set_params([0, 1, 2], localizationWindowSize=[6, 0, 6])
    m.set_params([0, 1, 2], localizationWindowSize=1)


# ------------------------------------------------------------------------------------------------ §4 multi-stream forms
def _multi_run(c, S, check_slots, blocks, atoms_blocks, mono_slot=None):
    """S slots, each its own audio; the checked slots against the model (stages, and the output block through the reference's
    rings around float32(model synthesis of the device's Y))."""
    from gcc_nmf_b200.realtime.multistream import MultiStreamRealtimeEngine
    m = MultiStreamRealtimeEngine(c['W'], c['E'], c['wa'], c['ws'], c['hop'], c['B'], c['nT'], S, historyLength=c['hist'],
                                  numInferenceIterations=c['inf'], sparsityAlpha=c['alpha'], epsilon=c['eps'])
    p = dict(PARAMS, targetTDOAIndex=c['D'] / 3.0)
    m.set_params(range(S), **p)
    p['targetTDOAIndex'] = None
    clips = [_audio(c['B'], blocks, seed=100 + i) for i in range(4)]
    x = np.stack([clips[s % 4] for s in range(S)], axis=1)                # (blocks, S, 2, B)
    if mono_slot is not None:
        x[:, mono_slot, 1] = x[:, mono_slot, 0]
    olas = {s: orc.OverlapAddProcessorOracle(2, c['N'], c['hop'], c['B'], c['nT']) for s in check_slots}
    H0 = rx.seeded_H0(c['K'], c['eps']) if c['inf'] else None
    for b in range(blocks):
        prev = {s: dict(hist=m.export(s, 7), index=int(m.export(s, 8)[0]), target=F32(m.export(s, 1)[0])) for s in check_slots}
        y = m.process_blocks(x[b]).copy()
        for s in check_slots:
            ex = {i: m.export(s, i) for i in range(9)}
            cut = {}

            def frames_fn(windowed):
                cut['in'] = windowed.copy()
                cut['out'] = rx.synthesis(ex[4], c['ws']).astype(F32)
                return cut['out']
            ref = olas[s].processFrames(x[b, s], frames_fn)
            assert np.abs(y[s] - ref).max() <= math.ceil(c['N'] / c['hop']) * SYNTHESIS_BAR * max(np.abs(cut['out']).max(), 1e-30)
            _check_stages(c, p, ex, cut['in'], cut['out'], prev[s], b in atoms_blocks, H0)
    _assert_x_bit_equal(c)
    return m


@pytest.mark.parametrize('D', [32, 64, 128])
def test_wide_atoms_tile_against_model(D):
    """Enough slots for the 128 x 128 atoms tile at 4, 2 and 1 (slot, frame) pairs per CTA, the last CTA row partial where it
    can be; mirrored TDOAs with a mono slot 0 (ties across row groups inside the wide tile)."""
    sm = _sm_count()
    c = _case(N=256, hop=64, B=64, nT=1, K=256, D=D, mirrored=True, seed=D + 1)
    ktiles = -(-c['K'] // 128)
    rows = -(-sm // ktiles)
    Dp = 32 if D <= 32 else 64 if D <= 64 else 128
    ppc = 128 // Dp
    S = (rows - 1) * ppc + max(ppc - 1, 1)
    form, per_cta = atoms_form(c['K'], D, S * c['nT'], sm)
    assert form == (8, 8) and per_cta == ppc and -(-S // ppc) * ktiles >= sm
    last_row = (rows - 1) * ppc
    _multi_run(c, S, sorted({0, last_row, S - 1}), 10, (8, 9), mono_slot=0)


def test_grouped_inference_and_filter_slots_against_model():
    """nT = 3 with inference: two slots per warp in rt_inf_ratio, rt_inf_update and rt_filter, the last group holding one slot."""
    sm = _sm_count()
    c = _case(N=256, hop=64, B=192, nT=3, K=64, D=32, inf=2, seed=7)
    F, K, nT = c['N'] // 2 + 1, c['K'], c['nT']
    SG_inf, SG_filter = 16 // (2 * nT), 8 // nT
    assert SG_inf == 2 and SG_filter == 2
    need = -(-4 * sm // min(-(-F // 8), -(-K // 8)))                   # slot groups for 4 waves in the narrowest grid
    S = 2 * need - 1
    for ctas_x, SG in ((-(-F // 8), SG_inf), (-(-K // 8), SG_inf), (-(-F // 8), SG_filter)):
        assert slots_grouped(ctas_x, S, SG, sm)
    assert S % 2 == 1
    _multi_run(c, S, [0, S - 2, S - 1], 10, (9,))
