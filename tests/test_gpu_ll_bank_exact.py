"""GPU: the low-latency engine's plain, steering-bank (llbank) and dictionary-bank (lldict) forms, every column of a call held to an
independent reference.  Each call is checked teacher-forced from the engine's own exports, on its whole (valid) frames, bit for bit
and NaN-equal, per (dictionary i, table j) group of columns:
  angular              h.phat_angspec(X, E_j) on the exported X
  coherence            offline_exact.coherence(X)
  argmax               h.tdoa_gccnmf(coherence, E_j, W_i), the float64 kernel: every decision equals its decision
  source values        the same kernel's values (D, K_i, T) gathered at the exported source targets (target_gccnmf's contract)
  masks                offline_exact.atom_mask (boxcar, each stream's epsilon) / coeff_mask of the exported values
  wiener, Y            offline_exact.wiener_apply(mask, W_i, X), or wiener_apply_h with the engine's H
  H                    oracle/ll_exact.infer from the exported X and the H0 the engine draws for K_i
Rows at or above a column's K_i hold the defined fill (argmax -1, masks, values and H 0).  Every engine runs as graphs and kernel
by kernel, and the two runs agree bit for bit.  The cases cover every TDOA count with both bank forms and P 0 and 2, stream counts
per entry that straddle every column tile the bank kernels cut, dictionaries of 1 .. 257 atoms, F = 17 and 129 and the configs[4]
shape, the tensor argmax with its float64 refinement and the gated float64 fallback, inference on every engine form, the
inference kernel's shared-memory edges, and digital silence."""
import numpy as np
import pytest

from gcc_nmf_b200 import lowlatency as ll
from gcc_nmf_b200._lib import ParameterError

pytestmark = pytest.mark.gpu

from oracle import ll_exact as lx  # noqa: E402
from oracle import offline_exact as ox  # noqa: E402

F32 = np.float32
SR = 16000
SPACINGS = [0.05, 0.1, 0.2, 0.3, 0.45, 0.6, 0.8, 1.0]
# column tiles the bank kernels cut from each entry's sorted columns (csrc/gcc.cu, csrc/gcc_tc.cu)
ANG_TILE, PLANE_TILE, SIMT_GN, WIENER_RN, GEMM_COLUMNS = 16, 32, 128, 128, 256
# streams per entry, spread unsorted: one entry empty, the last in use; with 1 and 3 hops per call the column counts straddle
# every tile width above
STEER_COUNTS = [9, 0, 17, 1, 33, 3]
ATOMS = [1, 8, 100, 127, 128, 129, 255, 257, 100]            # K_max 257; the last: a second K = 100 content
DICT_COUNTS = [3, 1, 0, 9, 17, 33, 2, 5, 43]


def _case(kind, D, P=0, C=1, N=256, inf=0, alpha=0.0, K=128, atoms=None, scounts=None, dcounts=None, mono=False, silence=False,
          full=True):
    if kind == 'lldict':
        atoms = list(ATOMS if atoms is None else atoms)
        dcounts = list(DICT_COUNTS[:len(atoms)] if dcounts is None else dcounts)
        S = sum(dcounts)
        if scounts is None:
            a, b = 17, 33 if S >= 52 else 0
            scounts = [a, 0, b, S - a - b] if S > a + b else [0, S]
    else:
        scounts = list(STEER_COUNTS if scounts is None else scounts) if kind == 'llbank' else [1]
        S = sum(scounts) if kind == 'llbank' else 5
        dcounts = None
    return dict(kind=kind, D=D, P=P, C=C, N=N, inf=inf, alpha=alpha, K=K, atoms=atoms, scounts=scounts, dcounts=dcounts, S=S,
                mono=mono, silence=silence, full=full)


def _id(c):
    parts = [c['kind'], 'D%d' % c['D'], 'P%d' % c['P'], 'C%d' % c['C'], 'N%d' % c['N']]
    if c['inf']:
        parts.append('inf%d-a%g' % (c['inf'], c['alpha']))
    parts.append('K%d' % (max(c['atoms']) if c['atoms'] else c['K']))
    return '-'.join(parts + (['mono'] if c['mono'] else []) + (['silence'] if c['silence'] else []))


TDOAS = [4, 8, 16, 32, 64, 128]
SWEEP = [_case(kind, D, P, C=3 if (i + P // 2) % 2 == 0 else 1) for i, D in enumerate(TDOAS) for kind in ('llbank', 'lldict') for P in (0, 2)]
SHAPES = [_case('lldict', 32, 0, C=3, N=32, atoms=[100, 8, 64, 33]),                 # F = 17: the dictionary argmax is SIMT at any D
          _case('llbank', 64, 2, C=1, N=32, K=64),
          _case('llbank', 128, 0, C=3, N=1024, K=256, scounts=[3, 0, 9, 1, 5]),       # configs[4]: N 1024, hop 64, D 128, K 256
          _case('lldict', 128, 0, C=1, N=1024, atoms=[256, 129, 64, 256], dcounts=[9, 3, 0, 17])]
FALLBACK = [_case('llbank', 64, 0, C=1, K=512, scounts=[128, 0, 192, 192], mono=True, full=False),
            _case('lldict', 128, 0, C=1, atoms=[512, 448, 384], dcounts=[200, 120, 192], mono=True, full=False)]
INFERENCE = [_case('ll', 16, 0, C=1, K=1, inf=1, alpha=0.0),
             _case('ll', 64, 2, C=3, K=33, inf=2, alpha=0.5, silence=True),
             _case('llbank', 32, 0, C=3, K=256, inf=7, alpha=0.5, scounts=[3, 0, 9, 1]),
             _case('llbank', 16, 2, C=1, K=31, inf=2, alpha=0.0, scounts=[2, 5, 0, 3]),
             _case('lldict', 32, 0, C=1, inf=2, alpha=0.0, atoms=[33, 100, 256, 1, 31], dcounts=[3, 9, 0, 1, 5], silence=True),
             _case('lldict', 8, 2, C=3, inf=7, alpha=0.5, atoms=[100, 31, 256, 257], dcounts=[2, 0, 3, 1])]
# ll_infer holds (K + F) floats of shared memory: just over 48 KiB (the opt-in branch) and exactly the 227 KiB limit ll_check allows
SMEM = [_case('ll', 4, 0, C=1, K=12160, inf=2, full=False),
        _case('lldict', 4, 0, C=1, atoms=[12160, 100], dcounts=[1, 1], inf=2, full=False),
        _case('ll', 4, 0, C=1, K=58112 - 129, inf=2, full=False),
        _case('lldict', 4, 0, C=1, atoms=[7, 58112 - 129], dcounts=[1, 1], inf=2, full=False)]
CASES = SWEEP + SHAPES + FALLBACK + INFERENCE + SMEM


def _setup(c, seed=0):
    from gcc_nmf_b200 import gccNMFFunctions as fn
    from gcc_nmf_b200.online import getAsymmetricAnalysisWindow, getAsymmetricSynthesisWindow
    N = c['N']
    F = N // 2 + 1
    m, hop = {32: (8, 8), 256: (32, 32), 1024: (64, 64)}[N]
    rng = np.random.RandomState(seed)
    E = [fn.getExpJOmegaTau(fn.getFrequenciesInHz(SR, F), fn.getTDOAsInSeconds(d, c['D'])) for d in SPACINGS[:len(c['scounts'])]]
    if c['kind'] == 'lldict':
        W = [(rng.random_sample((F, k)) + 0.01).astype(F32) for k in c['atoms']]
    else:
        W = (rng.random_sample((F, c['K'])) + 0.01).astype(F32)
    return dict(N=N, F=F, hop=hop, W=W, E=E if c['kind'] != 'll' else E[0], win=getAsymmetricAnalysisWindow(N, m, 0),
                syn=getAsymmetricSynthesisWindow(N, m, 0))


def _audio(S, hops, hop, seed=1, mono=False):
    """S different stereo streams: two delayed sources per stream, the second entering half way (mono: both channels equal)."""
    rng = np.random.RandomState(seed)
    n = hops * hop
    x = np.zeros((S, 2, n))
    for s in range(S):
        for i, d in enumerate((s % 7 - 3, 3 - s % 5)):
            v = rng.standard_normal(n + 16)
            part = np.stack([v[8:8 + n], v[8 - d:8 - d + n]])
            part[:, :i * n // 2] = 0
            x[s] += part
    if mono:
        x[:, 1] = x[:, 0]
    return (x / np.abs(x).max()).astype(F32)


def _spread(counts, rng):
    return rng.permutation(np.repeat(np.arange(len(counts)), counts))


def _engine(c, p):
    eng = ll.LowLatencyEngine(p['W'], p['E'], p['win'], p['syn'], p['hop'], numStreams=c['S'], hopsPerCall=c['C'], numSources=c['P'],
                              numInferenceIterations=c['inf'], sparsityAlpha=c['alpha'], targetTDOAEpsilon=2.5)
    rng = np.random.RandomState(c['D'] + 3 * c['C'] + c['P'])
    if c['kind'] != 'll':
        eng.assign_steering(None, _spread(c['scounts'], rng))
    if c['kind'] == 'lldict':
        eng.assign_dictionary(None, _spread(c['dcounts'], rng))
    eps = np.array([1.0, 2.5, 4.0, 0.5, 7.0])[np.arange(c['S']) % 5]
    eng.set_params(None, targetTDOAEpsilon=eps)
    return eng, eps.astype(F32)


def _eq(a, b, what):
    assert a.shape == b.shape, (what, a.shape, b.shape)
    same = np.array_equal(a, b, equal_nan=True)
    if not same:
        bad = np.argwhere(~((a == b) | (np.isnan(a) & np.isnan(b))) if a.dtype.kind in 'fc' else a != b)
        raise AssertionError('%s: %d elements differ, first at %s' % (what, len(bad), bad[:4].tolist()))


def _exports(eng):
    """Every column item of the last call the engine has."""
    items = [ll.EXPORT_X, ll.EXPORT_COHERENCE, ll.EXPORT_ANGULAR, ll.EXPORT_VALID]
    if eng.P:
        items += [ll.EXPORT_SOURCE_TARGETS, ll.EXPORT_SOURCE_VALUES, ll.EXPORT_SOURCE_MASKS, ll.EXPORT_SOURCE_WIENER, ll.EXPORT_SOURCE_Y]
    else:
        items += [ll.EXPORT_TARGETS, ll.EXPORT_ARGMAX, ll.EXPORT_MASKS, ll.EXPORT_WIENER, ll.EXPORT_Y, ll.EXPORT_REFINED, ll.EXPORT_STATUS]
    if eng.inference:
        items.append(ll.EXPORT_H)
    if eng.Qe:
        items.append(ll.EXPORT_ASSIGNMENT)
    if eng.Qd:
        items.append(ll.EXPORT_DICTIONARY_ASSIGNMENT)
    return {w: eng.export(w) for w in items}


def _check_call(c, p, eng, ex, eps):
    """One call's exports against the references (module docstring), on its valid columns."""
    h, torch = eng.h, eng.torch
    hops, P, Kmax = eng.last_hops, eng.P, eng.K
    T = eng.S * hops
    valid = ex[ll.EXPORT_VALID].astype(bool)
    X, coh = ex[ll.EXPORT_X], ex[ll.EXPORT_COHERENCE]
    _eq(coh[:, valid], ox.coherence(X)[:, valid], 'coherence')
    steer = ex.get(ll.EXPORT_ASSIGNMENT, np.zeros(eng.S, np.int32))
    dic = ex.get(ll.EXPORT_DICTIONARY_ASSIGNMENT, np.zeros(eng.S, np.int32))
    groups = lx.column_groups(hops, steer, dic)
    Ws = p['W'] if isinstance(p['W'], list) else [p['W']]
    Es = p['E'] if isinstance(p['E'], list) else [p['E']]
    dev = lambda a: torch.as_tensor(np.ascontiguousarray(a)).to(h.device)      # noqa: E731
    Xd, cohd = dev(X), dev(coh)
    for j in sorted(set(steer.tolist())):
        cols = np.flatnonzero(valid & (steer[np.arange(T) // hops] == j))
        _, ang, _ = h.phat_angspec(Xd, dev(Es[j]), want_mean=False)
        _eq(ex[ll.EXPORT_ANGULAR][:, cols], ang.cpu().numpy()[:, cols], 'angular, table %d' % j)
    eps_col = eps[np.arange(T) // hops]
    H = ex.get(ll.EXPORT_H)
    by_dict = {}
    for (i, j), cols in groups.items():
        cols = cols[valid[cols]]
        if len(cols) == 0:
            continue
        by_dict.setdefault(i, []).append(cols)
        K = Ws[i].shape[1]
        values, am = h.tdoa_gccnmf(cohd, dev(Es[j]), dev(Ws[i]), want_values=bool(P))
        am = am.cpu().numpy()
        tag = '(dictionary %d, table %d)' % (i, j)
        if P:
            tg = ex[ll.EXPORT_SOURCE_TARGETS]                                   # (T, P)
            vals = values.cpu().numpy()
            want = np.stack([vals[tg[cols, q], :, cols].T for q in range(P)])  # (P, K, n)
            got = ex[ll.EXPORT_SOURCE_VALUES]
            _eq(got[:, :K][:, :, cols], want, 'source values ' + tag)
            assert (got[:, K:][:, :, cols] == 0).all(), 'values fill ' + tag
            m = ex[ll.EXPORT_SOURCE_MASKS]
            _eq(m[:, :K][:, :, cols], ox.coeff_mask(got[:, :K][:, :, cols])[0], 'source masks ' + tag)
            assert (m[:, K:][:, :, cols] == 0).all(), 'source masks fill ' + tag
        else:
            got = ex[ll.EXPORT_ARGMAX]
            _eq(got[:K][:, cols], am[:, cols], 'argmax ' + tag)
            assert (got[K:][:, cols] == -1).all(), 'argmax fill ' + tag
            m = ex[ll.EXPORT_MASKS]
            want = ox.atom_mask(got[:K][:, cols], ex[ll.EXPORT_TARGETS][cols], None, eps_col[cols][None, :], 0)
            _eq(m[:K][:, cols], want, 'masks ' + tag)
            assert (m[K:][:, cols] == 0).all(), 'masks fill ' + tag
        if H is not None:
            want = lx.infer(X[:, :, cols], Ws[i], eng._draw_h0(K), c['inf'], c['alpha'], eng._epsilon)
            _eq(lx.split_h(H, cols, K), want, 'H ' + tag)
            assert (lx.split_h(H, cols, Kmax)[K:] == 0).all(), 'H fill ' + tag
    if not c['full']:
        return
    for i, parts in by_dict.items():                       # the filters read W_i only: one check per dictionary
        cols = np.sort(np.concatenate(parts))
        K = Ws[i].shape[1]
        Xc = X[:, :, cols]
        Hc = lx.split_h(H, cols, K) if H is not None else None
        masks = ex[ll.EXPORT_SOURCE_MASKS][:, :K][:, :, cols] if P else ex[ll.EXPORT_MASKS][None, :K][:, :, cols]
        for q in range(len(masks)):
            Y, w = ox.wiener_apply(masks[q], Ws[i], Xc) if Hc is None else ox.wiener_apply_h(masks[q], Ws[i], Hc, Xc)
            gw = ex[ll.EXPORT_SOURCE_WIENER][q] if P else ex[ll.EXPORT_WIENER]
            gy = ex[ll.EXPORT_SOURCE_Y][q] if P else ex[ll.EXPORT_Y]
            _eq(gw[..., cols], w, 'wiener, dictionary %d, source %d' % (i, q))
            _eq(gy[..., cols], Y, 'Y, dictionary %d, source %d' % (i, q))


def _tensor_argmax(c, p):
    """The P = 0 decisions come from the tensor-core GEMM (then the float64 refinement of near-ties) rather than a float64 kernel."""
    if c['P'] or c['D'] < 32 or p['F'] < 32:
        return False
    if c['kind'] == 'lldict':
        return True
    return c['K'] % 8 == 0 and c['K'] >= 64


def _run(c, p, x, use_graph, check):
    eng, eps = _engine(c, p)
    hops = x.shape[2] // p['hop']
    outs, calls, refined, status = [], [], 0, []
    for h0 in range(0, hops, c['C']):
        outs.append(eng.process(x[:, :, h0 * p['hop']:(h0 + c['C']) * p['hop']], use_graph=use_graph))
        ex = _exports(eng)
        if not c['P']:
            refined += int(ex[ll.EXPORT_REFINED][0])
            status.append(int(ex[ll.EXPORT_STATUS][0]))
        if ex[ll.EXPORT_VALID].any():
            if check:
                _check_call(c, p, eng, ex, eps)
            calls.append(ex)
    eng.close()
    return np.concatenate(outs, axis=-1), calls, refined, status


@pytest.mark.parametrize('c', CASES, ids=[_id(c) for c in CASES])
def test_every_column_matches_the_reference(c):
    p = _setup(c)
    Q = -(-p['N'] // p['hop'])
    hops = -(-(Q + c['C']) // c['C']) * c['C']            # the first whole frame ends in hop Q - 1: at least two checked calls
    x = _audio(c['S'], hops, p['hop'], mono=c['mono'])
    if c['silence']:
        x[0] = 0                                           # a silent stream
        x[1, 1] = 0                                        # a silent channel
    y, calls, refined, status = _run(c, p, x, True, True)
    y2, calls2, refined2, status2 = _run(c, p, x, False, False)
    _eq(y2, y, 'output, kernel by kernel')
    assert len(calls) == len(calls2) >= 2
    for a, b in zip(calls, calls2):
        for w in a:
            _eq(b[w], a[w], 'export %d, kernel by kernel' % w)
    if c['mono']:
        assert max(status) == 1                            # the refinement list overflowed: the gated float64 launch decided
    elif _tensor_argmax(c, p):
        assert max(status) == 0 and refined > 0            # the tensor path and its float64 refinement decided
    if c['silence']:
        H = calls[-1][ll.EXPORT_H]
        T = H.shape[1] // 2
        cols = np.arange(c['C'])                           # stream 0's columns
        assert np.isnan(H[:, cols]).any() and np.isnan(H[:, T + cols]).any()


def test_one_atom_past_the_shared_memory_limit_is_refused():
    """(K + F) x 4 = 227 KiB + 4: refused with ParameterError by the library before anything is enqueued."""
    import ctypes
    c = _case('ll', 4, 0, C=1, K=58112 - 129, inf=2)
    p = _setup(c)
    eng, _ = _engine(c, p)
    launches = eng.h.launches
    cfg = ll.LLConfig.from_buffer_copy(bytes(eng.cfg))
    cfg.num_atoms += 1
    assert eng.h.lib.gccnmf_ll_state_bytes(ctypes.byref(cfg)) == 0
    k = eng._const
    with pytest.raises(ParameterError, match='shared memory'):
        eng.h.check(eng.h.lib.gccnmf_ll_init(eng.h.h, ctypes.byref(cfg), k[0].data_ptr(), k[1].data_ptr(), k[2].data_ptr(), k[3].data_ptr(),
                                             float(eng.gain), k[4].data_ptr(), eng.state.data_ptr(), eng.state_bytes, eng.stream.cuda_stream))
    assert eng.h.launches == launches
    W = np.ones((p['F'], c['K'] + 1), F32)
    with pytest.raises(ValueError):
        ll.LowLatencyEngine(W, p['E'], p['win'], p['syn'], p['hop'], numInferenceIterations=1)
    with pytest.raises(ValueError):
        ll.LowLatencyEngine([W, W[:, :5]], [p['E']], p['win'], p['syn'], p['hop'], numInferenceIterations=1)
    eng.close()


# ---------------------------------------------------------------------------------------------- the case lists cover every form
def _columns(c):
    """Column counts of each entry's segment in a call: the steering segments, and the dictionary segments of an lldict engine."""
    s = [n * c['C'] for n in c['scounts']] if c['kind'] != 'll' else []
    d = [n * c['C'] for n in c['dcounts']] if c['kind'] == 'lldict' else []
    return s, d


def _straddles(n, k):
    """A segment of n columns cut into tiles of k: at least one whole tile and a partial last one."""
    return n > k and n % k != 0


def test_cases_cover_every_tdoa_count_and_engine_kind():
    pairs = {(c['D'], c['kind']) for c in CASES}
    for D in TDOAS:
        for kind in ('llbank', 'lldict'):
            assert (D, kind) in pairs
            assert {P for c in SWEEP if c['D'] == D and c['kind'] == kind for P in [c['P']]} == {0, 2}
    for kind in ('llbank', 'lldict'):
        assert {c['C'] for c in SWEEP if c['kind'] == kind} == {1, 3}
    kinds = {(c['kind'], c['P']) for c in INFERENCE}
    assert {('ll', 0), ('llbank', 0), ('lldict', 0)} <= kinds and any(P == 2 for _, P in kinds)
    assert any(c['kind'] == 'lldict' and min(c['atoms']) < max(c['atoms']) for c in INFERENCE)
    Ks = {k for c in INFERENCE for k in (c['atoms'] or [c['K']])}
    assert {1, 31, 33, 100, 256} <= Ks
    assert {c['inf'] for c in INFERENCE} == {1, 2, 7} and {c['alpha'] for c in INFERENCE} == {0.0, 0.5}
    assert {tuple(sorted(c['atoms'])) for c in SWEEP if c['kind'] == 'lldict'} == {tuple(sorted(ATOMS))}
    assert len(ATOMS) > len(set(ATOMS)) and max(ATOMS) % 128 != 0 and -(-max(ATOMS) // 128) == 3
    for cases in (SWEEP, INFERENCE):
        for c in cases:
            if c['kind'] != 'll':
                counts = c['dcounts'] if c['kind'] == 'lldict' else c['scounts']
                assert 0 in counts and counts[-1] > 0 and list(counts) != sorted(counts)


def test_cases_straddle_every_tile_width():
    steer = [n for c in CASES for n in _columns(c)[0]]
    assert any(_straddles(n, ANG_TILE) for n in steer) and any(_straddles(n, PLANE_TILE) for n in steer)
    dict_cases = [c for c in CASES if c['kind'] == 'lldict']
    for D in TDOAS:
        cut = [n for c in dict_cases if c['D'] == D for n in _columns(c)[1]]
        if SIMT_GN // D > 1:                                   # a tile of one frame has no partial tile
            assert any(_straddles(n, SIMT_GN // D) for n in cut), D
        if D >= 32:
            assert any(_straddles(n, GEMM_COLUMNS // D) for n in cut), D
    assert any(_straddles(n, WIENER_RN) for c in dict_cases for n in _columns(c)[1])
    assert any(_straddles(n, SIMT_GN // c['P']) for c in dict_cases if c['P'] for n in _columns(c)[1])


def test_cases_reach_every_grouped_gemm_with_partial_frame_and_m_tiles():
    for D in (32, 64, 128):
        hit = False
        for c in CASES:
            if c['kind'] == 'lldict' and c['D'] == D and c['N'] // 2 + 1 >= 32 and not c['P']:
                for n, K in zip(_columns(c)[1], c['atoms']):
                    hit |= _straddles(n, GEMM_COLUMNS // D) and K % 128 != 0 and K > 0
        assert hit, D
