"""Host model of the offline stage kernels: csrc/stft.cu, the localisation and masking kernels of csrc/gcc.cu, the masked
reconstruction of csrc/gcc_tc.cu and the peak picking of csrc/pipeline.cu.  Test infrastructure only.

Every function takes the device's output of the stage before (teacher forcing), so an error in one stage does not spread into
the next.
  Exact (the kernel's order is fixed and float32; the model reproduces it bit for bit): the PHAT coherence, |X|, the overlap-add
    gather, the SIMT masked reconstruction, wiener_apply (with rowsum_w's reduction order), wiener_apply_h, online_targets,
    atom_mask in boxcar mode, coeff_mask (numpy.nanargmax plus the all-NaN flag), argmax_mask, tdoa_lut, gather_steering and
    the peak picking (argrelmax, then the stable order of equal peaks).
  Bounded (float64 work whose summation order or contraction the model does not follow): the STFT (float64 FFT of the
    float64-windowed frame), the iFFT frames (float64 irfft of the Hermitian rebuild), the angular spectrogram and its mean,
    the tdoa_gccnmf values (float64 sums rounded once to float32) and the tensor-core reconstruction.
The float32 fused multiply-add, the warp butterfly and the ulp distance come from oracle/rt_exact.py.
"""
import numpy as np
from scipy.signal import argrelmax

from oracle.rt_exact import fma32, butterfly, ulps32, WARP  # noqa: F401  (ulps32 re-exported for the tests)

F32, F64 = np.float32, np.float64
C64 = np.complex64
SIMT_BK = 16              # k tile of the float32 SIMT GEMM (gcc.cu RK): the chain is padded to a multiple of it
ROWSUM_THREADS = 128      # rowsum_w_kernel's block


# ------------------------------------------------------------------------------------------------ exact float64 fma
def _two_sum(a, b):
    s = a + b
    bb = s - a
    return s, (a - (s - bb)) + (b - bb)


def _two_prod(a, b):
    """p + e == a * b exactly (Veltkamp split; no overflow at the magnitudes used here)."""
    p = a * b
    sp = F64(134217729.0)                                                     # 2^27 + 1
    ca, cb = sp * a, sp * b
    ah, bh = ca - (ca - a), cb - (cb - b)
    al, bl = a - ah, b - bh
    return p, ((ah * bh - p) + ah * bl + al * bh) + al * bl


def fma64(a, b, c):
    """Correctly rounded float64 a * b + c, elementwise (CUDA's DFMA): the product split exactly, its low part added to the
    TwoSum error in round-to-odd, then one rounding to nearest (Boldo and Melquiond's emulation)."""
    a, b, c = (np.asarray(v, F64) for v in (a, b, c))
    with np.errstate(all='ignore'):
        uh, ul = _two_prod(a, b)
        th, tl = _two_sum(c, uh)
        v, e = _two_sum(tl, ul)
        bits = v.view(np.int64)
        fix = (e != 0) & ((bits & 1) == 0) & np.isfinite(v)
        step = np.where((e > 0) == (v > 0), 1, -1)
        v = np.where(fix, bits + step, bits).view(F64)
        return th + v


# ------------------------------------------------------------------------------------------------ comparisons
def nearest_or_within(device, ref64, slack):
    """True where the float32 `device` is a float32 rounding of some value within `slack` of the float64 `ref64`:
    rn(ref - slack) <= device <= rn(ref + slack).  With slack 0 this is "the nearest float32"; a slack lets either neighbour
    through only where ref lies that close to a rounding midpoint.  NaN must match NaN."""
    d = np.asarray(device, F32)
    r = np.asarray(ref64, F64)
    s = np.asarray(slack, F64)
    with np.errstate(all='ignore'):
        lo, hi = (r - s).astype(F32), (r + s).astype(F32)
        ok = (d >= lo) & (d <= hi)
    return np.where(np.isnan(r), np.isnan(d), ok)


# ------------------------------------------------------------------------------------------------ STFT (bounded) and |X| (exact)
def stft_frames(samples, window, n_fft, hop):
    """(C, T, n) float64 windowed frames w * double(x), exactly the kernel's products."""
    samples = np.asarray(samples, F32)
    C, L = samples.shape
    T = 1 + (L - n_fft) // hop
    idx = np.arange(T)[:, None] * hop + np.arange(n_fft)[None, :]
    return np.asarray(window, F64)[None, None, :] * samples[:, idx].astype(F64)


def stft(samples, window, n_fft, hop, conjugate):
    """(C, F, T) complex128 float64 STFT and the (T,) slack of each frame: 1e-12 of sum |w x| over both channels (the kernel
    transforms the two channels of a frame as one complex signal, so each channel's rounding carries the other's magnitude)."""
    x = stft_frames(samples, window, n_fft, hop)
    X = np.fft.rfft(x, axis=2).transpose(0, 2, 1)
    if conjugate:
        X = np.conj(X)
    slack = 1e-12 * np.abs(x).sum(axis=(0, 2))
    return X, slack


def magnitudes(X, channels):
    """V (F, C T) float32 = float(sqrt(double re^2 + double im^2)) of the device's X (C, F, T)."""
    r, i = np.real(X).astype(F64), np.imag(X).astype(F64)
    m = np.sqrt(r * r + i * i).astype(F32)
    C, F, T = m.shape
    return np.ascontiguousarray(m.transpose(1, 0, 2).reshape(F, C * T))


# ------------------------------------------------------------------------------------------------ iSTFT
def ifft_frames(spec, n_fft, conjugate):
    """(B, T, n) float64 inverse FFT of each (conjugated) column's Hermitian extension, the imaginary parts at DC and Nyquist
    dropped (they only feed the discarded imaginary output of the packed transform)."""
    Z = np.asarray(spec, C64).astype(np.complex128)
    if conjugate:
        Z = np.conj(Z)
    Z = Z.copy()
    Z[:, 0, :] = Z[:, 0, :].real
    Z[:, n_fft // 2, :] = Z[:, n_fft // 2, :].real
    return np.fft.irfft(Z, n=n_fft, axis=1).transpose(0, 2, 1)


def ola(frames, window, hop, center, gain, fused=True):
    """y (B, length) float32 of ola_gather_kernel from the device's frames (B, T, n) float32: every output sample adds its
    frames in ascending order, acc = float(fma(w, double(frame), double(acc))) from 0.f (the compiler contracts the float64
    product and sum into one DFMA), then acc * gain in float32.  fused=False rounds the product first, as the reference does."""
    frames = np.asarray(frames, F32)
    B, T, n = frames.shape
    w = np.asarray(window, F64)
    total = n + hop * (T - 1)
    acc = np.zeros((B, total), F32)
    for i in range(T):
        s = i * hop
        x, a = frames[:, i, :].astype(F64), acc[:, s:s + n].astype(F64)
        acc[:, s:s + n] = (fma64(w[None, :], x, a) if fused else a + w[None, :] * x).astype(F32)
    if center:
        acc = acc[:, n // 2:total - n // 2]
    return (acc * F32(gain)).astype(F32)


def istft_length(n_fft, hop, T, center):
    return n_fft + hop * (T - 1) - (n_fft if center else 0)


# ------------------------------------------------------------------------------------------------ coherence (exact), angular (bounded)
def coherence(X):
    """phat_coherence of X[0], X[1] (F, T) complex64 -> (F, T) complex64: every product rounded on its own, magnitudes
    float(sqrt(double)), two multiplications by float32 reciprocals."""
    X = np.asarray(X, C64)
    a, b = X[0], X[1]
    ax, ay, bx, by = (np.real(a).astype(F32), np.imag(a).astype(F32), np.real(b).astype(F32), np.imag(b).astype(F32))
    with np.errstate(all='ignore'):
        re = ax * bx + ay * by
        im = ay * bx - ax * by
        ma = np.sqrt(ax.astype(F64) ** 2 + ay.astype(F64) ** 2).astype(F32)
        mb = np.sqrt(bx.astype(F64) ** 2 + by.astype(F64) ** 2).astype(F32)
        ia, ib = F32(1) / ma, F32(1) / mb
        re, im = (re * ia) * ib, (im * ia) * ib
    out = np.empty(re.shape, C64)
    out.real, out.imag = re, im
    return out


def numpy_coherence(X):
    """The reference's own expression X0 conj(X1) / |X0| / |X1| in numpy's complex64 arithmetic (host dependent)."""
    X = np.asarray(X, C64)
    with np.errstate(all='ignore'):
        return X[0] * X[1].conj() / np.abs(X[0]) / np.abs(X[1])


def angular(coh, E):
    """(D, T) float64 sum_f Re(c[f, t] E[f, d]) and the (D, T) bound 4 F 2^-53 sum_f (|c.x e.x| + |c.y e.y|)."""
    c = np.asarray(coh, C64).astype(np.complex128)
    E = np.asarray(E, np.complex128)
    cx, cy, ex, ey = c.real, c.imag, E.real, E.imag
    with np.errstate(all='ignore'):
        ref = ex.T @ cx - ey.T @ cy
        mag = np.abs(ex).T @ np.abs(cx) + np.abs(ey).T @ np.abs(cy)
    F = c.shape[0]
    return ref, 4.0 * F * 2.0 ** -53 * mag


def mean_bound(ang):
    """float64 mean over frames of the device's (D, T) angular output and its bound: (T + 16) 2^-53 mean |ang| + 1 ulp."""
    ang = np.asarray(ang, F64)
    T = ang.shape[1]
    with np.errstate(all='ignore'):
        ref = ang.sum(axis=1) / T
        bound = (T + 16) * 2.0 ** -53 * np.abs(ang).sum(axis=1) / T + np.spacing(np.abs(ref))
    return ref, bound


# ------------------------------------------------------------------------------------------------ GCC-NMF (bounded / argmax)
def tdoa_values(coh, E, W):
    """(D, K, T) float64 sum_f W[f, k] Re(c[f, t] E[f, d]) and its float64 slack 4 F 2^-53 sum_f |W| (|c.x e.x| + |c.y e.y|)."""
    c = np.asarray(coh, C64).astype(np.complex128)
    E = np.asarray(E, np.complex128)
    W = np.asarray(W, F32).astype(F64)
    with np.errstate(all='ignore'):
        G = np.einsum('ft,fd->dft', c.real, E.real) - np.einsum('ft,fd->dft', c.imag, E.imag)
        A = np.einsum('ft,fd->dft', np.abs(c.real), np.abs(E.real)) + np.einsum('ft,fd->dft', np.abs(c.imag), np.abs(E.imag))
        ref = np.einsum('fk,dft->dkt', W, G)
        mag = np.einsum('fk,dft->dkt', np.abs(W), A)
    F = c.shape[0]
    return ref, 4.0 * F * 2.0 ** -53 * mag


def tdoa_argmax(values64):
    """(K, T) int32 numpy.argmax over d of (D, K, T) float64 values: NaN wins, first occurrence."""
    return np.argmax(values64, axis=0).astype(np.int32)


# ------------------------------------------------------------------------------------------------ masks (exact)
def coeff_mask(G):
    """coeff_mask_kernel: numpy.nanargmax over s of (S, K, T) (NaN counts as -inf, first maximum wins); a column that is all
    NaN gets no source and raises the flag.  Returns (masks (S, K, T) float32, flag int)."""
    G = np.asarray(G, F32)
    all_nan = np.isnan(G).all(axis=0)
    best = np.argmax(np.where(np.isnan(G), -np.inf, G), axis=0)
    s = np.arange(G.shape[0])[:, None, None]
    return ((s == best[None]) & ~all_nan[None]).astype(F32), int(all_nan.any())


def argmax_mask(argmax, lut):
    a = np.asarray(argmax, np.int64)
    lut = np.asarray(lut, bool)
    D = len(lut)
    ok = (a >= 0) & (a < D)
    return np.where(ok, lut[np.clip(a, 0, D - 1)], False).astype(F32)


def tdoa_lut(tdoas, target, window):
    tdoas = np.asarray(tdoas, F64)
    return (np.abs(tdoas - tdoas[int(target)]) < F64(window)).astype(np.uint8)


def gather_steering(E, targets):
    return np.ascontiguousarray(np.asarray(E, np.complex128)[:, np.asarray(targets, np.int64)])


# ------------------------------------------------------------------------------------------------ reconstruction
def fma_chain(A, B, K):
    """acc = fmaf(A[k], B[k], acc) for k = 0 .. K-1 from 0.f, then fmaf(0, 0, acc) up to the next multiple of the k tile
    (the SIMT GEMM's zero-filled operands); A and B have k first and broadcast over the rest."""
    acc = np.zeros(np.broadcast_shapes(A.shape[1:], B.shape[1:]), F32)
    for k in range(K):
        acc = fma32(A[k], B[k], acc)
    pad = -(-K // SIMT_BK) * SIMT_BK - K
    zero = F32(0)
    for _ in range(pad):
        acc = fma32(zero, zero, acc)
    return acc


def phasor(X):
    """exp(1j angle(x)) of the device's epilogue: float(double(x) / |x|_double); angle(0) = 0; NaN passes through."""
    X = np.asarray(X, C64)
    r, i = np.real(X).astype(F64), np.imag(X).astype(F64)
    mag = np.sqrt(r * r + i * i)
    with np.errstate(all='ignore'):
        pr = np.where(mag > 0, r / mag, np.where(np.isnan(mag), np.nan, 1.0)).astype(F32)
        pi = np.where(mag > 0, i / mag, np.where(np.isnan(mag), np.nan, 0.0)).astype(F32)
    return pr, pi


def masked_products(masks, H):
    """(S, 2, K, T) float32 H_c * M_s rounded once, as the loaders build them."""
    masks = np.asarray(masks, F32)
    S, K, T = masks.shape
    H = np.asarray(H, F32).reshape(K, 2, T).transpose(1, 0, 2)
    return (H[None] * masks[:, None]).astype(F32)


def recon_simt(masks, X, W, H):
    """masked_recon_kernel: (S, 2, F, T) complex64, acc = ascending-k fmaf chain of W[f, k] float(H M), times the phasor."""
    HM = masked_products(masks, H)                                            # (S, 2, K, T)
    W = np.asarray(W, F32)
    K = W.shape[1]
    A = W.T[:, None, None, :, None]                                           # (K, 1, 1, F, 1)
    B = HM.transpose(2, 0, 1, 3)[:, :, :, None, :]                            # (K, S, 2, 1, T)
    acc = fma_chain(A, B, K)                                                  # (S, 2, F, T)
    pr, pi = phasor(X)
    out = np.empty(acc.shape, C64)
    with np.errstate(all='ignore'):
        out.real, out.imag = acc * pr[None], acc * pi[None]
    return out


def recon_bound(masks, X, W, H):
    """Tensor-core reconstruction: float64 reference (S, 2, F, T) of sum_k W float(H M) times the device's phasor, and the
    per-part bound (8e-6 + 4e-8 3K/16) sum_k W (H M) + one float32 ulp of the reference (DESIGN section 2's plane GEMM bar)."""
    HM = masked_products(masks, H).astype(F64)
    W = np.asarray(W, F32).astype(F64)
    K = W.shape[1]
    acc = np.einsum('fk,sckt->scft', W, HM)
    mag = np.einsum('fk,sckt->scft', np.abs(W), np.abs(HM))
    pr, pi = phasor(X)
    ref = acc * pr.astype(F64)[None] + 1j * (acc * pi.astype(F64)[None])
    c = (8e-6 + 4e-8 * 3 * K / 16) * mag
    ulp = lambda v: np.spacing(np.abs(v).astype(F32)).astype(F64)   # noqa: E731
    return ref, c + ulp(ref.real), c + ulp(ref.imag)


def rowsum(W):
    """rowsum_w_kernel (F,) float32: thread j of 128 adds W[f, j], W[f, j + 128], ... from 0.f; each warp's xor butterfly;
    the 4 warp partials (lanes >= 4 zero) through a second butterfly."""
    W = np.asarray(W, F32)
    F, K = W.shape
    steps = -(-K // ROWSUM_THREADS)
    Wp = np.zeros((F, steps * ROWSUM_THREADS), F32)
    Wp[:, :K] = W
    s = np.zeros((ROWSUM_THREADS, F), F32)
    for i in range(steps):
        s = (s + Wp[:, i * ROWSUM_THREADS:(i + 1) * ROWSUM_THREADS].T).astype(F32)
    warps = [butterfly(s[w * WARP:(w + 1) * WARP]) for w in range(ROWSUM_THREADS // WARP)]
    lanes = np.zeros((WARP, F), F32)
    lanes[:len(warps)] = warps
    return butterfly(lanes).astype(F32)


def wiener_apply(mask, W, X):
    """wiener_apply_kernel: (Y (2, F, T) complex64, wiener (F, T) float32), wiener = chain(W, mask) / rowsum(W)."""
    W = np.asarray(W, F32)
    mask = np.asarray(mask, F32)
    K = W.shape[1]
    acc = fma_chain(W.T[:, :, None], mask[:, None, :], K)
    with np.errstate(all='ignore'):
        w = (acc / rowsum(W)[:, None]).astype(F32)
    return _times(w[None], X), w


def wiener_apply_h(mask, W, H, X):
    """wiener_apply_h_kernel: per channel c, wiener[c] = chain(W, float(H_c mask)) / chain(W, H_c); Y[c] = wiener[c] X[c]."""
    W = np.asarray(W, F32)
    mask = np.asarray(mask, F32)
    K, T = mask.shape
    H = np.asarray(H, F32).reshape(K, 2, T)
    w = np.empty((2, W.shape[0], T), F32)
    for c in range(2):
        hc = H[:, c, :]
        num = fma_chain(W.T[:, :, None], (hc * mask).astype(F32)[:, None, :], K)
        den = fma_chain(W.T[:, :, None], hc[:, None, :], K)
        with np.errstate(all='ignore'):
            w[c] = num / den
    return _times(w, X), w


def _times(w, X):
    X = np.asarray(X, C64)
    Y = np.empty(X.shape, C64)
    with np.errstate(all='ignore'):
        Y.real, Y.imag = w * np.real(X), w * np.imag(X)
    return Y


# ------------------------------------------------------------------------------------------------ online localisation, atom masks
def online_targets(ang):
    """cummax_time_kernel + argmax_tdoa_kernel: running max over frames in which a NaN sticks, then numpy.argmax over d."""
    acc = np.maximum.accumulate(np.asarray(ang, F64), axis=1)
    return acc, np.argmax(acc, axis=0).astype(np.int32)


def atom_mask(argmax, targets, target_scalar, epsilon, mode, beta=1.0, noise_floor=0.0):
    """atom_mask_kernel in float32: dist = |float(argmax) - float(target)|; mode 0 exact (dist < eps); mode 1 in float64 from
    the float32 dist (compare with rt_exact.atom_mask_ulp_bound float32 ulps)."""
    a = np.asarray(argmax).astype(F32)
    mu = np.asarray(targets).astype(F32)[None, :] if targets is not None else F32(target_scalar)
    dist = np.abs(a - mu).astype(F32)
    if mode == 0:
        return (dist < F32(epsilon)).astype(F32)
    nf = F32(noise_floor)
    x = (dist / F32(epsilon)).astype(F32).astype(F64)
    return np.exp(-np.power(x, F64(F32(beta)))) / F64(F32(F32(1) + nf)) + F64(nf)


# ------------------------------------------------------------------------------------------------ peak picking
def pick_targets(x, S):
    """select_peaks: argrelmax's strict interior maxima, the S largest in stable order (of equal values the higher index
    ranks higher), ascending.  Returns (targets padded with 0 to S, number of peaks)."""
    x = np.asarray(x, F64)
    with np.errstate(invalid='ignore'):
        peaks = argrelmax(x)[0]
    chosen = sorted(peaks[np.argsort(x[peaks], kind='stable')][-S:].tolist()) if S > 0 else []
    return np.array(chosen + [0] * (S - len(chosen)), np.int32), len(peaks)
