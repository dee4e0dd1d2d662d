"""Online / low-latency speech enhancement (SURVEY.md section 8 row a11): the frame loops of
notebooks/onlineSpeechEnhancement.ipynb cell 23 (:406-447) and lowLatencySpeechEnhancement.ipynb cell 30
(:511-584), plus the asymmetric windows of cell 21 (:371-392).

The notebooks' loop is sequential only through one piece of state -- the accumulated maximum of the GCC-PHAT
angular spectrum (:416), a prefix maximum over time -- so here ALL frames are processed in one batch:
STFT (numpy.fft.rfft convention: not conjugated) -> PHAT coherence + angular spectrogram -> prefix max +
argmax (target TDOA per frame) -> all-TDOA GCC-NMF argmax per atom -> 0/1 atom mask -> Wiener-like filter ->
inverse FFT -> overlap-add of the raw frames (the notebooks never apply the synthesis window, :575-578).

Precision: the notebook keeps complex128 spectra (numpy.fft.rfft of float64); this path stores complex64 like
the offline path and the reference's real-time class (gccNMFProcessor.py:202), so float outputs agree to
float32 rounding and integer decisions (targets, atom masks) can differ only on float32-level near-ties.
"""
import numpy as np

from . import gccNMFFunctions as fn
from ._lib import default_handle


def getAsymmetricAnalysisWindow(k, m, d):
    """lowLatencySpeechEnhancement.ipynb cell 21 (:371-380)."""
    rising = np.sqrt(np.hanning(2 * (k - m - d) + 1)[:2 * (k - m - d)])
    falling = np.sqrt(np.hanning(2 * m + 1)[:2 * m])
    window = np.zeros(k)
    window[d:k - m] = rising[:k - m - d]
    window[k - m:] = falling[-m:]
    return window


def getAsymmetricSynthesisWindow(k, m, d):
    """lowLatencySpeechEnhancement.ipynb cell 21 (:382-392) (constructed by the notebook, never applied)."""
    risingAnalysis = np.sqrt(np.hanning(2 * (k - m - d) + 1)[:2 * (k - m - d)])
    risingNormalized = np.hanning(2 * m + 1)[:m] / risingAnalysis[k - 2 * m - d:k - m - d]
    falling = np.sqrt(np.hanning(2 * m + 1)[:2 * m])
    window = np.zeros(k)
    window[-2 * m:-m] = risingNormalized
    window[-m:] = falling[-m:]
    return window


def performOnlineSpeechEnhancement(stereoSamples, sampleRate, W, analysisWindow, synthesisWindow, hopSize, numTDOAs,
                                   microphoneSeparationInMetres, targetTDOAEpsilon, numInferenceIterations=0,
                                   gainPerFrame=False, device=0, sparsityAlpha=0, epsilon=1e-16, seedValue=0,
                                   _forcedTargetTDOAs=None, _forcedAtomMasks=None, applySynthesisWindow=False):
    """Returns the notebook's tuple (lowLatencySpeechEnhancement.ipynb:583-584):
    inputSpectrogram, outputSpectrogram, targetEstimateSamplesOLA, gccPHATAccumulatedMax, targetTDOAs,
    angularSpectrogram, atomMasks, wienerFilters.

    gainPerFrame=True is the online notebook (:376, :447: frames counted with the analysis window, gain applied per
    frame); False is the low-latency notebook (:513, :580: frames counted with len(synthesisWindow), gain at the end).

    numInferenceIterations > 0 is the branch of :433-438: per frame, H-only KL updates of the (K, 2) coefficients of the two
    channels from the seeded initial values (`inferCoefficientsKLNMF`, called by the notebooks and defined nowhere in the
    reference: gccNMFFunctions.inferCoefficientsKLNMF restates it from gccNMFFunctions.py:73,76), then
    wiener = (W . (H * mask)) / (W . H).  Every frame starts from the same seeded H0 (the call re-seeds), and H-only updates
    are independent per column, so all frames run as ONE (F, 2T) problem on the KL-NMF kernels.

    applySynthesisWindow=True weights every frame by synthesisWindow in the overlap-add (the gain stays at the end) instead of the
    notebooks' unweighted frames: with the asymmetric synthesis window a frame then touches only its last 2m samples, which is the
    low latency the windows were designed for (lowlatency.py streams it with 2m - hop - 1 samples of latency).

    _forcedTargetTDOAs / _forcedAtomMasks (tests): teacher-force the integer decisions of the loop.
    """
    stereoSamples = np.ascontiguousarray(stereoSamples, dtype=np.float32)
    analysisWindow = np.ascontiguousarray(analysisWindow, dtype=np.float64)
    N = len(analysisWindow)
    numSamples = stereoSamples.shape[1]
    W = np.ascontiguousarray(W, dtype=np.float32)
    F, K = W.shape
    synthLen = len(synthesisWindow)
    numFrames = (numSamples - (N if gainPerFrame else synthLen)) // hopSize
    numFrames = min(numFrames, 1 + (numSamples - N) // hopSize)
    gainFactor = hopSize / float(synthLen) * 2
    h = default_handle(device)
    used = (numFrames - 1) * hopSize + N
    x = h.to_device(stereoSamples[:, :used])
    infer = numInferenceIterations > 0
    stft_out = h.stft(x, h.to_device(analysisWindow), N, hopSize, conjugate=False, want_V=infer)   # :410 rfft(frame * window)
    X, V = stft_out if infer else (stft_out, None)
    frequenciesInHz = fn.getFrequenciesInHz(sampleRate, F)
    E = h.to_device(np.ascontiguousarray(fn.getExpJOmegaTau(frequenciesInHz, fn.getTDOAsInSeconds(microphoneSeparationInMetres, numTDOAs))))
    coh, ang, _ = h.phat_angspec(X, E, want_mean=False)                                           # :414-415
    accMax, targets = h.online_targets(ang)                                                       # :416-417
    if _forcedTargetTDOAs is not None:
        targets = h.to_device(np.ascontiguousarray(_forcedTargetTDOAs, dtype=np.int32))
    Wd = h.to_device(W)
    if _forcedAtomMasks is not None:
        atomMasks = h.to_device(np.ascontiguousarray(_forcedAtomMasks, dtype=np.float32))
    else:
        argmax, refined = h.tdoa_argmax(coh, E, Wd)                                               # :422-423
        if int(refined.item()) > h.lib.gccnmf_tdoa_argmax_refine_capacity(K, numFrames):
            _, argmax = h.tdoa_gccnmf(coh, E, Wd, want_values=False, want_argmax=True)
        atomMasks = h.atom_mask(argmax, targets=targets, epsilon=targetTDOAEpsilon, mode=0)      # :424-425
    if infer:
        np.random.seed(seedValue)                                                                 # gccNMFFunctions.py:70,73 with shape (K, 2)
        H0 = (np.random.random((K, 2)).astype(np.float32) + epsilon).astype(np.float32)
        H = h.to_device(np.ascontiguousarray(np.repeat(H0, numFrames, axis=1)))                   # (K, 2T): channel c in columns [cT, (c+1)T)
        h.klnmf(V, Wd, H, numInferenceIterations, sparsityAlpha, epsilon, update_W=False)         # :433 for every frame at once
        Y, wiener = h.wiener_apply_h(atomMasks, Wd, H, X, want_filter=True)                       # :434-440
        wf = wiener.cpu().numpy().astype(np.float64)
    else:
        Y, wiener = h.wiener_apply(atomMasks, Wd, X, want_filter=True)                            # :429-431, :440
        wf = wiener.cpu().numpy().astype(np.float64)
        wf = np.stack([wf, wf])
    if applySynthesisWindow:
        weights = np.ascontiguousarray(synthesisWindow, dtype=np.float64)
    else:
        weights = np.full(N, gainFactor if gainPerFrame else 1.0)
    y = h.istft_ola(Y, h.to_device(weights), N, hopSize, gain=np.float32(1.0 if gainPerFrame and not applySynthesisWindow else gainFactor),
                    center=False, conjugate=False)                                                # :443-447 / :575-580
    out = np.zeros_like(stereoSamples)
    out[:, :y.shape[1]] = y.cpu().numpy()
    return (X.cpu().numpy(), Y.cpu().numpy(), out, accMax[:, -1].cpu().numpy(), targets.cpu().numpy().astype(np.float64),
            ang.cpu().numpy(), atomMasks.cpu().numpy().astype(np.float64), wf)
