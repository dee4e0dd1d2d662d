"""Drop-in for gccNMF/gccNMFFunctions.py: same function names, argument order, array shapes and
dtypes (numpy in, numpy out), each numeric stage executed by the sm_90a kernels behind the C ABI.

Host-side pieces that stay on the host on purpose: the seeded numpy draw of the NMF initial values
(gccNMFFunctions.py:70-73 -- legacy global MT19937, bit-identical only if numpy draws it), the
float64 construction of the exp(-2 pi i f tau) table (:89,:128) and peak picking on the D-element
mean angular spectrum (:94-116, scipy.signal.argrelmax) so index semantics are the reference's by
construction.  For a device-resident end-to-end run use pipeline.GCCNMFPipeline.
"""
import logging

import numpy as np
from numpy import hanning  # noqa: F401  (re-exported like the reference's star-import surface)
from scipy.signal import argrelmax

from ._lib import GCCNMFError, ParameterError, default_handle  # noqa: F401

SPEED_OF_SOUND_IN_METRES_PER_SECOND = 340.29   # gccNMFFunctions.py:38


def getMixtureFileName(mixtureFileNamePrefix):
    return mixtureFileNamePrefix + '_mix.wav'


def getSourceEstimateFileName(mixtureFileNamePrefix, targetIndex):
    return mixtureFileNamePrefix + '_sim_%d.wav' % (targetIndex + 1)


def loadMixtureSignal(mixtureFileName):
    """gccNMFFunctions.py:47 -> wavfile.py:34-37: (channels, n) float32 in [-1, 1), sample rate."""
    from .wavio import wavread
    samples, sampleRate = wavread(mixtureFileName)
    return np.ascontiguousarray(samples, dtype=np.float32), sampleRate


def getMaxTDOA(microphoneSeparationInMetres):
    return microphoneSeparationInMetres / SPEED_OF_SOUND_IN_METRES_PER_SECOND


def getTDOAsInSeconds(microphoneSeparationInMetres, numTDOAs):
    maxTDOA = getMaxTDOA(microphoneSeparationInMetres)
    return np.linspace(-maxTDOA, maxTDOA, numTDOAs)


def getFrequenciesInHz(sampleRate, numFrequencies):
    return np.linspace(0, sampleRate / 2, numFrequencies)


def getExpJOmegaTau(frequenciesInHz, tdoasInSeconds):
    """(F, D) complex128 steering table, float64 on the host exactly as gccNMFFunctions.py:89."""
    return np.exp(np.outer(frequenciesInHz, -(2j * np.pi) * tdoasInSeconds))


# ----------------------------------------------------------------------------------------- a1
def computeComplexMixtureSpectrogram(stereoSamples, windowSize, hopSize, windowFunction, fftSize=None):
    """gccNMFFunctions.py:61-67 -> (2, F, T) complex64.  Like the reference the window actually
    applied is numpy.hanning (the windowFunction argument is ignored there, :65)."""
    if fftSize is None:
        fftSize = windowSize
    if fftSize != windowSize:
        raise ParameterError('fftSize != windowSize is not supported')
    stereoSamples = np.asarray(stereoSamples)
    if not np.isfinite(stereoSamples).all():
        raise ParameterError('Audio buffer is not finite everywhere')
    h = default_handle()
    samples = h.to_device(np.ascontiguousarray(stereoSamples[:2], dtype=np.float32))
    X = h.stft(samples, h.to_device(np.hanning(windowSize)), windowSize, hopSize, conjugate=True)
    return X.cpu().numpy()


# ----------------------------------------------------------------------------------------- a2
def _seededInit(numFrequencies, numColumns, dictionarySize, epsilon, seedValue):
    np.random.seed(seedValue)                                                         # :70
    W = np.random.random((numFrequencies, dictionarySize)).astype(np.float32) + epsilon   # :72
    H = np.random.random((dictionarySize, numColumns)).astype(np.float32) + epsilon       # :73
    return W.astype(np.float32), H.astype(np.float32)


def performKLNMF(V, dictionarySize, numIterations, sparsityAlpha, epsilon=1e-16, seedValue=0):
    """gccNMFFunctions.py:69-83 -> W (F, K) f32, H (K, T2) f32.  float64 V (the pre-training call,
    realtime/gccNMFPretraining.py:80) is converted to float32: the reference's float64 intermediates
    there differ from this float32 path only at float32 rounding level."""
    V = np.asarray(V)
    W0, H0 = _seededInit(V.shape[0], V.shape[1], dictionarySize, epsilon, seedValue)
    h = default_handle()
    W, H = h.to_device(W0), h.to_device(H0)
    h.klnmf(h.to_device(np.ascontiguousarray(V, dtype=np.float32)), W, H, numIterations, sparsityAlpha, epsilon, update_W=True)
    return W.cpu().numpy(), H.cpu().numpy()


def performKLNMFBatch(Vs, dictionarySize, numIterations, sparsityAlpha, epsilon=1e-16, seedValue=0):
    """performKLNMF on B clips in one batched call, clip b equal to performKLNMF(Vs[b], ...).  Vs (B, F, T2) -> W (B, F, K),
    H (B, K, T2); a list of (F, T2_b) arrays of any lengths -> W (B, F, K), [H_b (K, T2_b)].  The reference re-seeds on every call,
    so every clip starts from the same draw: drawn once here.  W0 does not depend on T2 and H0 for T2 frames is the first K T2
    values drawn after W0, so one draw at the longest clip serves every clip of a list."""
    if isinstance(Vs, (list, tuple)):
        Vs = [np.asarray(V) for V in Vs]
        if not Vs or any(V.ndim != 2 or V.shape[0] != Vs[0].shape[0] for V in Vs):
            raise ParameterError('performKLNMFBatch: Vs must be a non-empty list of (F, T2_b) arrays of one F')
        F, K = Vs[0].shape[0], dictionarySize
        W0, Hmax = _seededInit(F, max(V.shape[1] for V in Vs), K, epsilon, seedValue)
        h = default_handle()
        W = h.to_device(np.ascontiguousarray(np.broadcast_to(W0, (len(Vs),) + W0.shape)))
        Hs = [h.to_device(np.ascontiguousarray(Hmax.reshape(-1)[:K * V.shape[1]].reshape(K, V.shape[1]))) for V in Vs]
        h.klnmf_ragged([h.to_device(np.ascontiguousarray(V, dtype=np.float32)) for V in Vs], W, Hs, numIterations, sparsityAlpha, epsilon,
                       update_W=True)
        return W.cpu().numpy(), [H.cpu().numpy() for H in Hs]
    Vs = np.asarray(Vs)
    if Vs.ndim != 3:
        raise ParameterError('performKLNMFBatch: Vs must be (B, F, T2), got shape %s' % (Vs.shape,))
    B, F, T2 = Vs.shape
    W0, H0 = _seededInit(F, T2, dictionarySize, epsilon, seedValue)
    h = default_handle()
    W = h.to_device(np.ascontiguousarray(np.broadcast_to(W0, (B,) + W0.shape)))
    H = h.to_device(np.ascontiguousarray(np.broadcast_to(H0, (B,) + H0.shape)))
    h.klnmf_batched(h.to_device(np.ascontiguousarray(Vs, dtype=np.float32)), W, H, numIterations, sparsityAlpha, epsilon, update_W=True)
    return W.cpu().numpy(), H.cpu().numpy()


def inferCoefficientsKLNMF(V, W, numIterations, sparsityAlpha, epsilon=1e-16, seedValue=0):
    """The function the notebooks call but the reference never defines
    (onlineSpeechEnhancement.ipynb:433): H-only KL updates (:76) with a fixed dictionary from the
    seeded H init of :70,:73.  V (F, T2) -> H (K, T2)."""
    V = np.asarray(V)
    np.random.seed(seedValue)
    H0 = (np.random.random((W.shape[1], V.shape[1])).astype(np.float32) + epsilon).astype(np.float32)
    h = default_handle()
    Wd, H = h.to_device(np.ascontiguousarray(W, dtype=np.float32)), h.to_device(H0)
    h.klnmf(h.to_device(np.ascontiguousarray(V, dtype=np.float32)), Wd, H, numIterations, sparsityAlpha, epsilon, update_W=False)
    return H.cpu().numpy()


# ----------------------------------------------------------------------------------------- a3, a4, a5
def getSpectralCoherence(complexMixtureSpectrogram):
    """The inline expression of runGCCNMF.py:44 -> (F, T) complex64."""
    h = default_handle()
    coh, _, _ = h.phat_angspec(h.to_device(np.ascontiguousarray(complexMixtureSpectrogram, dtype=np.complex64)),
                               None, want_coherence=True, want_angular=False, want_mean=False)
    return coh.cpu().numpy()


def getAngularSpectrogram(spectralCoherenceV, frequenciesInHz, microphoneSeparationInMetres, numTDOAs):
    """gccNMFFunctions.py:85-92 -> (D, T) float64 = sum_f Re(C[f,t] E[f,tau]), float64 accumulation."""
    C = np.ascontiguousarray(spectralCoherenceV, dtype=np.complex64)
    E = getExpJOmegaTau(frequenciesInHz, getTDOAsInSeconds(microphoneSeparationInMetres, numTDOAs))
    h = default_handle()
    _, ang, _ = h.phat_angspec(h.to_device(C), h.to_device(np.ascontiguousarray(E)), want_coherence=False,
                               want_angular=True, want_mean=False)
    return ang.cpu().numpy()


def estimateTargetTDOAIndexesFromAngularSpectrum(angularSpectrum, microphoneSeparationInMetres, numTDOAs, numSources):
    """gccNMFFunctions.py:94-116 (host: D floats).  The reference's numSources=None branch uses
    un-imported names and cannot run; too few peaks raises ValueError (the reference logs and
    calls os._exit through an un-imported `os`)."""
    angularSpectrum = np.asarray(angularSpectrum)
    peakIndexes = argrelmax(angularSpectrum)[0]
    if not numSources:
        raise NotImplementedError('numSources=None: this branch cannot run in the reference either (:105-110)')
    logging.info('numSources provided, taking first %d peaks' % numSources)
    sourcePeakIndexes = peakIndexes[np.argsort(angularSpectrum[peakIndexes])[-numSources:]]
    if len(sourcePeakIndexes) != numSources:
        raise ValueError('did not find enough peaks in the angular spectrum')
    sourcePeakIndexes = sorted(sourcePeakIndexes)
    logging.info('Found target TDOAs: %s' % str(sourcePeakIndexes))
    return sourcePeakIndexes


# ----------------------------------------------------------------------------------------- a6, a7, a8, a9
def getTargetTDOAGCCNMFs(coherenceV, microphoneSeparationInMetres, numTDOAs, frequenciesInHz, targetTDOAIndexes, W, stereoH):
    """gccNMFFunctions.py:118-135 -> (S, K, T) float32."""
    hypothesisTDOAs = getTDOAsInSeconds(microphoneSeparationInMetres, numTDOAs)
    E = getExpJOmegaTau(frequenciesInHz, hypothesisTDOAs)[:, list(targetTDOAIndexes)]
    h = default_handle()
    values, _ = h.tdoa_gccnmf(h.to_device(np.ascontiguousarray(coherenceV, dtype=np.complex64)),
                              h.to_device(np.ascontiguousarray(E)), h.to_device(np.ascontiguousarray(W, dtype=np.float32)),
                              want_values=True, want_argmax=False)
    return values.cpu().numpy()


def getTargetCoefficientMasks(targetTDOAGCCNMFs, numTargets):
    """gccNMFFunctions.py:137-143 -> one-hot (S, K, T) float32; all-NaN slices raise like nanargmax."""
    h = default_handle()
    masks, flag = h.coeff_mask(h.to_device(np.ascontiguousarray(targetTDOAGCCNMFs[:numTargets], dtype=np.float32)))
    if int(flag.item()):
        raise ValueError('All-NaN slice encountered')
    return masks.cpu().numpy()


def getTargetSpectrogramEstimates(targetCoefficientMasks, complexMixtureSpectrogram, W, stereoH):
    """gccNMFFunctions.py:145-151 -> (S, 2, F, T) complex64."""
    h = default_handle()
    stereoH = np.asarray(stereoH)
    H = np.ascontiguousarray(np.concatenate(list(stereoH), axis=-1), dtype=np.float32)   # inverse of hsplit (runGCCNMF.py:42)
    out = h.masked_recon_phase(h.to_device(np.ascontiguousarray(targetCoefficientMasks, dtype=np.float32)),
                               h.to_device(np.ascontiguousarray(complexMixtureSpectrogram, dtype=np.complex64)),
                               h.to_device(np.ascontiguousarray(W, dtype=np.float32)), h.to_device(H))
    return out.cpu().numpy()


def getTargetSignalEstimates(targetSpectrogramEstimates, windowSize, hopSize, windowFunction):
    """gccNMFFunctions.py:153-163 -> (S, 2, hop (T - 1)) float32, gain 2 hop / N."""
    S, C, F, T = targetSpectrogramEstimates.shape
    gain = hopSize / float(windowSize) * 2
    h = default_handle()
    spec = h.to_device(np.ascontiguousarray(targetSpectrogramEstimates, dtype=np.complex64).reshape(S * C, F, T))
    window = windowFunction(windowSize) if callable(windowFunction) else np.asarray(windowFunction)
    y = h.istft_ola(spec, h.to_device(np.ascontiguousarray(window, dtype=np.float64)), windowSize, hopSize,
                    gain=np.float32(gain), center=True, conjugate=True)
    return y.cpu().numpy().reshape(S, C, -1)


def saveTargetSignalEstimates(targetSignalEstimates, sampleRate, mixtureFileNamePrefix):
    """gccNMFFunctions.py:165-169 -> wavfile.py:39-48 (int16 = x * 2^15 clipped; a peak >= 1 is rescaled to 0.99)."""
    from .wavio import wavwrite
    for targetIndex in range(targetSignalEstimates.shape[0]):
        wavwrite(np.asarray(targetSignalEstimates[targetIndex]), getSourceEstimateFileName(mixtureFileNamePrefix, targetIndex), sampleRate)


# ----------------------------------------------------------------------------------------- a10 (notebook)
def getGCCNMFArgMaxTDOA(spectralCoherenceV, frequenciesInHz, microphoneSeparationInMetres, numTDOAs, W):
    """argmax over all hypothesis TDOAs of the per-atom GCC-NMF (offlineSpeechEnhancement.ipynb
    cells 27+29, :444-467) -> (K, T) int32, without materialising the (K, D, T) float64 tensor."""
    E = getExpJOmegaTau(frequenciesInHz, getTDOAsInSeconds(microphoneSeparationInMetres, numTDOAs))
    h = default_handle()
    coh = h.to_device(np.ascontiguousarray(spectralCoherenceV, dtype=np.complex64))
    Ed, Wd = h.to_device(np.ascontiguousarray(E)), h.to_device(np.ascontiguousarray(W, dtype=np.float32))
    argmax, refined = h.tdoa_argmax(coh, Ed, Wd)
    if int(refined.item()) > h.lib.gccnmf_tdoa_argmax_refine_capacity(Wd.shape[1], coh.shape[1]):
        _, argmax = h.tdoa_gccnmf(coh, Ed, Wd, want_values=False, want_argmax=True)
    return argmax.cpu().numpy()


def getTargetTDOALookup(hypothesisTDOAs, targetTDOAIndex, targetTDOAWindowSize):
    """(D) bool: |tdoa[d] - tdoa[target]| < window, float64 on the host (ipynb:468-471)."""
    return np.abs(hypothesisTDOAs - hypothesisTDOAs[targetTDOAIndex]) < targetTDOAWindowSize
