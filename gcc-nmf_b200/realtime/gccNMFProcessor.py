"""Drop-in for the per-chunk processor of gccNMF/realtime/gccNMFProcessor.py:167-276 (SURVEY.md row a13).

Same constructor arguments, attributes and methods (`processFrames`, `reset`, `setTargetTDOARange`, settable `numTDOAs`,
`separationEnabled`, `localizationEnabled`, `localizationWindowSize`, `targetMode`).  The Theano graph (:238-270) and the
numpy code around it (:201-231) run as ONE stream-ordered sequence of sm_90a kernels without a host synchronisation inside
(csrc/rt.cu, `RealtimeEngine`): windowed FFT -> PHAT coherence -> real GCC -> float32 GCC-NMF `dot(realGCC.T, W)` -> argmax
over TDOA per atom -> boxcar / window atom mask (float64, like the int64 - float32 promotion of the reference's graph) ->
(W . mask) / rowsum(W) -> inverse FFT x synthesis window, plus the GCC-PHAT history ring and the sliding-window
localisation, whose target TDOA index stays on the device from one call to the next.  Per call the host does one H2D of
the windowed frames, one D2H of the result and one synchronisation.

`numHUpdates` is accepted and, exactly as in the reference, unused (it is plumbed everywhere there and never read);
`coefficientInferenceIterations` (an extension, default 0) switches on the per-frame H-only KL updates of
notebooks/onlineSpeechEnhancement.ipynb:433-438 in the same kernel sequence.  History buffers (the reference's
SharedMemoryCircularBuffer objects) are optional duck-typed objects with `.set(values)` / `.getUnraveledArray()`.

`targetMode = TARGET_MODE_MULTIPLE` with `numSources` = P >= 2 (set before `reset`) separates the input into P sources, one per
target TDOA index: the multi-target rule of gccNMFFunctions.py:118-143 per block (csrc/rt.cu, `MultiStreamRealtimeEngine` with
numSources).  `processFrames` / `processBlock` then return (P, 2, N, nT) / (P, 2, B); `setTargetTDOAIndexes(indexes)` (the
method the reference calls at gccNMFProcessor.py:111 but never defines) sets the targets, and with localisation on the device
replaces them block by block with the P largest peaks of the windowed GCC-PHAT mean.  `targetTDOAIndexes` mirrors the device's
targets after every call.
"""
import logging

import numpy as np

from .. import gccNMFFunctions as fn
from . import engine as rt
from . import multistream as rtm

TARGET_MODE_BOXCAR = 0               # gccNMFProcessor.py:35-37
TARGET_MODE_MULTIPLE = 1             # declared by the reference, not implemented there (its graph has no such branch, :262-265)
TARGET_MODE_WINDOW_FUNCTION = 2


def steeringVectors(frequenciesInHz, microphoneSeparationInMetres, numTDOAs):
    """(maxTDOA, hypothesisTDOAs (D,) float32, expJOmegaTau (F, D) complex64) of a microphone spacing (:241-248)."""
    maxTDOA = microphoneSeparationInMetres / fn.SPEED_OF_SOUND_IN_METRES_PER_SECOND
    hypothesisTDOAs = np.linspace(-maxTDOA, maxTDOA, numTDOAs).astype(np.float32)
    return maxTDOA, hypothesisTDOAs, np.exp(np.outer(frequenciesInHz, -(2j * np.pi) * hypothesisTDOAs)).astype(np.complex64)


class GCCNMFProcessor(object):
    def __init__(self, sampleRate, windowSize, numTimePerChunk, dictionariesW, dictionaryType, dictionarySize, numHUpdates,
                 microphoneSeparationInMetres, localizationEnabled, localizationWindowSize, gccPHATHistory=None, tdoaHistory=None,
                 inputSpectrogramHistory=None, outputSpectrogramHistory=None, coefficientMaskHistories=None, device=0,
                 coefficientInferenceIterations=0):
        self.sampleRate = sampleRate
        self.windowSize = windowSize
        self.numTimePerChunk = numTimePerChunk
        self.dictionariesW = dictionariesW
        self.dictionaryType = dictionaryType
        self.dictionarySize = dictionarySize
        self.numHUpdates = numHUpdates
        self.microphoneSeparationInMetres = microphoneSeparationInMetres
        self.gccPHATHistory = gccPHATHistory
        self.tdoaHistory = tdoaHistory
        self.inputSpectrogramHistory = inputSpectrogramHistory
        self.outputSpectrogramHistory = outputSpectrogramHistory
        self.coefficientMaskHistories = coefficientMaskHistories
        self.windowFunction = np.sqrt(np.hamming(self.windowSize).astype(np.float32))[:, np.newaxis]    # :186
        self.synthesisWindowFunction = self.windowFunction
        self.numTDOAs = None
        self.separationEnabled = True
        self.localizationEnabled = localizationEnabled
        self.localizationWindowSize = localizationWindowSize
        self.targetMode = TARGET_MODE_WINDOW_FUNCTION
        self.targetTDOAIndex = np.float32(10.0)      # :196-199 (Theano shared scalars in the reference)
        self.targetTDOAEpsilon = np.float32(2.0)
        self.targetTDOABeta = np.float32(1.0)
        self.targetTDOANoiseFloor = np.float32(0.0)
        self.numSources = None               # TARGET_MODE_MULTIPLE: sources per input (:131 lists it among the reset parameters)
        self.targetTDOAIndexes = None        # TARGET_MODE_MULTIPLE: the device's targets after the last call
        self._targets_pending = None
        self.coefficientInferenceIterations = coefficientInferenceIterations
        self.device = device
        self.engine = None
        self._sent = None
        self._target_dirty = True

    # ------------------------------------------------------------------ :233-270
    def reset(self):
        logging.info('GCCNMFProcessor: resetting...')
        self.buildFunctions()
        logging.info('GCCNMFProcessor: done reset.')

    def buildFunctions(self, hopSize=None, blockSize=None):
        """Device constants that the reference bakes into its Theano functions (:241-248) and the device-resident state.
        hopSize / blockSize only matter for the ring entry (`processBlock`); `processFrames` gets its frames cut by the caller."""
        self.buildConstants()
        historyLength = self.gccPHATHistory.size() if self.gccPHATHistory else 128
        if self.engine is not None:
            self.engine.close()
        self._geometry = (int(hopSize or self.windowSize), int(blockSize or self.windowSize * self.numTimePerChunk))
        if self.targetMode not in (TARGET_MODE_BOXCAR, TARGET_MODE_MULTIPLE, TARGET_MODE_WINDOW_FUNCTION):
            raise ValueError('targetMode %r: expected TARGET_MODE_BOXCAR, TARGET_MODE_MULTIPLE or TARGET_MODE_WINDOW_FUNCTION' % (self.targetMode,))
        if self.targetMode == TARGET_MODE_MULTIPLE:
            if self.numSources is None or not 2 <= int(self.numSources) <= rtm.MAX_SOURCES:
                raise ValueError('TARGET_MODE_MULTIPLE needs numSources in [2, %d] (got %r)' % (rtm.MAX_SOURCES, self.numSources))
            self.engine = rtm.MultiStreamRealtimeEngine(self.W, self.expJOmegaTau, self.windowFunction[:, 0], self.synthesisWindowFunction[:, 0],
                                                        self._geometry[0], self._geometry[1], self.numTimePerChunk, 1,
                                                        historyLength=historyLength, numInferenceIterations=self.coefficientInferenceIterations,
                                                        device=self.device, numSources=int(self.numSources))
            if self.targetTDOAIndexes is not None and self._targets_pending is None:
                self._targets_pending = self.targetTDOAIndexes
            self.targetTDOAIndexes = self.engine.export(0, rtm.EXPORT_TARGETS)
        else:
            self.engine = rt.RealtimeEngine(self.W, self.expJOmegaTau, self.windowFunction[:, 0], self.synthesisWindowFunction[:, 0],
                                            hopSize=self._geometry[0], blockSize=self._geometry[1], windowsPerBlock=self.numTimePerChunk,
                                            historyLength=historyLength, numInferenceIterations=self.coefficientInferenceIterations,
                                            device=self.device)
        self._builtTargetMode = self.targetMode        # the reference bakes the mode into the graph at build time (:262-265)
        self._sent = None
        self._target_dirty = True

    buildTheanoFunctions = buildFunctions      # the reference's name (:238)

    def buildConstants(self):
        """The dictionary and the steering vectors expJOmegaTau (:241-248), host-side, without building an engine."""
        self.W = np.ascontiguousarray(self.dictionariesW[self.dictionaryType][self.dictionarySize], dtype=np.float32)
        self.numFrequencies, self.numAtom = self.W.shape
        self.frequenciesInHz = np.linspace(0, self.sampleRate / 2, self.numFrequencies).astype(np.float32)
        self.maxTDOA, self.hypothesisTDOAs, self.expJOmegaTau = steeringVectors(self.frequenciesInHz, self.microphoneSeparationInMetres,
                                                                                self.numTDOAs)

    def slotParams(self):
        """The parameters `processBlock` would send to its engine, as keyword arguments of MultiStreamRealtimeEngine.set_params."""
        localize = bool(self.tdoaHistory) and bool(self.gccPHATHistory) and bool(self.localizationEnabled)     # :216-222
        return dict(targetTDOAIndex=float(self.targetTDOAIndex), epsilon=float(self.targetTDOAEpsilon), beta=float(self.targetTDOABeta),
                    noiseFloor=float(self.targetTDOANoiseFloor), mode=0 if self.targetMode == TARGET_MODE_BOXCAR else 1,
                    separationEnabled=bool(self.separationEnabled), localizationEnabled=localize,
                    localizationWindowSize=int(self.localizationWindowSize))

    def setTargetTDOARange(self, targetTDOAIndex, targetTDOAEpsilon, targetTDOABeta, targetTDOANoiseFloor):
        """:272-276."""
        self.targetTDOAIndex = np.float32(targetTDOAIndex)
        self.targetTDOAEpsilon = np.float32(targetTDOAEpsilon)
        self.targetTDOABeta = np.float32(targetTDOABeta)
        self.targetTDOANoiseFloor = np.float32(targetTDOANoiseFloor)
        self._target_dirty = True

    def setTargetTDOAIndexes(self, targetTDOAIndexes):
        """TARGET_MODE_MULTIPLE: the numSources target TDOA indexes (integers in [0, numTDOAs)) of the next call; -1 keeps one.
        With localisation on, the device replaces them after every block."""
        idx = np.asarray(targetTDOAIndexes)
        if self.numSources is None or idx.shape != (int(self.numSources),):
            raise ValueError('expected %r target TDOA indexes, got %r' % (self.numSources, idx.shape))
        self._targets_pending = [int(i) for i in idx]

    def _sync_params(self):
        """Pushes the Python-side attributes to the device when they changed (stream-ordered, no synchronisation)."""
        localize = bool(self.tdoaHistory) and bool(self.gccPHATHistory) and bool(self.localizationEnabled)     # :216-222
        now = (float(self.targetTDOAEpsilon), float(self.targetTDOABeta), float(self.targetTDOANoiseFloor), int(self._builtTargetMode),
               bool(self.separationEnabled), localize, int(self.localizationWindowSize))
        if self._builtTargetMode == TARGET_MODE_MULTIPLE:
            if now != self._sent:
                self.engine.set_params(0, None, now[0], now[1], now[2], 1, now[4], now[5], now[6])
                self._sent = now
            if self._targets_pending is not None:
                self.engine.set_targets(0, [self._targets_pending])
                self._targets_pending = None
            return
        if self._target_dirty or now != self._sent:
            self.engine.set_params(float(self.targetTDOAIndex) if self._target_dirty else None, now[0], now[1], now[2],
                                   0 if now[3] == TARGET_MODE_BOXCAR else 1, now[4], now[5], now[6])
            self._sent = now
            self._target_dirty = False

    def _mirror_histories(self):
        """Optional host-side mirrors for a GUI; the numbers are the device state of the call that just finished."""
        e = self.engine
        if self._builtTargetMode == TARGET_MODE_MULTIPLE:       # per-source masks and spectra: MultiStreamRealtimeEngine.export
            self.targetTDOAIndexes = e.export(0, rtm.EXPORT_TARGETS)
            if self.inputSpectrogramHistory:
                self.inputSpectrogramHistory.set(-np.mean(np.abs(e.export(0, rt.EXPORT_INPUT_SPEC)), axis=0) ** (1 / 3.0))
            if self.gccPHATHistory:
                self.gccPHATHistory.set(e.export(0, rt.EXPORT_GCCPHAT))
            return
        if self.separationEnabled and self.coefficientMaskHistories:
            self.coefficientMaskHistories[self.dictionarySize].set(1 - e.export(rt.EXPORT_ATOM_MASK))
        if self.inputSpectrogramHistory:
            self.inputSpectrogramHistory.set(-np.mean(np.abs(e.export(rt.EXPORT_INPUT_SPEC)), axis=0) ** (1 / 3.0))
        if self.gccPHATHistory:
            self.gccPHATHistory.set(e.export(rt.EXPORT_GCCPHAT))
        if self.tdoaHistory:
            self.targetTDOAIndex = np.float32(e.export(rt.EXPORT_TARGET)[0])      # the device took the localisation decision (:221-225)
            self.tdoaHistory.set(np.array([[self.targetTDOAIndex]]))
        if self.outputSpectrogramHistory:
            with np.errstate(all='ignore'):
                self.outputSpectrogramHistory.set(-np.nanmean(np.abs(e.export(rt.EXPORT_OUTPUT_SPEC)), axis=0) ** (1 / 3.0))

    # ------------------------------------------------------------------ :201-231
    def processFrames(self, windowedSamples, forcedAtomMask=None):
        """windowedSamples (2, N, nT) float32 -> (2, N, nT) float32, or (numSources, 2, N, nT) in TARGET_MODE_MULTIPLE.
        forcedAtomMask (K, nT): use this atom mask instead of the one derived from the TDOA argmax (teacher-forced parity tests;
        not in TARGET_MODE_MULTIPLE)."""
        if self.engine is None:
            self.buildFunctions()
        self._sync_params()
        x = np.asarray(windowedSamples, dtype=np.float32)
        if self._builtTargetMode == TARGET_MODE_MULTIPLE:
            out = self.engine.process_frames(x[None], forcedAtomMask)[0].copy()
        else:
            out = self.engine.process_frames(x, forcedAtomMask).copy()
        self._mirror_histories()
        return out

    def processBlock(self, inputFrames, hopSize, blockSize, useGraph=True, forcedAtomMask=None):
        """One audio block through the device-resident overlap-add rings AND processFrames as a single CUDA graph launch:
        OverlapAddProcessor.processFrames(self.processFrames) of gccNMF/realtime/utils.py:99-116 / gccNMFProcessor.py:97.
        inputFrames (2, blockSize) float32 -> the next output block (2, blockSize) float32 (two blocks of latency, utils.py:115),
        or (numSources, 2, blockSize) in TARGET_MODE_MULTIPLE."""
        if self.engine is None or self._geometry != (int(hopSize), int(blockSize)):
            self.buildFunctions(hopSize, blockSize)
        self._sync_params()
        x = np.asarray(inputFrames, dtype=np.float32)
        if self._builtTargetMode == TARGET_MODE_MULTIPLE:
            out = self.engine.process_blocks(x[None], use_graph=useGraph, forcedAtomMask=forcedAtomMask)[0].copy()
        else:
            out = self.engine.process_block(x, use_graph=useGraph, forcedAtomMask=forcedAtomMask)
        self._mirror_histories()
        return out
