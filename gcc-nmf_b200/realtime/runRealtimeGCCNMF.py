"""Headless real-time runner: wav file -> blocks -> GCC-NMF speech enhancement -> wav file (SURVEY.md row f-4).

Mirrors the no-GUI path of the reference (gccNMF/realtime/runRealtimeGCCNMF.py:122-179 `RealtimeGCCNMFNoGUI`,
the file-player callback of gccNMF/realtime/audioProcessor.py:106-132, the defaults of gccNMF/realtime/config.py:46-82
and the parameter messages of `initParams`, runRealtimeGCCNMF.py:141-167) without its process shell: the reference runs
the audio callback and the GCC-NMF processor in two OS processes that hand one block at a time through shared arrays and
a pair of Events, i.e. strictly synchronously -- here the same two steps are called in sequence per block:

    inputFrames <- next blockSize samples of the file          (audioProcessor.py:112-116, int16 -> float32 / 32768)
    oladProcessor.processFrames(gccNMFProcessor.processFrames) (gccNMFProcessor.py:97)
    outputFrames -> int16 with clipping                        (audioProcessor.py:123, wavfile.py:92-110)

PyAudio, Qt and the parameter queues are out of scope (SURVEY.md section 2, rows 8, 10, 13); the per-block processing
times the reference logs every 2 s (audioProcessor.py:98-102) are returned as min / max / mean.

`numSources` = P >= 2 separates the file into P sources instead (GCCNMFProcessor in TARGET_MODE_MULTIPLE, targets from the
localisation): every block goes through the device-resident rings (`GCCNMFProcessor.processBlock`), the arrays gain a leading
source axis and `run` writes one wav file per source.
"""
import argparse
import logging
import time
from collections import namedtuple

import numpy as np

from ..wavio import float2pcm, pcm2float  # noqa: F401  (re-exported: the reference keeps them in gccNMF/wavfile.py)
from .utils import OverlapAddProcessor

# gccNMF/realtime/config.py:46-82 (getDefaultConfig) -- the reference never reads a config file (:104-111)
DEFAULT_PARAMS = dict(
    numTDOAs=64, numTDOAHistory=128, numSpectrogramHistory=128, gccPHATNLAlpha=2.0, gccPHATNLEnabled=False,
    microphoneSeparationInMetres=0.1, targetTDOAEpsilon=5.0, targetTDOABeta=2.0, targetTDOANoiseFloor=0.0,
    localizationEnabled=True, localizationWindowSize=6,
    numChannels=2, sampleRate=16000, deviceIndex=None,
    windowSize=1024, hopSize=512, blockSize=512,
    dictionarySize=64, dictionarySizes=[64, 128, 256, 512, 1024], dictionaryType='Pretrained', numHUpdates=0,
    numSources=0)                            # 0: enhancement (one output); P >= 2: P separated sources
HEADLESS_TARGET_TDOA_INDEX = 9.60          # runRealtimeGCCNMF.py:144


def getGCCNMFConfigParams(audioPath=None, dataDir=None, dictionariesW=None, **overrides):
    """config.py:107-120.  `dictionariesW` ({type: {size: W}}) replaces the CHiME pre-training when given; otherwise the
    dictionaries are loaded / pre-trained from `dataDir` (gccNMFPretraining.getDictionariesW)."""
    p = dict(DEFAULT_PARAMS)
    unknown = set(overrides) - set(p)
    if unknown:
        raise ValueError('unknown configuration options: %s' % sorted(unknown))
    p.update(overrides)
    p['audioPath'] = audioPath
    p['numFreq'] = p['windowSize'] // 2 + 1
    p['windowsPerBlock'] = p['blockSize'] // p['hopSize']
    if dictionariesW is None:
        if dataDir is None:
            raise ValueError('either dictionariesW or dataDir (with chimeTrainSet.npy or pretrainedW/) is required')
        from .gccNMFPretraining import getDictionariesW
        dictionariesW = getDictionariesW(p['windowSize'], p['dictionarySizes'], dataDir, ordered=True)
    p['dictionariesW'] = dictionariesW
    return namedtuple('ParamsDict', p.keys())(**p)


class RealtimeGCCNMFNoGUI(object):
    """File in, file out.  `processFramesFunction` (windowedSamples (2, N, windowsPerBlock) -> same shape) defaults to a
    GCCNMFProcessor built from `params` exactly as GCCNMFProcess.run builds it (gccNMFProcessor.py:66-75)."""

    def __init__(self, audioPath=None, params=None, processFramesFunction=None, device=0, **overrides):
        self.params = params if params is not None else getGCCNMFConfigParams(audioPath, **overrides)
        p = self.params
        self.inputFrames = np.zeros((p.numChannels, p.blockSize), np.float32)     # the reference's shared arrays (runRealtimeGCCNMF.py:64-72)
        self.outputFrames = np.zeros((p.numChannels, p.blockSize), np.float32)
        self.oladProcessor = OverlapAddProcessor(p.numChannels, p.windowSize, p.hopSize, p.blockSize, p.windowsPerBlock,
                                                 self.inputFrames, self.outputFrames)
        self.gccNMFProcessor = None
        if processFramesFunction is None:
            from .gccNMFProcessor import GCCNMFProcessor
            from .utils import CircularBuffer
            # the sliding-window localisation reads the GCC-PHAT history (gccNMFProcessor.py:216-227)
            self.gccPHATHistory = CircularBuffer((p.numTDOAs, p.numTDOAHistory)) if p.localizationEnabled else None
            self.tdoaHistory = CircularBuffer((1, p.numTDOAHistory)) if p.localizationEnabled else None
            g = GCCNMFProcessor(p.sampleRate, p.windowSize, p.windowsPerBlock, p.dictionariesW, p.dictionaryType, p.dictionarySize,
                                p.numHUpdates, p.microphoneSeparationInMetres, p.localizationEnabled, p.localizationWindowSize,
                                gccPHATHistory=self.gccPHATHistory, tdoaHistory=self.tdoaHistory, device=device)
            # the messages of initParams (runRealtimeGCCNMF.py:141-161)
            g.setTargetTDOARange(HEADLESS_TARGET_TDOA_INDEX, p.targetTDOAEpsilon, p.targetTDOABeta, p.targetTDOANoiseFloor)
            g.numTDOAs = p.numTDOAs
            g.separationEnabled = True
            if p.numSources:
                from .gccNMFProcessor import TARGET_MODE_MULTIPLE
                g.targetMode = TARGET_MODE_MULTIPLE
                g.numSources = p.numSources
            g.reset()
            self.gccNMFProcessor = g
            processFramesFunction = g.processFrames
        elif p.numSources:
            raise ValueError('numSources runs the built-in GCCNMFProcessor; this runner was given a processFramesFunction')
        self.processFramesFunction = processFramesFunction
        self.processingTimes = []

    @property
    def latencySamples(self):
        """The overlap-add ring emits block [-3B:-2B] (utils.py:116): the output lags the input by two blocks."""
        return 2 * self.params.blockSize

    def processBlock(self, block):
        """block (numChannels, blockSize) float32 -> the next output block (a view that is overwritten by the next call), or
        (numSources, numChannels, blockSize) with sources."""
        p = self.params
        startTime = time.time()
        if p.numSources:
            out = self.gccNMFProcessor.processBlock(block, p.hopSize, p.blockSize)
        else:
            self.inputFrames[:] = block
            self.oladProcessor.processFrames(self.processFramesFunction)
            out = self.outputFrames
        self.processingTimes.append(time.time() - startTime)
        return out

    def processSamples(self, samples, flush=True):
        """samples (numChannels, n) float32 -> (numChannels, n_out) float32 ((numSources, numChannels, n_out) with sources): whole
        blocks of the file, then (flush) two silent blocks so that the tail leaves the overlap-add ring; n_out = (blocks [+ 2]) * blockSize."""
        p = self.params
        samples = np.asarray(samples, dtype=np.float32)
        if samples.ndim != 2 or samples.shape[0] != p.numChannels:
            raise ValueError('expected (%d, n) samples, got %s' % (p.numChannels, samples.shape))
        B = p.blockSize
        numBlocks = (samples.shape[1] + B - 1) // B
        total = numBlocks + (2 if flush else 0)
        padded = np.zeros((p.numChannels, total * B), np.float32)
        padded[:, :samples.shape[1]] = samples
        out = np.empty(((p.numSources,) if p.numSources else ()) + padded.shape, np.float32)
        for b in range(total):
            out[..., b * B:(b + 1) * B] = self.processBlock(padded[:, b * B:(b + 1) * B])
        return out

    def processingTimeStats(self):
        """audioProcessor.py:98-102: (min, max, mean) seconds per block."""
        t = np.asarray(self.processingTimes)
        return (float(t.min()), float(t.max()), float(t.mean())) if t.size else (0.0, 0.0, 0.0)

    def _readSamples(self, audioPath):
        """int16 (or float) stereo wav -> (numChannels, n) float32 (audioProcessor.py:112-116)."""
        from scipy.io import wavfile
        sampleRate, data = wavfile.read(audioPath)
        if sampleRate != self.params.sampleRate:
            raise ValueError('sample rate of %s is %d, configured %d' % (audioPath, sampleRate, self.params.sampleRate))
        return pcm2float(data).T if data.dtype.kind in 'iu' else np.asarray(data, np.float32).T

    def _writeOutput(self, out, numSamples, outputPath, alignOutput):
        from scipy.io import wavfile
        if alignOutput:
            out = out[..., self.latencySamples:self.latencySamples + numSamples]
        if outputPath is not None:
            wavfile.write(outputPath, self.params.sampleRate, float2pcm(np.ascontiguousarray(out.T)))
        return out

    def run(self, outputPath=None, alignOutput=True):
        """Reads params.audioPath (int16 stereo wav), enhances it block by block and, when `outputPath` is given, writes
        the int16 result.  alignOutput drops the two-block latency so that output sample i corresponds to input sample i.
        With sources, `outputPath` is a list of numSources paths (one wav per source) and the result is (numSources, 2, n)."""
        p = self.params
        samples = self._readSamples(p.audioPath)
        out = self.processSamples(samples, flush=True)
        logging.info('Processing times (min/max/avg): %f, %f, %f' % self.processingTimeStats())
        if not p.numSources:
            return self._writeOutput(out, samples.shape[1], outputPath, alignOutput)
        if outputPath is not None and len(outputPath) != p.numSources:
            raise ValueError('%d sources, %d output paths' % (p.numSources, len(outputPath)))
        return np.stack([self._writeOutput(out[s], samples.shape[1], outputPath[s] if outputPath is not None else None, alignOutput)
                         for s in range(p.numSources)])

    def runMany(self, audioPaths, outputPaths=None, alignOutput=True, dictionarySizes=None, microphoneSeparations=None):
        """Several wav files enhanced concurrently, each in its own slot of ONE MultiStreamRealtimeEngine: per block, one graph
        launch for all files.  Each file gets exactly what `run` gives it alone (same parameters, same kernels, bit for bit);
        once a file has had its two flush blocks its slot is deactivated.  Returns the output arrays in the order of
        `audioPaths` and writes them to `outputPaths` when given.  `processingTimes` gets one entry per block of the longest file.
        dictionarySizes / microphoneSeparations: one per file (None: the runner's own), built into one bank of the distinct
        dictionaries of params.dictionariesW[dictionaryType] and the steering tables of the distinct spacings; each file then gets
        what `run` gives it with that dictionary size and spacing."""
        from .gccNMFProcessor import steeringVectors
        from .multistream import MultiStreamRealtimeEngine
        g = self.gccNMFProcessor
        if g is None:
            raise ValueError('runMany runs the built-in GCCNMFProcessor; this runner was given another processFramesFunction')
        if self.params.numSources:
            raise ValueError('runMany enhances one source per file; numSources is not supported there')
        if outputPaths is not None and len(outputPaths) != len(audioPaths):
            raise ValueError('%d input paths, %d output paths' % (len(audioPaths), len(outputPaths)))
        p = self.params
        B, S = p.blockSize, len(audioPaths)
        signals = [self._readSamples(path) for path in audioPaths]
        totals = [(x.shape[1] + B - 1) // B + 2 for x in signals]          # whole blocks + two flush blocks, as processSamples
        g.buildConstants()
        W, E, entries = g.W, g.expJOmegaTau, None
        if dictionarySizes is not None or microphoneSeparations is not None:
            sizes = [g.dictionarySize] * S if dictionarySizes is None else [int(k) for k in dictionarySizes]
            seps = [g.microphoneSeparationInMetres] * S if microphoneSeparations is None else [float(m) for m in microphoneSeparations]
            if len(sizes) != S or len(seps) != S:
                raise ValueError('one dictionary size and one microphone separation per file (%d files)' % S)
            distinctSizes, distinctSeps = sorted(set(sizes)), sorted(set(seps))
            W = [np.ascontiguousarray(p.dictionariesW[g.dictionaryType][k], dtype=np.float32) for k in distinctSizes]
            E = [steeringVectors(g.frequenciesInHz, m, g.numTDOAs)[2] for m in distinctSeps]
            entries = ([distinctSizes.index(k) for k in sizes], [distinctSeps.index(m) for m in seps])
        engine = MultiStreamRealtimeEngine(W, E, g.windowFunction[:, 0], g.synthesisWindowFunction[:, 0], p.hopSize, B,
                                           p.windowsPerBlock, S, historyLength=g.gccPHATHistory.size() if g.gccPHATHistory else 128,
                                           numInferenceIterations=g.coefficientInferenceIterations, device=g.device)
        try:
            if entries is not None:
                engine.assign(range(S), *entries)
            engine.set_params(range(S), **g.slotParams())
            outs = [np.empty((p.numChannels, t * B), np.float32) for t in totals]
            blocks = np.zeros((S, p.numChannels, B), np.float32)
            for b in range(max(totals)):
                done = [s for s in range(S) if totals[s] == b]
                if done:
                    engine.set_active(done, False)
                for s, x in enumerate(signals):
                    chunk = x[:, b * B:(b + 1) * B]
                    blocks[s] = 0
                    blocks[s, :, :chunk.shape[1]] = chunk
                startTime = time.time()
                y = engine.process_blocks(blocks)
                self.processingTimes.append(time.time() - startTime)
                for s in range(S):
                    if b < totals[s]:
                        outs[s][:, b * B:(b + 1) * B] = y[s]
        finally:
            engine.close()
        logging.info('Processing times (min/max/avg): %f, %f, %f' % self.processingTimeStats())
        return [self._writeOutput(outs[s], signals[s].shape[1], outputPaths[s] if outputPaths is not None else None, alignOutput)
                for s in range(S)]


def parseArguments(argv=None):
    """config.py:122-127 plus the output path and the dictionary directory (the reference takes DATA_DIR from defs.py)."""
    parser = argparse.ArgumentParser(description='Headless real-time GCC-NMF speech enhancement (H100)')
    parser.add_argument('-i', '--input', nargs='+', help='input wav file path(s); several are enhanced concurrently in one engine', required=True)
    parser.add_argument('-o', '--output', nargs='+', help='output wav file path(s): one per input, or one per source with --num-sources',
                        required=True)
    parser.add_argument('-d', '--data-dir', help='directory with chimeTrainSet.npy and / or pretrainedW/', required=True)
    parser.add_argument('--dictionary-size', type=int, default=DEFAULT_PARAMS['dictionarySize'])
    parser.add_argument('--num-sources', type=int, default=0, help='separate one input into this many sources (2 .. 8) instead of enhancing it')
    return parser.parse_args(argv)


if __name__ == '__main__':
    logging.getLogger().setLevel(logging.INFO)
    args = parseArguments()
    if args.num_sources:
        if len(args.input) != 1 or len(args.output) != args.num_sources:
            raise SystemExit('--num-sources %d: one input path and %d output paths' % (args.num_sources, args.num_sources))
    elif len(args.input) != len(args.output):
        raise SystemExit('%d input paths, %d output paths' % (len(args.input), len(args.output)))
    runner = RealtimeGCCNMFNoGUI(args.input[0], dataDir=args.data_dir, dictionarySize=args.dictionary_size,
                                 dictionarySizes=[args.dictionary_size], numSources=args.num_sources)
    if args.num_sources:
        runner.run(args.output)
    elif len(args.input) == 1:
        runner.run(args.output[0])
    else:
        runner.runMany(args.input, args.output)
