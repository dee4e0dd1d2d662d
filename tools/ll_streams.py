"""Per-launch latency of the streamed low-latency loop (lowlatency.LowLatencyEngine, gccnmf_ll_*) at the BASELINE.json configs[4]
shape: 1024-sample asymmetric analysis window (m = 64), hop 64, K = 256, D = 128, one hop per call, so one graph launch per 4 ms
of audio at 16 kHz.

    python tools/ll_streams.py [--streams 1 16 64 256 1024] [--inference 0 5] [--calls 300] [--warmup 30] [--single-max 64]
                               [--batch-seconds 30] [--json out.json]
    torchrun --nproc-per-node G tools/ll_streams.py ...      (one engine per rank, each on its own GPU; every rank reports)

For every S and inference count: device time (CUDA events on the engine's stream around each graph launch) and wall time (host,
launch to the synchronised output in pinned memory), p50 / p99, microseconds per stream; S single-stream engines launched back to
back in one timed window (up to --single-max streams); the largest S whose p99 fits the hop period.  Then the batch rate of
performOnlineSpeechEnhancement on --batch-seconds of audio at the same shape, per frame, against the single-stream launch.
Dictionaries are random; the audio is synthetic.  The card's name and power limit come from the same run.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from rt_streams import card, pct  # noqa: E402

N, M, HOP, K, D, SR = 1024, 64, 64, 256, 128, 16000


def setup():
    from gcc_nmf_b200 import gccNMFFunctions as fn
    from gcc_nmf_b200.online import getAsymmetricAnalysisWindow, getAsymmetricSynthesisWindow
    F = N // 2 + 1
    W = (np.random.default_rng(0).random((F, K)) ** 3 + 1e-3).astype(np.float32)
    E = fn.getExpJOmegaTau(fn.getFrequenciesInHz(SR, F), fn.getTDOAsInSeconds(0.1, D))
    return W, E, getAsymmetricAnalysisWindow(N, M, 0), getAsymmetricSynthesisWindow(N, M, 0)


def audio(S, calls):
    from gcc_nmf_b200.synth import synthetic_stereo
    base = synthetic_stereo(calls * HOP / float(SR) + 0.05, seed=7)[:, :calls * HOP].astype(np.float32)
    return np.stack([np.roll(base, 131 * s, axis=1) for s in range(S)])


def timed(engines, x, calls, warmup):
    """Per call: every engine's graph launched back to back on the first engine's stream; events around all of them."""
    import torch
    s = engines[0].stream
    graphs = [e.build_graph(1) for e in engines]
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    dev, wall = [], []
    per = x.shape[0] // len(engines)
    for c in range(warmup + calls):
        for i, e in enumerate(engines):
            e._buffers(1)[0].numpy()[:] = x[i * per:(i + 1) * per, :, (c % calls) * HOP:(c % calls + 1) * HOP]
        t0 = time.perf_counter()
        e0.record(s)
        for e, g in zip(engines, graphs):
            e.h.check(e.h.lib.gccnmf_rt_graph_launch(e.h.h, g, s.cuda_stream))
        e1.record(s)
        s.synchronize()
        t1 = time.perf_counter()
        if c >= warmup:
            dev.append(e0.elapsed_time(e1))
            wall.append((t1 - t0) * 1e3)
    return dev, wall


def batch_rate(W, E, win, syn, seconds):
    import torch
    from gcc_nmf_b200.online import performOnlineSpeechEnhancement
    from gcc_nmf_b200.synth import synthetic_stereo
    x = synthetic_stereo(seconds, seed=3).astype(np.float32)
    run = lambda: performOnlineSpeechEnhancement(x, SR, W, win, syn, HOP, D, 0.1, 0.05 * D, gainPerFrame=False)   # noqa: E731
    run()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = run()
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3
    frames = out[0].shape[2]
    return {'seconds': seconds, 'frames': frames, 'ms': ms, 'us_per_frame': ms * 1e3 / frames}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--streams', type=int, nargs='+', default=[1, 16, 64, 256, 1024])
    ap.add_argument('--inference', type=int, nargs='+', default=[0, 5])
    ap.add_argument('--calls', type=int, default=300)
    ap.add_argument('--warmup', type=int, default=30)
    ap.add_argument('--single-max', type=int, default=64)
    ap.add_argument('--batch-seconds', type=float, default=30.0)
    ap.add_argument('--json', default=None)
    a = ap.parse_args()
    import torch
    rank = int(os.environ.get('LOCAL_RANK', '0'))
    torch.cuda.set_device(rank)
    from gcc_nmf_b200.lowlatency import LowLatencyEngine
    W, E, win, syn = setup()
    hop_ms = HOP * 1e3 / SR
    rows = []
    for inf in a.inference:
        fits = 0
        for S in a.streams:
            x = audio(S, a.calls)
            eng = LowLatencyEngine(W, E, win, syn, HOP, numStreams=S, synthesis='windowed', targetTDOAEpsilon=0.05 * D,
                                   numInferenceIterations=inf, device=rank)
            dev, wall = timed([eng], x, a.calls, a.warmup)
            row = {'S': S, 'inference': inf, 'device': pct(dev), 'wall': pct(wall), 'us_per_stream_p50': pct(dev)['p50_ms'] * 1e3 / S}
            eng.close()
            del eng
            if S <= a.single_max:
                singles = [LowLatencyEngine(W, E, win, syn, HOP, numStreams=1, synthesis='windowed', targetTDOAEpsilon=0.05 * D,
                                            numInferenceIterations=inf, device=rank) for _ in range(S)]
                sdev, swall = timed(singles, x, a.calls, a.warmup)
                row['singles_device'] = pct(sdev)
                row['singles_wall'] = pct(swall)
                for e in singles:
                    e.close()
                del singles
            torch.cuda.empty_cache()
            if row['wall']['p99_ms'] <= hop_ms:
                fits = max(fits, S)
            rows.append(row)
            print(json.dumps({'rank': rank, **row}), flush=True)
        print(json.dumps({'rank': rank, 'inference': inf, 'largest_S_with_wall_p99_within_hop': fits, 'hop_ms': hop_ms}), flush=True)
    batch = batch_rate(W, E, win, syn, a.batch_seconds) if a.batch_seconds > 0 else None
    result = {'rank': rank, 'card': card(), 'shape': dict(N=N, m=M, hop=HOP, K=K, D=D, C=1, sr=SR), 'rows': rows, 'batch': batch}
    print(json.dumps({'rank': rank, 'card': result['card'], 'batch': batch}), flush=True)
    if a.json:
        with open(a.json if rank == 0 else '%s.rank%d' % (a.json, rank), 'w') as f:
            json.dump(result, f, indent=1)


if __name__ == '__main__':
    main()
