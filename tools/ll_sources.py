"""Per-launch latency of the streamed low-latency loop with several sources per stream (lowlatency.LowLatencyEngine(numSources=P),
gccnmf_llsep_*) at the BASELINE.json configs[4] shape: 1024-sample asymmetric analysis window (m = 64), hop 64, K = 256, D = 128,
`windowed` synthesis, one hop per call, so one graph launch per 4 ms of audio at 16 kHz.

    python tools/ll_sources.py [--streams 1 64 256 1024] [--sources 0 2 4] [--inference 0 5] [--calls 300] [--warmup 30]
                               [--json out.json]

For every S, P and inference count: device time (CUDA events on the engine's stream around each graph launch) and wall time (host,
launch to the synchronised output in pinned memory), p50 / p99, and whether the p99 wall time fits the hop period.  P = 0 is the
single-target engine.  Dictionaries are random; the audio is synthetic (ll_streams.audio).  The card's name and power limit come
from the same run.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from ll_streams import D, HOP, SR, audio, setup, timed  # noqa: E402
from rt_streams import card, pct  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--streams', type=int, nargs='+', default=[1, 64, 256, 1024])
    ap.add_argument('--sources', type=int, nargs='+', default=[0, 2, 4])
    ap.add_argument('--inference', type=int, nargs='+', default=[0, 5])
    ap.add_argument('--calls', type=int, default=300)
    ap.add_argument('--warmup', type=int, default=30)
    ap.add_argument('--json', default=None)
    a = ap.parse_args()
    import torch
    from gcc_nmf_b200.lowlatency import LowLatencyEngine
    W, E, win, syn = setup()
    hop_ms = HOP * 1e3 / SR
    rows = []
    for inf in a.inference:
        for S in a.streams:
            x = audio(S, a.calls)
            for P in a.sources:
                eng = LowLatencyEngine(W, E, win, syn, HOP, numStreams=S, synthesis='windowed', targetTDOAEpsilon=0.05 * D,
                                       numInferenceIterations=inf, numSources=P)
                dev, wall = timed([eng], x, a.calls, a.warmup)
                eng.close()
                del eng
                torch.cuda.empty_cache()
                row = {'S': S, 'P': P, 'inference': inf, 'device': pct(dev), 'wall': pct(wall),
                       'wall_p99_within_hop': pct(wall)['p99_ms'] <= hop_ms}
                rows.append(row)
                print(json.dumps(row), flush=True)
    result = {'card': card(), 'shape': dict(N=1024, m=64, hop=HOP, K=256, D=D, C=1, sr=SR, synthesis='windowed'), 'hop_ms': hop_ms,
              'rows': rows}
    print(json.dumps({'card': result['card'], 'hop_ms': hop_ms}), flush=True)
    if a.json:
        with open(a.json, 'w') as f:
            json.dump(result, f, indent=1)


if __name__ == '__main__':
    main()
