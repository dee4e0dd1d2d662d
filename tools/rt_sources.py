"""Device time per block of the real-time path with P sources per stream (MultiStreamRealtimeEngine(numSources=P),
gccnmf_rtsep_*) at the BASELINE.json configs[2] shape: 512-FFT, hop 128, K = 1024, D = 64, one frame per block (8 ms of audio at
16 kHz), with 0 and 10 inference iterations.  P = 0 is the single-target multi-stream engine (gccnmf_rtm_*).

    python tools/rt_sources.py [--streams 1 64 256] [--sources 0 2 3 4] [--inference 0 10] [--blocks 400] [--warmup 50] [--json out.json]

Per (inference, S, P): CUDA events on the engine's stream around each graph launch (H2D + kernels + D2H), p50 / p99 in ms, and
the p50 per stream and source.  Localisation is on in every slot, so the sources' targets follow the audio.  The card's name and
power limit come from the same run.  The dictionary is random (its values do not change the work).
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from rt_streams import audio, card, pct, setup  # noqa: E402


def run(W, E, win, hop, B, nT, S, P, inference, blocks, warmup, x):
    import torch
    from gcc_nmf_b200.realtime.multistream import MultiStreamRealtimeEngine
    eng = MultiStreamRealtimeEngine(W, E, win, win, hop, B, nT, S, numInferenceIterations=inference, numSources=P)
    eng.set_params(range(S), targetTDOAIndex=10.0, epsilon=5.0, beta=2.0, localizationEnabled=True)
    dev = []
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    graph = eng.build_graph()
    for b in range(warmup + blocks):
        eng.in_host.numpy()[:] = x[b % x.shape[0]]
        e0.record(eng.stream)
        eng.h.check(eng.h.lib.gccnmf_rt_graph_launch(eng.h.h, graph, eng.stream.cuda_stream))
        e1.record(eng.stream)
        eng.stream.synchronize()
        if b >= warmup:
            dev.append(e0.elapsed_time(e1))
    eng.close()
    return dev


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--streams', type=int, nargs='*', default=[1, 64, 256])
    ap.add_argument('--sources', type=int, nargs='*', default=[0, 2, 3, 4])
    ap.add_argument('--inference', type=int, nargs='*', default=[0, 10])
    ap.add_argument('--blocks', type=int, default=400)
    ap.add_argument('--warmup', type=int, default=50)
    ap.add_argument('--json', default=None)
    args = ap.parse_args()
    import torch
    name = torch.cuda.get_device_name(0)
    power = card()
    K, N, hop, D, nT = 1024, 512, 128, 64, 1
    B = hop * nT
    W, E, win = setup(K, N, D)
    print('card: %s | nvidia-smi name, power limit: %s' % (name, power), flush=True)
    print('%d-FFT hop %d K=%d D=%d, %d frame per block, block period %.1f ms' % (N, hop, K, D, nT, B / 16.0), flush=True)
    results = []
    for inf in args.inference:
        for S in args.streams:
            x = audio(S, B, 32)
            for P in args.sources:
                r = {'inference': inf, 'S': S, 'P': P, 'device': pct(run(W, E, win, hop, B, nT, S, P, inf, args.blocks, args.warmup, x))}
                r['us_per_stream_source_p50'] = r['device']['p50_ms'] * 1e3 / (S * max(P, 1))
                results.append(r)
                print('inference %2d S=%4d P=%d: device p50 %.3f p99 %.3f ms, %.2f us per stream and source' % (
                    inf, S, P, r['device']['p50_ms'], r['device']['p99_ms'], r['us_per_stream_source_p50']), flush=True)
    if args.json:
        json.dump({'card': name, 'nvidia_smi': power, 'results': results}, open(args.json, 'w'), indent=1)


if __name__ == '__main__':
    main()
