"""Device time per block of the real-time path over a bank of dictionaries and steering tables (MultiStreamRealtimeEngine with
sequences of W and expJOmegaTau, gccnmf_rtbank_*) at the BASELINE.json configs[2] shape: 512-FFT, hop 128, D = 64, one frame per
block (8 ms of audio at 16 kHz), with 0 and 10 inference iterations.

    python tools/rt_bank.py [--streams 256] [--inference 0 10] [--blocks 300] [--warmup 50] [--rounds 3] [--json out.json]

Two comparisons, each run alternately for --rounds rounds (CUDA events on the engine's stream around each graph launch):
  one entry   S streams on a bank of one dictionary (K = 1024) and one steering table, against the rtm engine of the same W, E:
              the cost of the indirection;
  spread      S streams spread evenly over K in {64, 128, 256, 512, 1024} (K_max = 1024) and two microphone spacings, against
              five rtm engines (one per K, S / 5 streams each) launched back to back in one timed window.
Localisation is on in every slot.  The card's name and power limit come from the same run.  Dictionaries are random.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from rt_streams import audio, card, pct  # noqa: E402

SIZES = [64, 128, 256, 512, 1024]


def steering(N, D, sep):
    from gcc_nmf_b200.realtime.gccNMFProcessor import steeringVectors
    return steeringVectors(np.linspace(0, 8000, N // 2 + 1).astype(np.float32), sep, D)[2]


def engine(W, E, win, hop, B, nT, S, inference):
    from gcc_nmf_b200.realtime.multistream import MultiStreamRealtimeEngine
    e = MultiStreamRealtimeEngine(W, E, win, win, hop, B, nT, S, numInferenceIterations=inference)
    e.set_params(range(S), targetTDOAIndex=10.0, epsilon=5.0, beta=2.0, localizationEnabled=True)
    return e


def timed(engines, xs, blocks, warmup):
    """Per block: every engine's graph launched back to back on the first engine's stream, one event pair around all of them."""
    import torch
    s = engines[0].stream
    graphs = [e.build_graph() for e in engines]
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    dev = []
    for b in range(warmup + blocks):
        for e, x in zip(engines, xs):
            e.in_host.numpy()[:] = x[b % x.shape[0]]
        e0.record(s)
        for e, g in zip(engines, graphs):
            e.h.check(e.h.lib.gccnmf_rt_graph_launch(e.h.h, g, s.cuda_stream))
        e1.record(s)
        s.synchronize()
        if b >= warmup:
            dev.append(e0.elapsed_time(e1))
    return dev


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--streams', type=int, nargs='*', default=[256])
    ap.add_argument('--inference', type=int, nargs='*', default=[0, 10])
    ap.add_argument('--blocks', type=int, default=300)
    ap.add_argument('--warmup', type=int, default=50)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--json', default=None)
    args = ap.parse_args()
    import torch
    name = torch.cuda.get_device_name(0)
    power = card()
    N, hop, D, nT = 512, 128, 64, 1
    B = hop * nT
    F = N // 2 + 1
    rng = np.random.default_rng(0)
    Ws = {K: (rng.random((F, K)) ** 3).astype(np.float32) for K in SIZES}
    Es = [steering(N, D, 0.1), steering(N, D, 0.2)]
    win = np.sqrt(np.hamming(N).astype(np.float32))
    print('card: %s | nvidia-smi name, power limit: %s' % (name, power), flush=True)
    print('%d-FFT hop %d D=%d, %d frame per block, block period %.1f ms' % (N, hop, D, nT, B / 16.0), flush=True)
    results = []
    for inf in args.inference:
        for S in args.streams:
            x = audio(S, B, 32)
            one_bank = engine([Ws[1024]], [Es[0]], win, hop, B, nT, S, inf)
            one_rtm = engine(Ws[1024], Es[0], win, hop, B, nT, S, inf)
            spread = engine([Ws[K] for K in SIZES], Es, win, hop, B, nT, S, inf)
            spread.assign(range(S), [s % len(SIZES) for s in range(S)], [s % 2 for s in range(S)])
            per = [[s for s in range(S) if s % len(SIZES) == i] for i in range(len(SIZES))]
            five = [engine(Ws[K], Es[0], win, hop, B, nT, len(per[i]), inf) for i, K in enumerate(SIZES)]
            t = {k: [] for k in ('bank_one', 'rtm_one', 'bank_spread', 'rtm_five')}
            for _ in range(args.rounds):
                t['bank_one'] += timed([one_bank], [x], args.blocks, args.warmup)
                t['rtm_one'] += timed([one_rtm], [x], args.blocks, args.warmup)
                t['bank_spread'] += timed([spread], [x], args.blocks, args.warmup)
                t['rtm_five'] += timed(five, [x[:, p] for p in per], args.blocks, args.warmup)
            for e in [one_bank, one_rtm, spread] + five:
                e.close()
            r = {'inference': inf, 'S': S}
            r.update({k: pct(v) for k, v in t.items()})
            results.append(r)
            print('inference %2d S=%4d: one entry bank p50 %.3f p99 %.3f ms | rtm p50 %.3f p99 %.3f ms || spread bank p50 %.3f p99 %.3f ms | '
                  'five rtm p50 %.3f p99 %.3f ms' % (inf, S, r['bank_one']['p50_ms'], r['bank_one']['p99_ms'], r['rtm_one']['p50_ms'],
                                                     r['rtm_one']['p99_ms'], r['bank_spread']['p50_ms'], r['bank_spread']['p99_ms'],
                                                     r['rtm_five']['p50_ms'], r['rtm_five']['p99_ms']), flush=True)
    if args.json:
        json.dump({'card': name, 'nvidia_smi': power, 'results': results}, open(args.json, 'w'), indent=1)


if __name__ == '__main__':
    main()
