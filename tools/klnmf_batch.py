"""Batched offline KL-NMF (gccnmf_klnmf_batched): one call over B clips against B back-to-back gccnmf_klnmf calls, device time per
clip, 100 iterations, alternated for --rounds rounds in one session.

    python tools/klnmf_batch.py [--batches 1 8 32 128] [--iterations 100] [--rounds 3] [--json out.json]

Shapes: BASELINE.json configs[0] (F 513, 2T 622, K 128: a 10 s clip at hop 512) for every B in --batches, and a 10 s clip at hop
256 with K = 1024 (F 513, 2T 1250) for B in {1, 8}.  B = 1 against solo shows the batch form's own overhead.  Then the stage split
of GCCNMFPipeline.separate_batch on three 10 s clips at configs[0] settings (CUDA events between stages; the per-clip stages are
summed over the clips).  V is random; W0, H0 the seeded draw.  The card's name and power limit come from the same run.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from rt_streams import card  # noqa: E402


def events_ms(fn, reps=1):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / reps


def compare(h, B, F, T2, K, iters, rounds):
    import torch
    from gcc_nmf_b200 import gccNMFFunctions as fn
    rng = np.random.default_rng(B)
    V = h.to_device((rng.random((B, F, T2)) ** 3 + 1e-3).astype(np.float32))
    W0, H0 = fn._seededInit(F, T2, K, 1e-16, 0)
    W0, H0 = h.to_device(W0), h.to_device(H0)
    Wb, Hb, Ws, Hs = (torch.empty(s, dtype=torch.float32, device=h.device) for s in ((B, F, K), (B, K, T2)) * 2)   # (not views of W0, H0)

    def batch():
        Wb.copy_(W0.expand_as(Wb))
        Hb.copy_(H0.expand_as(Hb))
        h.klnmf_batched(V, Wb, Hb, iters)

    def solo():
        Ws.copy_(W0.expand_as(Ws))
        Hs.copy_(H0.expand_as(Hs))
        for b in range(B):
            h.klnmf(V[b], Ws[b], Hs[b], iters)
    batch(), solo()                                   # warm-up: modules, tensor maps, workspaces
    tb, ts = [], []
    for _ in range(rounds):
        tb.append(events_ms(batch))
        ts.append(events_ms(solo))
    same = all(bool(torch.all((a == b) | (torch.isnan(a) & torch.isnan(b)))) for a, b in ((Wb, Ws), (Hb, Hs)))   # NaN-equal
    row = dict(B=B, F=F, T2=T2, K=K, iterations=iters, batch_ms=float(np.median(tb)), solo_ms=float(np.median(ts)),
               batch_ms_per_clip=float(np.median(tb)) / B, solo_ms_per_clip=float(np.median(ts)) / B, bit_identical=same)
    row['speedup'] = row['solo_ms'] / row['batch_ms']
    print('B %4d  F %4d  2T %5d  K %4d:  batch %9.2f ms (%7.3f ms/clip)   solo %9.2f ms (%7.3f ms/clip)   x%.2f   same bits %s'
          % (B, F, T2, K, row['batch_ms'], row['batch_ms_per_clip'], row['solo_ms'], row['solo_ms_per_clip'], row['speedup'], same), flush=True)
    return row


def stage_split(h, iters):
    from gcc_nmf_b200.pipeline import GCCNMFPipeline
    from gcc_nmf_b200.synth import synthetic_stereo
    x = np.stack([synthetic_stereo(10.0, seed=s) for s in range(3)])
    pipe = GCCNMFPipeline(16000, 1024, 512, 64, 1.0, 128, iters, handle=h)
    xd = h.to_device(x)
    pipe.separate_batch(xd, 2)
    pipe.separate_batch(xd, 2, collect_stage_times=True)
    import torch
    torch.cuda.synchronize()
    times = pipe.stage_times_ms()
    print('separate_batch, 3 clips of 10 s: ' + ', '.join('%s %.2f ms' % kv for kv in times.items()), flush=True)
    return times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batches', type=int, nargs='+', default=[1, 8, 32, 128])
    ap.add_argument('--iterations', type=int, default=100)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--json', default=None)
    args = ap.parse_args()
    import torch
    from gcc_nmf_b200._lib import default_handle
    h = default_handle()
    out = dict(card=card(), device=torch.cuda.get_device_name(0), rows=[])
    print(out['card'], flush=True)
    for B in args.batches:
        out['rows'].append(compare(h, B, 513, 622, 128, args.iterations, args.rounds))
    for B in (1, 8):
        out['rows'].append(compare(h, B, 513, 1250, 1024, args.iterations, args.rounds))
    out['separate_batch_stages_ms'] = stage_split(h, args.iterations)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, 'w') as f:
            json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
