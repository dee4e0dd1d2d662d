"""Ragged offline KL-NMF (gccnmf_klnmf_ragged): one call over B clips of different lengths against B back-to-back gccnmf_klnmf calls
on the same clips, device time per clip, median of --rounds alternating rounds in one session, bit identity checked in every row.

    python tools/klnmf_ragged.py [--batches 8 32 128] [--iterations 100] [--rounds 3] [--json out.json]

Workloads: clip lengths drawn uniformly from 2 to 30 s at 16 kHz (seeded), 2T = 2 (1 + (n - N) / hop) frames, at two settings:
N 1024, hop 512, K 128 (BASELINE.json configs[0]) and N 1024, hop 256, K 1024.  Each row also gives the launches of the ragged call
and its host enqueue time (plans, tensor-map encodes, the table copy and the launches), and the distinct tile widths of each
contraction.  One more row per setting puts the ragged call on 32 equal-length 10 s clips beside gccnmf_klnmf_batched on the same
clips.  V is random; W0, H0 the seeded draw.  The card's name and power limit come from the same run.
"""
import argparse
import ctypes
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from klnmf_batch import events_ms  # noqa: E402
from rt_streams import card  # noqa: E402

SR, N_FFT = 16000, 1024


def frames2(seconds, hop):
    return 2 * (1 + (int(seconds * SR) - N_FFT) // hop)


def same(a, b):
    import torch
    return bool(torch.all((a == b) | (torch.isnan(a) & torch.isnan(b))))


def compare(h, T2s, K, iters, rounds, label):
    import torch
    from gcc_nmf_b200 import gccNMFFunctions as fn
    F, B = N_FFT // 2 + 1, len(T2s)
    rng = np.random.default_rng(B)
    Vs = [h.to_device((rng.random((F, t)) ** 3 + 1e-3).astype(np.float32)) for t in T2s]
    W0, Hmax = fn._seededInit(F, max(T2s), K, 1e-16, 0)
    W0, Hflat = h.to_device(W0), h.to_device(Hmax).reshape(-1)
    H0 = [Hflat[:K * t].view(K, t) for t in T2s]
    Wr, Ws = (torch.empty((B, F, K), dtype=torch.float32, device=h.device) for _ in range(2))
    Hr, Hs = ([torch.empty((K, t), dtype=torch.float32, device=h.device) for t in T2s] for _ in range(2))
    enqueue = []

    def ragged():
        Wr.copy_(W0.expand_as(Wr))
        for H, H0b in zip(Hr, H0):
            H.copy_(H0b)
        t0 = time.perf_counter()
        h.klnmf_ragged(Vs, Wr, Hr, iters)
        enqueue.append(time.perf_counter() - t0)

    def solo():
        Ws.copy_(W0.expand_as(Ws))
        for b in range(B):
            Hs[b].copy_(H0[b])
            h.klnmf(Vs[b], Ws[b], Hs[b], iters)
    ragged(), solo()                                  # warm-up: modules, tensor maps, workspaces
    launches = h.launches
    ragged()
    launches = h.launches - launches
    torch.cuda.synchronize()
    tr, ts = [], []
    for _ in range(rounds):
        tr.append(events_ms(ragged))
        ts.append(events_ms(solo))
    bits = same(Wr, Ws) and all(same(a, b) for a, b in zip(Hr, Hs))
    plan = (ctypes.c_int * 8)()
    sm = torch.cuda.get_device_properties(h.device).multi_processor_count
    widths = [set(), set(), set(), set()]
    for t in T2s:
        h.lib.gccnmf_klnmf_tile_plan(sm, F, t, K, plan)
        for i in range(4):
            widths[i].add(plan[i])
    row = dict(workload=label, B=B, K=K, T2_min=min(T2s), T2_max=max(T2s), T2_sum=int(sum(T2s)), iterations=iters,
               ragged_ms=float(np.median(tr)), solo_ms=float(np.median(ts)), launches=launches,
               host_enqueue_ms=1e3 * float(np.median(enqueue[2:])),
               widths=dict(wh=sorted(widths[0]), h=sorted(widths[1]), w=sorted(widths[2]), w_splits=sorted(widths[3])), bit_identical=bits)
    row['ragged_ms_per_clip'] = row['ragged_ms'] / B
    row['solo_ms_per_clip'] = row['solo_ms'] / B
    row['speedup'] = row['solo_ms'] / row['ragged_ms']
    print('%-10s B %4d  K %4d  2T %4d..%4d:  ragged %9.2f ms (%7.3f ms/clip)  solo %9.2f ms (%7.3f ms/clip)  x%.2f  launches %d  enqueue %.2f ms  '
          'widths %s  same bits %s' % (label, B, K, row['T2_min'], row['T2_max'], row['ragged_ms'], row['ragged_ms_per_clip'], row['solo_ms'],
                                       row['solo_ms_per_clip'], row['speedup'], launches, row['host_enqueue_ms'], row['widths'], bits), flush=True)
    return row


def equal_lengths(h, B, T2, K, iters, rounds, label):
    """The ragged call on B equal-length clips beside gccnmf_klnmf_batched on the same clips."""
    import torch
    from gcc_nmf_b200 import gccNMFFunctions as fn
    F = N_FFT // 2 + 1
    rng = np.random.default_rng(7)
    V = h.to_device((rng.random((B, F, T2)) ** 3 + 1e-3).astype(np.float32))
    W0, H0 = (h.to_device(x) for x in fn._seededInit(F, T2, K, 1e-16, 0))
    Wb, Wr = (torch.empty((B, F, K), dtype=torch.float32, device=h.device) for _ in range(2))
    Hb, Hr = (torch.empty((B, K, T2), dtype=torch.float32, device=h.device) for _ in range(2))

    def batched():
        Wb.copy_(W0.expand_as(Wb))
        Hb.copy_(H0.expand_as(Hb))
        h.klnmf_batched(V, Wb, Hb, iters)

    def ragged():
        Wr.copy_(W0.expand_as(Wr))
        Hr.copy_(H0.expand_as(Hr))
        h.klnmf_ragged(list(V), Wr, list(Hr), iters)
    batched(), ragged()
    tb, tr = [], []
    for _ in range(rounds):
        tb.append(events_ms(batched))
        tr.append(events_ms(ragged))
    bits = same(Wb, Wr) and same(Hb, Hr)
    row = dict(workload=label, B=B, K=K, T2=T2, iterations=iters, batched_ms=float(np.median(tb)), ragged_ms=float(np.median(tr)), bit_identical=bits)
    print('%-10s B %4d  K %4d  2T %4d equal:  batched %9.2f ms  ragged %9.2f ms  (ragged / batched %.3f)  same bits %s'
          % (label, B, K, T2, row['batched_ms'], row['ragged_ms'], row['ragged_ms'] / row['batched_ms'], bits), flush=True)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batches', type=int, nargs='+', default=[8, 32, 128])
    ap.add_argument('--iterations', type=int, default=100)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--json', default=None)
    args = ap.parse_args()
    import torch
    from gcc_nmf_b200._lib import default_handle
    h = default_handle()
    out = dict(card=card(), device=torch.cuda.get_device_name(0), rows=[], equal_length_rows=[])
    print(out['card'], flush=True)
    for label, hop, K in (('hop512_K128', 512, 128), ('hop256_K1024', 256, 1024)):
        rng = np.random.default_rng(hop)
        for B in args.batches:
            T2s = [frames2(s, hop) for s in rng.uniform(2.0, 30.0, B)]
            out['rows'].append(compare(h, T2s, K, args.iterations, args.rounds, label))
            torch.cuda.empty_cache()
        out['equal_length_rows'].append(equal_lengths(h, 32, frames2(10.0, hop), K, args.iterations, args.rounds, label))
        torch.cuda.empty_cache()
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, 'w') as f:
            json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
