"""Where one KL-NMF iteration spends its time, contraction by contraction, at the benchmark shape on one GPU.

  python tools/nmf_phases.py [--iterations 100] [--gemm-cluster 10CN+CM] [--gemm-pair -1|0|1] [--wh-tile BN] [--out FILE.json]

Runs the KL-NMF loop (F = 513, T2 = 3744, K = 1024) with the plane GEMM's timing records on (gccnmf_debug_timing: 8 uint64 per
CTA; see csrc/tma_gemm.cuh) and prints for G1 - G4 and the W update: the exclusive time of each launch (end of the previous
one to its own end) and the gap to the next one, the median and maximum per-CTA fill (start -> first stage full), main loop (first stage full -> last MMA retired) and epilogue (accumulators staged -> epilogue end), and the executed
tensor rate over the main-loop windows only.  The card's name and power limit come from the same run.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

F, T2, K = 513, 3744, 1024


def card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out.splitlines()[0] if out else 'unknown'
    except Exception:   # noqa: BLE001
        return 'unknown'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iterations', type=int, default=100)
    ap.add_argument('--gemm-cluster', type=int, default=-1, help='option gemm_cluster (10 CN + CM; -1: automatic)')
    ap.add_argument('--gemm-pair', type=int, default=-1, help='option gemm_pair (-1: where a call site prefers CTA pairs)')
    ap.add_argument('--wh-tile', type=int, default=0, help='option wh_tile: tile width of G1 / G3 (0: planned)')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    import torch
    from gcc_nmf_b200._lib import default_handle
    h = default_handle()
    h.set_option('gemm_cluster', args.gemm_cluster)
    h.set_option('gemm_pair', args.gemm_pair)
    h.set_option('wh_tile', args.wh_tile)
    sms = torch.cuda.get_device_properties(h.device).multi_processor_count
    plan = (ctypes.c_int * 8)()
    h.check(h.lib.gccnmf_klnmf_tile_plan(sms, F, T2, K, plan))
    bn_wh, bn_h, bn_w, splits_w, _, rec_wh, rec_h, rec_w = list(plan)
    if args.wh_tile:
        bn_wh, rec_wh = args.wh_tile, (F // 128) * ((T2 + args.wh_tile - 1) // args.wh_tile)
    rng = np.random.default_rng(5)
    V = h.to_device((rng.random((F, T2)) ** 3 + 1e-3).astype(np.float32))
    W0 = h.to_device((rng.random((F, K)) + 1e-2).astype(np.float32))
    H0 = h.to_device((rng.random((K, T2)) + 1e-2).astype(np.float32))
    W, H = W0.clone(), H0.clone()
    h.klnmf(V, W, H, 5)                          # warm-up: modules, tensor maps, attributes
    per_it = 2 * rec_wh + rec_h + rec_w + 1
    buf = torch.zeros(per_it * 8 * args.iterations + 64, dtype=torch.int64, device=h.device)
    torch.cuda.synchronize()
    h.lib.gccnmf_debug_timing(h.h, buf.data_ptr(), 1)
    W, H = W0.clone(), H0.clone()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    h.klnmf(V, W, H, args.iterations)
    e1.record()
    e1.synchronize()
    used = h.lib.gccnmf_debug_timing(h.h, None, 1)
    assert used == per_it * 8 * args.iterations, (used, per_it * 8 * args.iterations)
    s = buf.cpu().numpy()[:used].reshape(args.iterations, per_it, 8).astype(np.int64)

    # executed tensor FLOP per launch (3 hi / lo products per k-step in every contraction; tail rows excluded)
    m_wh = (F // 128) * 128
    flops = {'G1': 3 * 2.0 * m_wh * T2 * K, 'G2': 3 * 2.0 * K * T2 * F, 'G3': 3 * 2.0 * m_wh * T2 * K, 'G4': 3 * 2.0 * K * F * T2}
    layout = [('G1', rec_wh), ('G2', rec_h), ('G3', rec_wh), ('G4', rec_w), ('W update', 1)]
    # ns per clock64 cycle, from records whose globaltimer and clock64 windows cover the same stretch
    spans = []
    rows = {}
    off = 0
    for name, n in layout:
        rows[name] = s[:, off:off + n, :]
        off += n
    for name in ('G1', 'G2', 'G3'):
        r = rows[name].reshape(-1, 8)
        ok = (r[:, 6] > r[:, 1]) & (r[:, 7] > r[:, 0])
        spans.append(np.median((r[ok, 7] - r[ok, 0]) / (r[ok, 6] - r[ok, 1])))
    ns_per_cycle = float(np.median(spans))
    result = {'card': card(), 'iterations': args.iterations, 'gemm_cluster': args.gemm_cluster, 'gemm_pair': args.gemm_pair, 'wh_tile': args.wh_tile,
              'plan': {'bn_wh': bn_wh, 'bn_h': bn_h, 'bn_w': bn_w, 'splits_w': splits_w, 'records': [rec_wh, rec_h, rec_w]},
              'loop_ms_events': e0.elapsed_time(e1), 'ns_per_cycle_est': ns_per_cycle, 'launches': {}}
    starts = {name: rows[name][:, :, 0].min(axis=1) for name, _ in layout}
    ends = {name: rows[name][:, :, 7].max(axis=1) for name, _ in layout}
    order = [name for name, _ in layout]
    print('card: %s | %d iterations, %.1f us per iteration (CUDA events) | plan: G1/G3 bn %d (%d records), G2 bn %d (%d), G4 bn %d x %d splits (%d)' % (
        result['card'], args.iterations, e0.elapsed_time(e1) * 1e3 / args.iterations, bn_wh, rec_wh, bn_h, rec_h, bn_w, splits_w, rec_w))
    # exclusive time of a launch: from the end of the previous launch to its own end (they add up to the iteration; with
    # programmatic dependent launch a grid's first CTAs start before the previous grid ends)
    print('%-9s %9s %9s | %-23s | %-23s | %-23s | %10s %7s' % ('', 'excl us', 'gap us', 'fill us p50 / max', 'main us p50 / max',
                                                              'epilogue us p50 / max', 'TFLOP/s', 'SMs'))
    for i, name in enumerate(order):
        nxt_start = starts[order[i + 1]] if i + 1 < len(order) else np.concatenate([starts['G1'][1:], [np.nan]])
        prev_end = ends[order[i - 1]] if i > 0 else np.concatenate([[np.nan], ends['W update'][:-1]])
        span = float(np.nanmedian(ends[name] - prev_end)) / 1e3
        gap = float(np.nanmedian(nxt_start - ends[name])) / 1e3
        entry = {'exclusive_us': span, 'gap_to_next_us': gap}
        if name == 'W update':
            print('%-9s %9.1f %9.1f |' % (name, span, gap))
            result['launches'][name] = entry
            continue
        r = rows[name].reshape(-1, 8)
        r = r[(r[:, 2] > 0) & (r[:, 3] > 0)]
        cyc = lambda a, b: (r[:, b] - r[:, a]) * ns_per_cycle / 1e3   # noqa: E731
        fill, main_, epi = cyc(1, 2), cyc(2, 3), cyc(5, 6)
        # rate over the main-loop windows: the launch's executed FLOP over its summed main-loop time, spread over the SMs that ran it
        # (one CTA per SM: min(SM count, CTAs of the launch))
        n_sm = min(sms, rows[name].shape[1])
        main_total_s = main_.sum() / args.iterations * 1e-6
        rate = flops[name] / (main_total_s / n_sm) / 1e12
        entry.update({'fill_us': [float(np.median(fill)), float(fill.max())], 'main_us': [float(np.median(main_)), float(main_.max())],
                      'epilogue_us': [float(np.median(epi)), float(epi.max())], 'main_loop_tflops': rate, 'sms': n_sm})
        result['launches'][name] = entry
        print('%-9s %9.1f %9.1f | %10.2f / %10.2f | %10.2f / %10.2f | %10.2f / %10.2f | %10.0f %7d' % (
            name, span, gap, np.median(fill), fill.max(), np.median(main_), main_.max(), np.median(epi), epi.max(), rate, n_sm))
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(result, f, indent=1)
    return 0


if __name__ == '__main__':
    sys.exit(main())
