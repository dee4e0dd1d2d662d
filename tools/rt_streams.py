"""Many streams through one real-time engine (MultiStreamRealtimeEngine) at the BASELINE.json configs[2] shape: 512-FFT, hop 128,
K = 1024, D = 64, one frame per block (8 ms of audio at 16 kHz), with 0 and 10 inference iterations.

    python tools/rt_streams.py [--streams 1 8 64 256 1024] [--inference 0 10] [--blocks 400] [--warmup 50] [--singles-max 64] [--json out.json]

For each S it reports:
  graph    device time per graph launch (CUDA events around the launch on the engine's stream: H2D + kernels + D2H), p50 / p99,
           and wall time per block (host copy into the pinned buffer, graph launch, synchronisation), p50 / p99; microseconds per stream
  singles  (S <= --singles-max) the same S as S separate RealtimeEngines, one graph launch + synchronisation each, back to back:
           the sum of their device times and the wall time per block
  atoms    the batched atoms kernel alone (torch.profiler, separate run) and its FP32 rate 2 S nT D F K / time against the
           67 TFLOP/s data-sheet figure of the H100 SXM
and the largest S whose p99 wall time per block stays within the block period.  The card's name and power limit come from the
same run.  The dictionary is random (its values do not change the work); every slot gets its own synthetic two-source mixture.
"""
import argparse
import json
import os
import re
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FP32_PEAK_TFLOPS = 67.0       # H100 SXM data sheet, FP32 (non-tensor)


def card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out.splitlines()[0] if out else 'unknown'
    except Exception:   # noqa: BLE001
        return 'unknown'


def pct(a):
    a = np.asarray(a, np.float64)
    return {'p50_ms': float(np.percentile(a, 50)), 'p99_ms': float(np.percentile(a, 99)), 'mean_ms': float(a.mean())}


def setup(K, N, D, sr=16000):
    from gcc_nmf_b200 import gccNMFFunctions as fn
    F = N // 2 + 1
    W = (np.random.default_rng(0).random((F, K)) ** 3).astype(np.float32)
    freq = np.linspace(0, sr / 2, F).astype(np.float32)
    maxT = 0.1 / fn.SPEED_OF_SOUND_IN_METRES_PER_SECOND
    E = np.exp(np.outer(freq, -(2j * np.pi) * np.linspace(-maxT, maxT, D).astype(np.float32))).astype(np.complex64)
    win = np.sqrt(np.hamming(N).astype(np.float32))
    return W, E, win


def audio(S, B, blocks):
    from gcc_nmf_b200.synth import synthetic_stereo
    base = synthetic_stereo(blocks * B / 16000.0 + 0.05, seed=7)[:, :blocks * B]
    # distinct streams without S synthesis runs: circular shifts of one mixture
    return np.stack([np.roll(base, 131 * s, axis=1) for s in range(S)]).reshape(S, 2, blocks, B).transpose(2, 0, 1, 3).copy()


def run_multi(W, E, win, hop, B, nT, S, inference, blocks, warmup, x):
    import torch
    from gcc_nmf_b200.realtime.multistream import MultiStreamRealtimeEngine
    eng = MultiStreamRealtimeEngine(W, E, win, win, hop, B, nT, S, numInferenceIterations=inference)
    eng.set_params(range(S), targetTDOAIndex=10.0, epsilon=5.0, beta=2.0, localizationEnabled=True)
    dev, wall = [], []
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for b in range(warmup + blocks):
        blk = x[b % x.shape[0]]
        t0 = time.perf_counter()
        eng.in_host.numpy()[:] = blk
        e0.record(eng.stream)
        eng.h.check(eng.h.lib.gccnmf_rt_graph_launch(eng.h.h, eng.build_graph(), eng.stream.cuda_stream))
        e1.record(eng.stream)
        eng.stream.synchronize()
        t1 = time.perf_counter()
        if b >= warmup:
            wall.append((t1 - t0) * 1e3)
            dev.append(e0.elapsed_time(e1))
    eng.close()
    return dev, wall


def run_singles(W, E, win, hop, B, nT, S, inference, blocks, warmup, x):
    import torch
    from gcc_nmf_b200.realtime.engine import RealtimeEngine
    engines = []
    for s in range(S):
        e = RealtimeEngine(W, E, win, win, hop, B, nT, numInferenceIterations=inference)
        e.set_params(10.0, 5.0, 2.0, 0.0, 1, True, True, 6)
        engines.append(e)
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(S)]
    dev, wall = [], []
    for b in range(warmup + blocks):
        blk = x[b % x.shape[0]]
        t0 = time.perf_counter()
        for s, e in enumerate(engines):
            e.in_host.numpy()[:] = blk[s]
            ev[s][0].record(e.stream)
            e.h.check(e.h.lib.gccnmf_rt_graph_launch(e.h.h, e.build_graph(), e.stream.cuda_stream))
            ev[s][1].record(e.stream)
            e.stream.synchronize()
        t1 = time.perf_counter()
        if b >= warmup:
            wall.append((t1 - t0) * 1e3)
            dev.append(sum(a.elapsed_time(c) for a, c in ev))
    for e in engines:
        e.close()
    return dev, wall


def atoms_kernel_ms(W, E, win, hop, B, nT, S, inference, x, reps=20):
    """Mean time of the atoms kernel per block from torch.profiler (kernel-by-kernel launches)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    from gcc_nmf_b200.realtime.multistream import MultiStreamRealtimeEngine
    eng = MultiStreamRealtimeEngine(W, E, win, win, hop, B, nT, S, numInferenceIterations=inference)
    for b in range(3):
        eng.process_blocks(x[b % x.shape[0]], use_graph=False)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for b in range(reps):
            eng.process_blocks(x[b % x.shape[0]], use_graph=False)
        torch.cuda.synchronize()
    times, names = [], set()
    for evt in prof.events():
        if 'rt_atoms_kernel' in evt.name and evt.device_type == torch.autograd.DeviceType.CUDA:
            times.append(evt.device_time if hasattr(evt, 'device_time') else evt.cuda_time)
            names.add(re.search(r'rt_atoms_kernel<[^>]*>', evt.name).group(0) if '<' in evt.name else 'rt_atoms_kernel')
    eng.close()
    if not times:
        return None, None
    return float(np.mean(times)) / 1e3, sorted(names)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--streams', type=int, nargs='*', default=[1, 8, 64, 256, 1024])
    ap.add_argument('--inference', type=int, nargs='*', default=[0, 10])
    ap.add_argument('--blocks', type=int, default=400)
    ap.add_argument('--warmup', type=int, default=50)
    ap.add_argument('--singles-max', type=int, default=64)
    ap.add_argument('--K', type=int, default=1024)
    ap.add_argument('--N', type=int, default=512)
    ap.add_argument('--hop', type=int, default=128)
    ap.add_argument('--D', type=int, default=64)
    ap.add_argument('--json', default=None)
    args = ap.parse_args()
    import torch
    name = torch.cuda.get_device_name(0)
    power = card()
    K, N, hop, D, nT = args.K, args.N, args.hop, args.D, 1
    B, F = hop * nT, N // 2 + 1
    budget = B / 16000.0 * 1e3
    W, E, win = setup(K, N, D)
    print('card: %s | nvidia-smi name, power limit: %s' % (name, power), flush=True)
    print('%d-FFT hop %d K=%d D=%d, %d frame per block, block period %.1f ms' % (N, hop, K, D, nT, budget), flush=True)
    results = []
    for inf in args.inference:
        fits = 0
        for S in args.streams:
            x = audio(S, B, 32)
            dev, wall = run_multi(W, E, win, hop, B, nT, S, inf, args.blocks, args.warmup, x)
            r = {'S': S, 'inference': inf, 'device': pct(dev), 'wall': pct(wall), 'us_per_stream_device_p50': pct(dev)['p50_ms'] * 1e3 / S}
            if S <= args.singles_max:
                sd, sw = run_singles(W, E, win, hop, B, nT, S, inf, max(args.blocks // 4, 50), 10, x)
                r['singles'] = {'device_sum': pct(sd), 'wall': pct(sw)}
            ms, kern = atoms_kernel_ms(W, E, win, hop, B, nT, S, inf, x)
            if ms:
                tflops = 2.0 * S * nT * D * F * K / (ms * 1e-3) / 1e12
                r['atoms'] = {'kernel': kern, 'ms': ms, 'tflops': tflops, 'fraction_of_fp32_peak': tflops / FP32_PEAK_TFLOPS}
            if r['wall']['p99_ms'] <= budget:
                fits = max(fits, S)
            results.append(r)
            line = ('inference %2d S=%5d: device p50 %.3f p99 %.3f ms, wall p50 %.3f p99 %.3f ms, %.2f us/stream' % (
                inf, S, r['device']['p50_ms'], r['device']['p99_ms'], r['wall']['p50_ms'], r['wall']['p99_ms'], r['us_per_stream_device_p50']))
            if 'singles' in r:
                line += ' | %d single engines: device sum p50 %.3f ms, wall p50 %.3f ms' % (S, r['singles']['device_sum']['p50_ms'], r['singles']['wall']['p50_ms'])
            if 'atoms' in r:
                line += ' | atoms %.3f ms %.1f TFLOP/s (%.0f %% of %.0f) %s' % (ms, r['atoms']['tflops'], 100 * r['atoms']['fraction_of_fp32_peak'],
                                                                             FP32_PEAK_TFLOPS, ','.join(kern))
            print(line, flush=True)
        print('inference %d: largest S with p99 wall <= %.1f ms: %d' % (inf, budget, fits), flush=True)
        results.append({'inference': inf, 'largest_S_within_block_period': fits})
    if args.json:
        json.dump({'card': name, 'nvidia_smi': power, 'results': results}, open(args.json, 'w'), indent=1)


if __name__ == '__main__':
    main()
