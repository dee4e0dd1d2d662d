"""Per-launch latency of the low-latency engine with a localisation window (LowLatencyEngine(historyLength=1024), gccnmf_llhist_*) at
the BASELINE.json configs[4] shape of tools/ll_streams.py: 1024-sample asymmetric analysis window (m = 64), hop 64, K = 256, D = 128,
'windowed' synthesis, no inference, one hop per call, so one graph launch per 4 ms of audio at 16 kHz.

    python tools/ll_window.py [--streams 1 64 256 1024] [--windows 0 6 64 256 1024] [--sources 0 4] [--history 1024]
                              [--calls 200] [--warmup 20] [--json out.json]

For every S, P and window w (every stream on w; w = 0 is the running maximum): device time (CUDA events on the engine's stream
around each graph launch) and wall time (host, launch to the synchronised output in pinned memory), p50 / p99, and whether the wall
p99 fits the hop; then per S and P the largest w whose wall p99 fits.  At the largest S, the targets kernel alone
(ll_hist_targets_kernel / ll_hist_src_targets_kernel, torch.profiler over kernel-by-kernel calls) for every w.  Dictionaries are
random; the audio is synthetic.  The card's name and power limit come from the same run.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.abspath(os.path.dirname(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from ll_streams import D, HOP, SR, audio, setup, timed  # noqa: E402
from rt_streams import card, pct  # noqa: E402


def kernel_us(eng, x, calls, names=('ll_hist_targets_kernel', 'll_hist_src_targets_kernel', 'll_targets_kernel', 'll_src_targets_kernel')):
    """Mean device time of the targets kernel over `calls` kernel-by-kernel calls (torch.profiler)."""
    from torch.profiler import ProfilerActivity, profile
    n = x.shape[2] // HOP
    for c in range(3):
        eng.process(x[:, :, c * HOP:(c + 1) * HOP], use_graph=False)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for c in range(calls):
            eng.process(x[:, :, (c % n) * HOP:(c % n + 1) * HOP], use_graph=False)
    times = [e.device_time_total / e.count for e in prof.key_averages() if any(k in e.key for k in names) and e.count]
    return float(times[0]) if times else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--streams', type=int, nargs='+', default=[1, 64, 256, 1024])
    ap.add_argument('--windows', type=int, nargs='+', default=[0, 6, 64, 256, 1024])
    ap.add_argument('--sources', type=int, nargs='+', default=[0, 4])
    ap.add_argument('--history', type=int, default=1024)
    ap.add_argument('--calls', type=int, default=200)
    ap.add_argument('--warmup', type=int, default=20)
    ap.add_argument('--profile-calls', type=int, default=20)
    ap.add_argument('--json', default=None)
    a = ap.parse_args()
    import torch
    from gcc_nmf_b200.lowlatency import LowLatencyEngine
    W, E, win, syn = setup()
    hop_ms = HOP * 1e3 / SR
    rows, fits, kernels = [], [], []
    for P in a.sources:
        for S in a.streams:
            x = audio(S, a.calls)
            eng = LowLatencyEngine(W, E, win, syn, HOP, numStreams=S, synthesis='windowed', targetTDOAEpsilon=0.05 * D, numSources=P,
                                   historyLength=a.history)
            best = None
            for w in a.windows:
                eng.set_localization(None, w)
                dev, wall = timed([eng], x, a.calls, a.warmup)
                row = {'S': S, 'P': P, 'window': w, 'history': a.history, 'device': pct(dev), 'wall': pct(wall),
                       'wall_p99_fits_hop': pct(wall)['p99_ms'] <= hop_ms}
                if row['wall_p99_fits_hop']:
                    best = w
                if S == max(a.streams):
                    row['targets_kernel_us'] = kernel_us(eng, x, a.profile_calls)
                    kernels.append({'S': S, 'P': P, 'window': w, 'targets_kernel_us': row['targets_kernel_us']})
                rows.append(row)
                print(json.dumps(row), flush=True)
            fits.append({'S': S, 'P': P, 'largest_window_with_wall_p99_within_hop': best, 'hop_ms': hop_ms})
            print(json.dumps(fits[-1]), flush=True)
            eng.close()
            del eng
            torch.cuda.empty_cache()
    result = {'card': card(), 'shape': dict(N=1024, m=64, hop=HOP, K=256, D=D, C=1, sr=SR, synthesis='windowed', inference=0),
              'rows': rows, 'fits': fits, 'targets_kernel': kernels}
    print(json.dumps({'card': result['card'], 'fits': fits, 'targets_kernel': kernels}), flush=True)
    if a.json:
        with open(a.json, 'w') as f:
            json.dump(result, f, indent=1)


if __name__ == '__main__':
    main()
