"""Per-launch latency of the low-latency engine with a bank of steering tables (LowLatencyEngine(expJOmegaTau=[...]),
gccnmf_llbank_*) at the BASELINE.json configs[4] shape of tools/ll_streams.py: 1024-sample asymmetric analysis window (m = 64), hop
64, K = 256, D = 128, 'windowed' synthesis, no inference, one hop per call, so one graph launch per 4 ms of audio at 16 kHz.

    python tools/ll_bank.py [--streams 1 64 256 1024] [--sources 0 4] [--calls 200] [--warmup 20] [--json out.json]

For every S and P, device time (CUDA events on the engine's stream around the launches of a call) and wall time (host, launch to the
synchronised output in pinned memory), p50 / p99, and whether the wall p99 fits the hop, of:
  plain      the plain engine (one table)
  bank1      a one-entry bank holding that table
  bank8      one bank of 8 tables (0.05 .. 1 m) with the streams spread over them unsorted (S >= 8)
  plain8     8 plain engines, one per table, S / 8 streams each, their graphs launched back to back (S >= 8)
Dictionaries are random; the audio is synthetic.  The card's name and power limit come from the same run.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(os.path.dirname(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from ll_streams import D, HOP, SR, audio, setup, timed  # noqa: E402
from rt_streams import card, pct  # noqa: E402

SPACINGS = [0.05, 0.1, 0.2, 0.3, 0.45, 0.6, 0.8, 1.0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--streams', type=int, nargs='+', default=[1, 64, 256, 1024])
    ap.add_argument('--sources', type=int, nargs='+', default=[0, 4])
    ap.add_argument('--calls', type=int, default=200)
    ap.add_argument('--warmup', type=int, default=20)
    ap.add_argument('--json', default=None)
    a = ap.parse_args()
    import torch
    from gcc_nmf_b200 import gccNMFFunctions as fn
    from gcc_nmf_b200.lowlatency import LowLatencyEngine
    W, E, win, syn = setup()
    F = W.shape[0]
    tables = [fn.getExpJOmegaTau(fn.getFrequenciesInHz(SR, F), fn.getTDOAsInSeconds(d, D)) for d in SPACINGS]
    hop_ms = HOP * 1e3 / SR
    rows = []

    def make(S, P, E):
        return LowLatencyEngine(W, E, win, syn, HOP, numStreams=S, synthesis='windowed', targetTDOAEpsilon=0.05 * D, numSources=P)

    def run(name, S, P, engines, x):
        dev, wall = timed(engines, x, a.calls, a.warmup)
        row = {'form': name, 'S': S, 'P': P, 'device': pct(dev), 'wall': pct(wall), 'wall_p99_fits_hop': pct(wall)['p99_ms'] <= hop_ms}
        rows.append(row)
        print(json.dumps(row), flush=True)
        for e in engines:
            e.close()
        torch.cuda.empty_cache()

    for P in a.sources:
        for S in a.streams:
            x = audio(S, a.calls)
            run('plain', S, P, [make(S, P, E)], x)
            run('bank1', S, P, [make(S, P, [E])], x)
            if S >= 8:
                eng = make(S, P, tables)
                eng.assign_steering(None, np.random.RandomState(0).permutation(np.arange(S) % 8))
                run('bank8', S, P, [eng], x)
                run('plain8', S, P, [make(S // 8, P, t) for t in tables], x)
    result = {'card': card(), 'shape': dict(N=1024, m=64, hop=HOP, K=256, D=D, C=1, sr=SR, synthesis='windowed', inference=0), 'rows': rows}
    print(json.dumps({'card': result['card']}), flush=True)
    if a.json:
        with open(a.json, 'w') as f:
            json.dump(result, f, indent=1)


if __name__ == '__main__':
    main()
