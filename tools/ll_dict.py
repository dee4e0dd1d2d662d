"""Per-launch latency of the low-latency engine with a bank of dictionaries (LowLatencyEngine(W=[...]), gccnmf_lldict_*) at the
BASELINE.json configs[4] shape of tools/ll_streams.py: 1024-sample asymmetric analysis window (m = 64), hop 64, K_max = 256, D = 128,
'windowed' synthesis, no inference, one hop per call, so one graph launch per 4 ms of audio at 16 kHz.

    python tools/ll_dict.py [--streams 1 64 256 1024] [--sources 0 4] [--calls 200] [--warmup 20] [--json out.json]
                            [--ab-tree PARENT_CHECKOUT --ab-rounds 3]

For every S and P, device time (CUDA events on the engine's stream around the launches of a call) and wall time (host, launch to the
synchronised output in pinned memory), p50 / p99, and whether the wall p99 fits the hop, of:
  plain      the plain engine (K = 256)
  dict1      a one-entry dictionary bank holding that dictionary
  dict6      one bank of 6 dictionaries (K 64 / 128 / 256, two contents each) with the streams spread over them unsorted (S >= 6)
  plain6     6 plain engines, one per dictionary, S / 6 streams each, their graphs launched back to back (S >= 6)
With --ab-tree, the plain engine is also timed from another built checkout of the project (e.g. the parent commit's, built there
with `python gcc-nmf_b200/build.py`), alternating the two trees in child processes of this script, --ab-rounds times per S and P.
Dictionaries are random; the audio is synthetic.  The card's name and power limit come from the same run.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(os.path.dirname(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from ll_streams import D, HOP, SR, audio, setup, timed  # noqa: E402
from rt_streams import card, pct  # noqa: E402

ATOMS = [64, 64, 128, 128, 256, 256]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--streams', type=int, nargs='+', default=[1, 64, 256, 1024])
    ap.add_argument('--sources', type=int, nargs='+', default=[0, 4])
    ap.add_argument('--calls', type=int, default=200)
    ap.add_argument('--warmup', type=int, default=20)
    ap.add_argument('--forms', nargs='+', default=['plain', 'dict1', 'dict6', 'plain6'])
    ap.add_argument('--tree', default=None, help='import the engine from this built checkout instead of this one')
    ap.add_argument('--ab-tree', default=None)
    ap.add_argument('--ab-rounds', type=int, default=3)
    ap.add_argument('--json', default=None)
    a = ap.parse_args()
    if a.tree:
        sys.path.insert(0, os.path.abspath(a.tree))
        for m in [m for m in sys.modules if m == 'gcc_nmf_b200' or m.startswith('gcc_nmf_b200.')]:
            del sys.modules[m]
    import torch
    from gcc_nmf_b200.lowlatency import LowLatencyEngine
    W, E, win, syn = setup()
    F = W.shape[0]
    rng = np.random.default_rng(1)
    dicts = [W if k == 256 and i == 4 else (rng.random((F, k)) ** 3 + 1e-3).astype(np.float32) for i, k in enumerate(ATOMS)]
    hop_ms = HOP * 1e3 / SR
    rows = []

    def make(S, P, W_):
        return LowLatencyEngine(W_, E, win, syn, HOP, numStreams=S, synthesis='windowed', targetTDOAEpsilon=0.05 * D, numSources=P)

    def run(name, S, P, engines, x):
        dev, wall = timed(engines, x, a.calls, a.warmup)
        row = {'form': name, 'S': S, 'P': P, 'device': pct(dev), 'wall': pct(wall), 'wall_p99_fits_hop': pct(wall)['p99_ms'] <= hop_ms}
        if a.tree:
            row['tree'] = a.tree
        rows.append(row)
        print(json.dumps(row), flush=True)
        for e in engines:
            e.close()
        torch.cuda.empty_cache()

    for P in a.sources:
        for S in a.streams:
            x = audio(S, a.calls)
            if 'plain' in a.forms:
                run('plain', S, P, [make(S, P, W)], x)
            if 'dict1' in a.forms:
                run('dict1', S, P, [make(S, P, [W])], x)
            if S >= 6 and 'dict6' in a.forms:
                eng = make(S, P, dicts)
                eng.assign_dictionary(None, np.random.RandomState(0).permutation(np.arange(S) % 6))
                run('dict6', S, P, [eng], x)
            if S >= 6 and 'plain6' in a.forms:
                run('plain6', S, P, [make(S // 6, P, w) for w in dicts], x[:S // 6 * 6])
            if a.ab_tree:
                for r in range(a.ab_rounds):
                    for tree in (a.ab_tree, None):          # alternate: the other tree, then this one
                        cmd = [sys.executable, os.path.abspath(__file__), '--streams', str(S), '--sources', str(P), '--forms', 'plain',
                               '--calls', str(a.calls), '--warmup', str(a.warmup)] + (['--tree', tree] if tree else [])
                        out = subprocess.run(cmd, capture_output=True, text=True, check=True).stdout
                        row = [json.loads(line) for line in out.splitlines() if line.startswith('{"form"')][0]
                        row.update(form='ab_plain', tree=tree or 'this', round=r)
                        rows.append(row)
                        print(json.dumps(row), flush=True)
    result = {'card': card(), 'shape': dict(N=1024, m=64, hop=HOP, K_max=256, D=D, C=1, sr=SR, synthesis='windowed', inference=0), 'rows': rows}
    print(json.dumps({'card': result['card']}), flush=True)
    if a.json:
        with open(a.json, 'w') as f:
            json.dump(result, f, indent=1)


if __name__ == '__main__':
    main()
