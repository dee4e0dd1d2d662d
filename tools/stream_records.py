"""Cost of moving low-latency streams (LowLatencyEngine.save_streams / load_streams, gccnmf_llrec_*) at the BASELINE.json configs[4]
shape (1024-sample asymmetric window, m = 64, hop 64, K = 256, D = 128, one hop per call; a hop is 4 ms at 16 kHz).

    python tools/stream_records.py [--streams 1 64 1024] [--reps 50] [--json out.json]
    python tools/stream_records.py --process-libs A.so B.so [--rounds 4] [--calls 300]

First mode: for S streams in one engine (all of them saved, then loaded back into the same slots), per save and per load:
  device   CUDA events on the engine's stream around the C entry (the read-back of the synthesis weights, the copy kernel and the
           host copy);
  wall     host clock around the C entry and a synchronise of the stream, into a pinned record allocated once;
  python   host clock around save_streams / load_streams (which also allocate the pinned record, for a save).
p50 / p99 over --reps, with the record size.  Second mode: the device p50 per graph launch of `process` at S = 1 and 1024, each
library in a process of its own, alternating A, B, A, B ... for --rounds, so that two builds are compared in one session.  The
card's name and power limit come from the same run.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from ll_streams import HOP, audio, setup, timed  # noqa: E402
from rt_streams import card, pct  # noqa: E402


def _engine(S):
    from gcc_nmf_b200.lowlatency import LowLatencyEngine
    W, E, win, syn = setup()
    return LowLatencyEngine(W, E, win, syn, HOP, numStreams=S, synthesis='windowed', targetTDOAEpsilon=6.4)


def records(a):
    import torch
    rows = []
    for S in a.streams:
        eng = _engine(S)
        x = audio(S, 20)
        for c in range(20):
            eng.process(x[:, :, c * HOP:(c + 1) * HOP])
        rec = eng.save_streams()
        n = int(eng.h.lib.gccnmf_llrec_workspace_bytes(ctypes.byref(eng.cfg), eng.P, S))
        ws = torch.empty(n, dtype=torch.uint8, device=eng.h.device)
        st = eng.stream
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        row = {'S': S, 'record_bytes': eng.record_bytes}
        for name in ('save_streams', 'load_streams'):
            fn = getattr(eng.h.lib, 'gccnmf_llrec_' + name)
            dev, wall, py = [], [], []
            for i in range(a.warmup + a.reps):
                t0 = time.perf_counter()
                e0.record(st)
                eng.h.check(fn(eng.h.h, ctypes.byref(eng.cfg), eng.P, eng.state.data_ptr(), eng.state_bytes, 0, S, rec.data.data_ptr(),
                               rec.data.numel(), ws.data_ptr(), n, st.cuda_stream))
                e1.record(st)
                st.synchronize()
                t1 = time.perf_counter()
                if name == 'save_streams':
                    eng.save_streams()
                else:
                    eng.load_streams(range(S), rec)
                t2 = time.perf_counter()
                if i >= a.warmup:
                    dev.append(e0.elapsed_time(e1))
                    wall.append((t1 - t0) * 1e3)
                    py.append((t2 - t1) * 1e3)
            row[name.split('_')[0]] = {'device': pct(dev), 'wall': pct(wall), 'python': pct(py)}
        rows.append(row)
        print(json.dumps(row), flush=True)
        eng.close()
        del eng, ws, rec
        torch.cuda.empty_cache()
    return rows


def process_child(lib, streams, calls, warmup):
    from gcc_nmf_b200 import _lib
    _lib.LIB_PATH = os.path.abspath(lib)
    exported = ctypes.CDLL(_lib.LIB_PATH)
    for name in [n for n in _lib.SIGNATURES if not hasattr(exported, n)]:     # an older build lacks the newer entries
        del _lib.SIGNATURES[name]
    out = {}
    for S in streams:
        eng = _engine(S)
        dev, _ = timed([eng], audio(S, calls), calls, warmup)
        out[S] = pct(dev)['p50_ms']
        eng.close()
    print(json.dumps(out))


def process_compare(a):
    runs = {lib: {str(S): [] for S in (1, 1024)} for lib in a.process_libs}
    for r in range(a.rounds):
        for lib in a.process_libs:
            p = subprocess.run([sys.executable, os.path.abspath(__file__), '--process-child', lib, '--calls', str(a.calls)], capture_output=True,
                               text=True)
            if p.returncode != 0:
                raise RuntimeError('%s: %s' % (lib, p.stderr[-2000:]))
            for S, v in json.loads(p.stdout.strip().splitlines()[-1]).items():
                runs[lib][S].append(v)
            print(json.dumps({'round': r, 'lib': lib, 'p50_ms': json.loads(p.stdout.strip().splitlines()[-1])}), flush=True)
    return {lib: {S: {'p50_ms_per_round': v, 'median_ms': float(np.median(v))} for S, v in d.items()} for lib, d in runs.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--streams', type=int, nargs='+', default=[1, 64, 1024])
    ap.add_argument('--reps', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--process-libs', nargs='+', default=None)
    ap.add_argument('--process-child', default=None)
    ap.add_argument('--rounds', type=int, default=4)
    ap.add_argument('--calls', type=int, default=300)
    ap.add_argument('--json', default=None)
    a = ap.parse_args()
    if a.process_child:
        return process_child(a.process_child, (1, 1024), a.calls, 30)
    result = {'card': card(), 'shape': dict(N=1024, m=64, hop=HOP, K=256, D=128, C=1, sr=16000)}
    if a.process_libs:
        result['process'] = process_compare(a)
    else:
        result['records'] = records(a)
    print(json.dumps({'card': result['card']}), flush=True)
    if a.json:
        with open(a.json, 'w') as f:
            json.dump(result, f, indent=1)


if __name__ == '__main__':
    main()
