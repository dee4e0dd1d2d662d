"""Cost of moving real-time slots (save_streams / load_streams of MultiStreamRealtimeEngine, gccnmf_rtrec_*) at the BASELINE.json
configs[2] shape (512-FFT, hop 128, B 128, one frame per block, D 64, history 128, K 1024).

    python tools/rt_records.py [--streams 1 64 1024] [--sources 0 4] [--reps 30] [--json out.json]
    python tools/rt_records.py --process-libs A.so B.so [--rounds 4] [--blocks 300]

First mode: for S slots, P sources and two banks -- one entry (Qd = Qe = 1) and 64 dictionaries of K 1024 (Qe = 1) -- all S slots
saved, then loaded back into the same slots, per save and per load:
  device   CUDA events on the engine's stream around the C entry (digest kernels, copy kernel, copies; a load's one wait included);
  wall     host clock around the C entry and a synchronise of the stream, into a pinned record allocated once;
  python   host clock around save_streams / load_streams (a save also allocates its pinned record; a load checks every header);
p50 / p99 over --reps, with the record size.  Then, in a separate torch.profiler run of one save and one load, the device time of
the digest kernels, the copy kernel, the sort and the copies.  Second mode: the device p50 per graph launch of `process_blocks` at
S = 1 and 1024 with 0 and 10 inference iterations, each library in a process of its own, alternating A, B, A, B ... for --rounds,
so that two builds are compared in one session.  The card's name and power limit come from the same run.
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

from rt_streams import audio, card, pct, setup  # noqa: E402

N, HOP, B, NT, D, HIST, K = 512, 128, 128, 1, 64, 128, 1024
BANKS = {'one entry': 1, '64 dictionaries of K 1024': 64}


def _engine(S, P, Qd, inference=0):
    from gcc_nmf_b200.realtime.multistream import MultiStreamRealtimeEngine
    W, E, win = setup(K, N, D)
    Ws = [W] + [(np.random.default_rng(i).random(W.shape) ** 3).astype(np.float32) for i in range(1, Qd)]
    return MultiStreamRealtimeEngine(Ws, [E], win, win, HOP, B, NT, S, historyLength=HIST, numInferenceIterations=inference, numSources=P)


def _c_call(eng, name, S, rec, ws, n):
    return getattr(eng.h.lib, 'gccnmf_rtrec_' + name)(eng.h.h, ctypes.byref(eng.cfg), *eng._record_dims, eng.state.data_ptr(), eng.state_bytes, 0,
                                                       S, rec.data.data_ptr(), rec.data.numel(), ws.data_ptr(), n, eng.stream.cuda_stream)


def _split(eng, S, rec, ws, n):
    """Device microseconds per category of one save and of one load, from torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    out = {}
    for name in ('save_slots', 'load_slots'):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            eng.h.check(_c_call(eng, name, S, rec, ws, n))
            eng.stream.synchronize()
            torch.cuda.synchronize()
        split = out[name.split('_')[0]] = {}
        for evt in prof.events():
            if evt.device_type != torch.autograd.DeviceType.CUDA:
                continue
            t = evt.device_time if hasattr(evt, 'device_time') else evt.cuda_time
            key = ('digest kernels' if 'rt_digest' in evt.name else 'copy kernel' if 'rt_record_copy' in evt.name
                   else 'sort' if 'sort_by_entry' in evt.name else 'copies' if 'Memcpy' in evt.name or 'memcpy' in evt.name else evt.name)
            split[key] = round(split.get(key, 0.0) + t, 2)
    return out


def records(a):
    import torch
    rows = []
    for bank, Qd in BANKS.items():
        for P in a.sources:
            for S in a.streams:
                eng = _engine(S, P, Qd)
                eng.assign(range(S), [s % Qd for s in range(S)], 0)
                x = audio(S, B, 12)
                for b in range(12):
                    eng.process_blocks(x[b])
                rec = eng.save_streams()
                n = int(eng.h.lib.gccnmf_rtrec_workspace_bytes(ctypes.byref(eng.cfg), *eng._record_dims, S))
                ws = torch.empty(n, dtype=torch.uint8, device=eng.h.device)
                st = eng.stream
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                row = {'bank': bank, 'S': S, 'P': P, 'record_bytes': eng.record_bytes}
                for name in ('save_slots', 'load_slots'):
                    dev, wall, py = [], [], []
                    for i in range(a.warmup + a.reps):
                        t0 = time.perf_counter()
                        e0.record(st)
                        eng.h.check(_c_call(eng, name, S, rec, ws, n))
                        e1.record(st)
                        st.synchronize()
                        t1 = time.perf_counter()
                        if name == 'save_slots':
                            eng.save_streams()
                        else:
                            eng.load_streams(range(S), rec)
                        t2 = time.perf_counter()
                        if i >= a.warmup:
                            dev.append(e0.elapsed_time(e1))
                            wall.append((t1 - t0) * 1e3)
                            py.append((t2 - t1) * 1e3)
                    row[name.split('_')[0]] = {'device': pct(dev), 'wall': pct(wall), 'python': pct(py)}
                row['profile_us'] = _split(eng, S, rec, ws, n)
                rows.append(row)
                print(json.dumps(row), flush=True)
                eng.close()
                del eng, ws, rec
                torch.cuda.empty_cache()
    return rows


def process_child(lib, blocks, warmup):
    import torch
    from gcc_nmf_b200 import _lib
    _lib.LIB_PATH = os.path.abspath(lib)
    exported = ctypes.CDLL(_lib.LIB_PATH)
    for name in [n for n in _lib.SIGNATURES if not hasattr(exported, n)]:     # an older build lacks the newer entries
        del _lib.SIGNATURES[name]
    from gcc_nmf_b200.realtime.multistream import MultiStreamRealtimeEngine
    W, E, win = setup(K, N, D)
    out = {}
    for inference in (0, 10):
        for S in (1, 1024):
            eng = MultiStreamRealtimeEngine(W, E, win, win, HOP, B, NT, S, historyLength=HIST, numInferenceIterations=inference)
            eng.set_params(range(S), targetTDOAIndex=10.0, epsilon=5.0, beta=2.0, localizationEnabled=True)
            x = audio(S, B, 16)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            dev = []
            for b in range(warmup + blocks):
                eng.in_host.numpy()[:] = x[b % 16]
                e0.record(eng.stream)
                eng.h.check(eng.h.lib.gccnmf_rt_graph_launch(eng.h.h, eng.build_graph(), eng.stream.cuda_stream))
                e1.record(eng.stream)
                eng.stream.synchronize()
                if b >= warmup:
                    dev.append(e0.elapsed_time(e1))
            out['S%d_inf%d' % (S, inference)] = pct(dev)['p50_ms']
            eng.close()
    print(json.dumps(out))


def process_compare(a):
    runs = {lib: {} for lib in a.process_libs}
    for r in range(a.rounds):
        for lib in a.process_libs:
            p = subprocess.run([sys.executable, os.path.abspath(__file__), '--process-child', lib, '--blocks', str(a.blocks)], capture_output=True,
                               text=True)
            if p.returncode != 0:
                raise RuntimeError('%s: %s' % (lib, p.stderr[-2000:]))
            got = json.loads(p.stdout.strip().splitlines()[-1])
            for k, v in got.items():
                runs[lib].setdefault(k, []).append(v)
            print(json.dumps({'round': r, 'lib': lib, 'p50_ms': got}), flush=True)
    return {lib: {k: {'p50_ms_per_round': v, 'median_ms': float(np.median(v))} for k, v in d.items()} for lib, d in runs.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--streams', type=int, nargs='+', default=[1, 64, 1024])
    ap.add_argument('--sources', type=int, nargs='+', default=[0, 4])
    ap.add_argument('--reps', type=int, default=30)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--process-libs', nargs='+', default=None)
    ap.add_argument('--process-child', default=None)
    ap.add_argument('--rounds', type=int, default=4)
    ap.add_argument('--blocks', type=int, default=300)
    ap.add_argument('--json', default=None)
    a = ap.parse_args()
    if a.process_child:
        return process_child(a.process_child, a.blocks, 30)
    result = {'card': card(), 'shape': dict(N=N, hop=HOP, B=B, nT=NT, D=D, history=HIST, K=K, sr=16000)}
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
