"""Offline flows that follow a moving talker (localizationWindow): device time of the tracked flow against the static flow, and of the
window kernels (gccnmf_window_targets) alone.

    python tools/offline_tracking.py [--rounds 5] [--json out.json]

Flows, each as the one-call fused form (run_fused) and the Python stage form (separate / enhance), static and with w = 64,
alternating static and tracked within each round, median over rounds:
  configs[0] shape: separation into 3 sources of the shipped 1 min recording, N 1024, hop 512, K 128, 64 TDOAs, 100 iterations;
  configs[1] shape: enhancement of 30 s synthetic stereo, N 1024, hop 256, K 1024, 64 TDOAs, 100 iterations.
Window kernels: a random (64, T) angular spectrogram at T = 1872 (configs[1]) and T = 18747 (configs[3]'s length), w in
{6, 64, 1024, T}, P in {1, 3}, events around 20 calls (5 at w = T: each output then adds up to T terms in sequence).  The card's name and power limit come from the same run.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from klnmf_batch import events_ms  # noqa: E402
from rt_streams import card  # noqa: E402

SR = 16000


def flows(h, rounds):
    from gcc_nmf_b200.pipeline import GCCNMFPipeline
    from gcc_nmf_b200.synth import synthetic_stereo
    from gcc_nmf_b200.wavio import wavread
    rec, sr = wavread(os.path.join(ROOT, 'tests', 'golden', 'dev1_female3_liverec_130ms_1m_mix.wav'))
    settings = [('configs[0] separation, 3 sources', GCCNMFPipeline(sr, 1024, 512, 64, 1.0, 128, 100, handle=h),
                 np.ascontiguousarray(np.asarray(rec, np.float32)[:2]), 3),
                ('configs[1] enhancement', GCCNMFPipeline(SR, 1024, 256, 64, 0.1, 1024, 100, handle=h), synthetic_stereo(30.0, SR, seed=1234), 0)]
    rows = []
    for label, pipe, x, S in settings:
        xd = h.to_device(x)
        python = (lambda w: pipe.separate(xd, S, localizationWindow=w)) if S else (lambda w: pipe.enhance(xd, localizationWindow=w))
        forms = {'fused': lambda w: pipe.run_fused(xd, S, localizationWindow=w), 'python': python}
        for form, run in forms.items():
            run(None)
            run(64)
            times = {None: [], 64: []}
            for _ in range(rounds):
                for w in (None, 64):
                    times[w].append(events_ms(lambda: run(w)))
            static, tracked = float(np.median(times[None])), float(np.median(times[64]))
            rows.append(dict(setting=label, form=form, frames=pipe.num_frames(x.shape[1]), static_ms=static, tracked_ms=tracked,
                             overhead_ms=tracked - static, ratio=tracked / static))
            print('%-34s %-6s T %5d  static %8.3f ms  tracked (w 64) %8.3f ms  (%+.3f ms, x%.4f)' % (
                label, form, rows[-1]['frames'], static, tracked, tracked - static, tracked / static), flush=True)
    return rows


def window_kernels(h):
    rng = np.random.default_rng(0)
    rows = []
    for T in (1872, 18747):
        ang = h.to_device(rng.standard_normal((64, T)))
        for w in (6, 64, 1024, T):
            for P in (1, 3):
                h.window_targets(ang, w, P)
                ms = events_ms(lambda: h.window_targets(ang, w, P), reps=5 if w == T else 20)
                rows.append(dict(D=64, T=T, w=w, P=P, ms=ms))
                print('window_targets D 64  T %5d  w %5d  P %d  %8.3f ms' % (T, w, P, ms), flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--json')
    args = ap.parse_args()
    from gcc_nmf_b200._lib import default_handle
    h = default_handle()
    gpu = card()
    print('card:', gpu, flush=True)
    out = dict(card=gpu, window_kernels=window_kernels(h), flows=flows(h, args.rounds))
    if args.json:
        with open(args.json, 'w') as f:
            json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
