"""Run under torchrun on >= 2 GPUs (not collected by pytest: needs NCCL + several devices):

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29511 tests/multi_gpu_check.py

Checks that the frame-sharded enhancement pipeline (joint dictionary, one all-reduce per KL-NMF
iteration, iSTFT seam exchange) reproduces the single-GPU pipeline run on the whole recording.

With --pull-forms it instead runs distributed.klnmf_sharded_pull in every form of the pull exchange the ranks agree on, on a
synthetic V whose frame count does not divide evenly (the ranks have different T2 and row-sum slot counts), and checks each
rank's H slice and W element by element against a float64 run of the joint problem (the bars of tests/test_gpu_klnmf.py), W
bit-identical across ranks, and the direct forms 0 and 1 and form 2 bit-identical to each other: they add the numerator in rank
order and the row sums rank-major within each of the W update's 8 strided groups."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def pull_forms(local, rank, world):
    from test_gpu_klnmf import BOUNDS, atom_error, klnmf64, tile_plan
    from oracle import gccnmf_oracle as orc
    from gcc_nmf_b200 import distributed as d
    from gcc_nmf_b200._lib import default_handle
    h = default_handle(local)
    sm = torch.cuda.get_device_properties(h.device).multi_processor_count
    F, K, T, iters = 263, 72, 257, 3          # 257 frames per channel: 129 + 128 at 2 ranks, T2 = 258 and 256
    rng = np.random.default_rng(7)
    V = (rng.random((F, 2 * T)) ** 3 + 1e-3).astype(np.float32)
    W0, H0 = orc.initKLNMF(F, 2 * T, K)
    ref = klnmf64(V, W0, H0, (iters,))[iters]
    t0, t1 = d.shard_frames(T, world, rank)
    cols = np.r_[t0:t1, T + t0:T + t1]
    Vs, H0s = np.ascontiguousarray(V[:, cols]), np.ascontiguousarray(H0[:, cols])
    T2 = Vs.shape[1]
    layout_T2 = 2 * max(b - a for a, b in (d.shard_frames(T, world, r) for r in range(world)))
    level = torch.tensor([(h.lib.gccnmf_klnmf_pull_supported(h.h, F, T2, K) >> b) & 1 for b in range(3)], dtype=torch.int32, device=h.device)
    dist.all_reduce(level, op=dist.ReduceOp.MIN)
    level = sum(int(v) << b for b, v in enumerate(level.tolist()))
    forms = [(f, dr) for f, dr in [(0, True), (0, False), (1, True), (1, False), (2, False)] if level & 1 and (not dr or level & 2) and (f < 2 or level & 4)]
    print('rank %d: T2 %d, layout_T2 %d, row-sum slots %d, forms %s' % (rank, T2, layout_T2, tile_plan(h, sm, F, T2, K)[4], forms), flush=True)
    ok, out = True, {}
    for form, direct in forms:
        px = d.PullExchange.create(h.lib, F, layout_T2, K, h.device, None, two_shot=form)
        assert px is not None, 'no peer-mapped symmetric buffer'
        px.direct = direct
        Vd, W, H = h.to_device(Vs), h.to_device(W0.copy()), h.to_device(H0s.copy())
        d.klnmf_sharded_pull(h, px, Vd, W, H, iters, 0.0, 1e-16)
        torch.cuda.synchronize()
        W, H = W.cpu().numpy(), H.cpu().numpy()
        eW, eH = atom_error(W, ref[0], 0), atom_error(H, ref[1][:, cols], 1)
        Ws = [None] * world
        dist.all_gather_object(Ws, W)
        same = all(np.array_equal(Ws[0], w) for w in Ws)
        good = eW <= BOUNDS[iters, 'W'] and eH <= BOUNDS[iters, 'H'] and same
        print('rank %d form %d %s: W %.3e H %.3e (bars %.1e %.1e), W identical across ranks: %s' % (
            rank, form, 'direct' if direct else 'packed', eW, eH, BOUNDS[iters, 'W'], BOUNDS[iters, 'H'], same), flush=True)
        ok &= good
        out[form, direct] = (W, H)
    same_order = [out[k] for k in [(0, True), (1, True), (2, False)] if k in out]
    for W, H in same_order[1:]:
        ok &= np.array_equal(W, same_order[0][0]) and np.array_equal(H, same_order[0][1])
    print('rank %d: %d forms with the same additions, bit-identical: %s' % (rank, len(same_order), ok), flush=True)
    verdict = torch.tensor([1 if ok else 0], dtype=torch.int32, device=h.device)
    dist.all_reduce(verdict, op=dist.ReduceOp.MIN)
    if rank == 0:
        print('PULL_FORMS_CHECK', 'PASS' if int(verdict.item()) == 1 else 'FAIL')


def main():
    local = int(os.environ.get('LOCAL_RANK', '0'))
    torch.cuda.set_device(local)
    dist.init_process_group('nccl', device_id=torch.device('cuda', local))
    rank, world = dist.get_rank(), dist.get_world_size()
    if '--pull-forms' in sys.argv:
        pull_forms(local, rank, world)
        dist.destroy_process_group()
        return
    from gcc_nmf_b200.distributed import ShardedGCCNMFPipeline
    from gcc_nmf_b200.pipeline import GCCNMFPipeline
    from gcc_nmf_b200.synth import synthetic_stereo
    cfg = dict(sampleRate=16000, windowSize=1024, hopSize=256, numTDOAs=64, microphoneSeparationInMetres=0.1,
               dictionarySize=256, numIterations=20)
    clip = 4.0
    sp = ShardedGCCNMFPipeline(device=local, clip_seconds=clip, **cfg)
    x_local = torch.from_numpy(sp.local_samples()).to(sp.h.device)
    r = sp.enhance(x_local)
    y_local = r['targetSignalEstimates'][0].cpu().numpy()
    sizes = [None] * world
    dist.all_gather_object(sizes, y_local.shape[1])
    ys = [None] * world
    dist.all_gather_object(ys, y_local)
    Ws = [None] * world
    dist.all_gather_object(Ws, r['W'].cpu().numpy())
    if rank == 0:
        full = np.concatenate([synthetic_stereo(clip, seed=1234 + c) for c in range(world)], axis=1)
        single = GCCNMFPipeline(device=local, handle=sp.h, **cfg)
        r1 = single.enhance(single.h.to_device(full))
        y1 = r1['targetSignalEstimates'][0].cpu().numpy()
        y = np.concatenate(ys, axis=1)
        W1 = r1['W'].cpu().numpy()

        def rel(a, b):
            return float(np.linalg.norm(a - b) / np.linalg.norm(b))
        print('collective:', sp.collective)
        print('world', world, 'frames', sp.total_frames, 'target', r['targetTDOAIndexes'], r1['targetTDOAIndexes'])
        print('W identical across ranks:', all(np.array_equal(Ws[0], w) for w in Ws))
        print('rel W sharded vs single: %.3e' % rel(Ws[0], W1))
        print('signal shape', y.shape, y1.shape, 'rel signal: %.3e' % rel(y, y1))
        ok = (y.shape == y1.shape and r['targetTDOAIndexes'] == r1['targetTDOAIndexes'] and rel(Ws[0], W1) < 1e-4)
        print('MULTI_GPU_CHECK', 'PASS' if ok else 'FAIL')
    dist.destroy_process_group()


if __name__ == '__main__':
    main()
