"""CPU, world_size 2, gloo: the host logic of the frame-sharded path (gcc-nmf_b200/distributed.py):
shard bookkeeping, sharded NMF init, the per-iteration all-reduce protocol and the iSTFT seam
exchange.  The three C-ABI building blocks are replaced by a test-only numpy stand-in that follows
the oracle's arithmetic, so what is under test is the sharding logic, not the kernels (those are
covered on the GPU by tests/test_gpu_parity.py::test_klnmf_building_blocks_equal_fused)."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import gccnmf_oracle as orc


class NumpyOps(object):
    """Stand-in for Handle.klnmf_begin / klnmf_step_numer / klnmf_step_apply / klnmf_end on CPU tensors
    (gccNMFFunctions.py:76, :77 numerator, :77-81 apply)."""

    @staticmethod
    def klnmf_begin(V, W, H):
        pass

    @staticmethod
    def klnmf_step_numer(V, W, H, iteration, numer, alpha, eps):
        Vn, Wn, Hn = V.numpy(), W.numpy(), H.numpy()
        Hn *= np.dot(Wn.T, Vn / np.dot(Wn, Hn)) / (np.sum(Wn, axis=0)[:, None] + np.float32(alpha) + np.float32(eps))
        F, K = Wn.shape
        numer.numpy()[:F * K] = np.dot(Vn / np.dot(Wn, Hn), Hn.T).ravel()
        numer.numpy()[F * K:] = np.sum(Hn, axis=1)

    @staticmethod
    def klnmf_step_apply(W, H, numer):
        Wn, Hn = W.numpy(), H.numpy()
        F, K = Wn.shape
        Wn *= numer.numpy()[:F * K].reshape(F, K) / numer.numpy()[F * K:]
        norms = np.sqrt(np.sum(Wn ** 2, 0))
        Wn /= norms
        Hn *= norms[:, None]

    @staticmethod
    def klnmf_end(W, H, iterations_done):
        pass


def _free_port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        from gcc_nmf_b200 import distributed as d
        comm = d.ShardComm()
        F, K, T, I = 33, 6, 37, 5
        rng = np.random.default_rng(0)
        Vfull = (rng.random((F, 2 * T)) + 0.05).astype(np.float32)      # [L frames | R frames]
        t0, t1 = d.shard_frames(T, world, rank)
        W0, H0s = d.sharded_nmf_init(F, T, K, 1e-16, 0, t0, t1)
        Vs = np.ascontiguousarray(np.concatenate([Vfull[:, t0:t1], Vfull[:, T + t0:T + t1]], axis=1))
        W, H = torch.from_numpy(W0.copy()), torch.from_numpy(H0s.copy())
        numer = torch.empty(F * K + K, dtype=torch.float32)
        d.klnmf_sharded(NumpyOps, comm, torch.from_numpy(Vs), W, H, I, 0.0, 1e-16, numer)
        # seam exchange: local un-trimmed overlap-adds of random frames must sum to the global one
        N, hop = 16, 4
        frames = np.random.default_rng(1).standard_normal((1, T, N)).astype(np.float32)
        y_local = torch.zeros(1, N + hop * (t1 - t0 - 1))
        for i in range(t0, t1):
            y_local[0, (i - t0) * hop:(i - t0) * hop + N] += torch.from_numpy(frames[0, i])
        y_owned = d.overlap_add_seams(comm, y_local, hop * (t1 - t0), N - hop)
        # cross-rank agreement helpers of the sharded pipeline (exchange form, buffer layout): AND over bits via MIN, MAX, MIN
        import types
        fake = types.SimpleNamespace(torch=torch, comm=comm, h=types.SimpleNamespace(device='cpu'))
        agree = (d.ShardedGCCNMFPipeline._all_and(fake, 7 if rank == 0 else 5), d.ShardedGCCNMFPipeline._all_max(fake, 10 + rank),
                 d.ShardedGCCNMFPipeline._all_min(fake, 3 - rank))
        out[rank] = dict(W=W.numpy().copy(), H=H.numpy().copy(), t=(t0, t1), y=y_owned.numpy().copy(), agree=agree)
    finally:
        dist.destroy_process_group()


class RecordingOps(object):
    """Stand-in for Handle.klnmf_begin / klnmf_step_pull / klnmf_end that records every call klnmf_sharded_pull makes."""

    def __init__(self):
        self.calls = []

    def klnmf_begin(self, V, W, H):
        self.calls.append(('begin', V, W, H))

    def klnmf_step_pull(self, V, W, H, iteration, epoch, rank, world, bases, layout_T2, two_shot, direct, sparsity_alpha=0.0, epsilon=1e-16):
        self.calls.append(('step', V, W, H, iteration, epoch, rank, world, bases, layout_T2, two_shot, direct, sparsity_alpha, epsilon))

    def klnmf_end(self, W, H, iterations_done):
        self.calls.append(('end', W, H, iterations_done))


@pytest.mark.parametrize('two_shot,direct', [(0, False), (0, True), (1, True), (2, False)])
def test_klnmf_sharded_pull_bookkeeping(two_shot, direct):
    """Two runs on one exchange: begin first, end(numIterations) last, and every step gets the iteration, the epoch the run
    started at (0, then the first run's count: the buffer's counters keep counting), and the exchange's rank, world, bases,
    layout_T2, form and direct flag unchanged; the exchange's epoch ends at the total."""
    import types
    from gcc_nmf_b200 import distributed as d
    bases = object()
    px = types.SimpleNamespace(epoch=0, rank=2, world=3, bases=bases, layout_T2=1000, two_shot=two_shot, direct=direct)
    V, W, H = object(), object(), object()
    for iters, epoch in ((3, 0), (2, 3)):
        ops = RecordingOps()
        assert d.klnmf_sharded_pull(ops, px, V, W, H, iters, 0.3, 0.25) == (W, H)
        assert ops.calls[0] == ('begin', V, W, H)
        assert ops.calls[-1] == ('end', W, H, iters)
        assert ops.calls[1:-1] == [('step', V, W, H, it, epoch, 2, 3, bases, 1000, two_shot, direct, 0.3, 0.25) for it in range(iters)]
        assert all(c[8] is bases for c in ops.calls[1:-1])
    assert px.epoch == 5


def test_shard_bookkeeping():
    from gcc_nmf_b200 import distributed as d
    for total, world in [(1872, 8), (37, 2), (10, 3), (7, 7)]:
        ranges = [d.shard_frames(total, world, r) for r in range(world)]
        assert ranges[0][0] == 0 and ranges[-1][1] == total
        assert all(a[1] == b[0] for a, b in zip(ranges, ranges[1:]))
        assert max(b - a for a, b in ranges) - min(b - a for a, b in ranges) <= 1
    assert d.shard_sample_range(3, 5, 1024, 256) == (768, 4 * 256 + 1024)


def test_sharded_nmf_and_seams_world2():
    world = 2
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_worker, args=(world, _free_port(), out), nprocs=world, join=True)
    F, K, T, I = 33, 6, 37, 5
    rng = np.random.default_rng(0)
    Vfull = (rng.random((F, 2 * T)) + 0.05).astype(np.float32)
    Wref, Href = orc.performKLNMF(Vfull, K, I, 0)
    for r in range(world):
        t0, t1 = out[r]['t']
        np.testing.assert_allclose(out[r]['W'], Wref, rtol=2e-5, atol=1e-7)       # identical dictionary on every rank
        Hs_ref = np.concatenate([Href[:, t0:t1], Href[:, T + t0:T + t1]], axis=1)
        np.testing.assert_allclose(out[r]['H'], Hs_ref, rtol=2e-5, atol=1e-7)
    assert np.array_equal(out[0]['W'], out[1]['W'])
    assert out[0]['agree'] == out[1]['agree'] == (5, 11, 2)
    N, hop = 16, 4
    frames = np.random.default_rng(1).standard_normal((1, T, N)).astype(np.float32)
    y = np.zeros((1, N + hop * (T - 1)), np.float32)
    for i in range(T):
        y[0, i * hop:i * hop + N] += frames[0, i]
    got = np.concatenate([out[r]['y'] for r in range(world)], axis=1)
    assert got.shape == y.shape
    np.testing.assert_allclose(got, y, rtol=0, atol=1e-5)
