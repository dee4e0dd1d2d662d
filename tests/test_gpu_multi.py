"""GPU, >= 2 devices: the frame-sharded enhancement pipeline (joint dictionary with the cross-rank sum of the W-update numerator
formed in the NVSwitch and signalled between kernels, one all-reduce of the mean angular spectrum, iSTFT seam exchange) against the
single-GPU pipeline run on the whole recording.  Spawns tests/multi_gpu_check.py under torchrun with 2 ranks, once per form of the
numerator exchange: pull exchange inside the W update / one-shot / two-shot (GCCNMF_COLLECTIVE=pullw / pull1 / pull2), reduction inside the switch
two- / one-shot (=multimem / multimem1), NCCL all-reduce (=nccl); and once with --pull-forms, which holds every form of the pull
exchange to float64 rank by rank on uneven shards.  Skipped on a single-GPU box (tests/test_gpu_klnmf_pull.py runs the pull exchange
at world 1)."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _gpus():
    import torch
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


def _torchrun(port, *args, env=None):
    cmd = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', '2', '--master-addr', '127.0.0.1',
           '--master-port', str(port), os.path.join(ROOT, 'tests', 'multi_gpu_check.py')] + list(args)
    return subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=env, cwd=ROOT)


def test_pull_forms_per_rank_match_float64():
    """Every pull-exchange form on uneven shards: each rank's H slice and W against the joint float64 run, W bit-identical across
    ranks, the direct forms and form 2 bit-identical to each other."""
    if _gpus() < 2:
        pytest.skip('needs >= 2 GPUs')
    r = _torchrun(29521, '--pull-forms')
    print(r.stdout[-3000:])
    assert r.returncode == 0, r.stderr[-3000:]
    assert 'PULL_FORMS_CHECK PASS' in r.stdout, r.stdout[-3000:]


@pytest.mark.parametrize('collective', ['pullw', 'pull1', 'pull2', 'multimem', 'multimem1', 'nccl'])
def test_sharded_pipeline_matches_single_gpu(collective):
    if _gpus() < 2:
        pytest.skip('needs >= 2 GPUs')
    env = dict(os.environ, GCCNMF_COLLECTIVE=collective)
    r = _torchrun(29511 + ['pullw', 'pull1', 'pull2', 'multimem', 'multimem1', 'nccl'].index(collective), env=env)
    print(r.stdout[-3000:])
    assert r.returncode == 0, r.stderr[-3000:]
    assert 'MULTI_GPU_CHECK PASS' in r.stdout, r.stdout[-3000:]
    assert 'W identical across ranks: True' in r.stdout
    if collective.startswith('pull'):
        assert 'pull exchange' in r.stdout.split('collective:')[1].splitlines()[0], r.stdout[-2000:]
    if collective.startswith('multimem'):
        assert 'multimem' in r.stdout.split('collective:')[1].splitlines()[0] or 'nccl' in r.stdout     # NVLS may be unavailable on a given box
