"""Two-rank REPS (tests/reps_peer_worker.py under torchrun): the sharded update equals the whole-batch update (eta, v and
theta close) and every rank ends with bit-identical theta, eta and v.  Over both multi-GPU transports (peer memory and the
NCCL all-gather; skipped on a box with fewer than two GPUs) and over gloo with both ranks on one GPU."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


def _n_gpus():
    try:
        import torch
    except ImportError:
        return 0
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


def _run(port, **env):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tests", "reps_peer_worker.py")]
    e = dict(os.environ)
    e.update(env)
    out = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=600, env=e)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-4000:]
    assert "REPS_PEER_OK" in out.stdout, out.stdout[-2000:]
    print("\n".join(out.stdout.strip().splitlines()[-2:]))
    return out.stdout


@pytest.mark.skipif(_n_gpus() < 2, reason="needs two GPUs")
def test_two_rank_reps_peer_memory():
    out = _run(29661, REPS_BACKEND="nccl", B200RL_PEER="1")
    assert "peer=True" in out and "exchanges=0 " not in out


@pytest.mark.skipif(_n_gpus() < 2, reason="needs two GPUs")
def test_two_rank_reps_nccl_gather():
    assert "peer=False" in _run(29662, REPS_BACKEND="nccl", B200RL_PEER="0")


@pytest.mark.skipif(_n_gpus() < 1, reason="needs a GPU")
def test_two_rank_reps_gloo_one_gpu():
    assert "peer=False" in _run(29663, REPS_BACKEND="gloo")
