"""Two-rank PPO (tests/ppo_peer_worker.py under torchrun): the sharded update equals the whole-batch update (same
penalties tried, theta close) and every rank ends with bit-identical theta and carried penalty.  Over both multi-GPU
transports (peer memory fused into the passes, and the NCCL all-gather; skipped on a box with fewer than two GPUs) and
over gloo with both ranks on one GPU, which runs the same unfused exchange path on a single-GPU box."""
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
           "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tests", "ppo_peer_worker.py")]
    e = dict(os.environ)
    e.update(env)
    out = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=600, env=e)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-4000:]
    assert "PPO_PEER_OK" in out.stdout, out.stdout[-2000:]
    print(out.stdout.strip().splitlines()[-1])
    return out.stdout


@pytest.mark.skipif(_n_gpus() < 2, reason="needs two GPUs")
def test_two_rank_ppo_peer_memory():
    out = _run(29651, PPO_BACKEND="nccl", B200RL_PEER="1")
    assert "peer=True" in out and "exchanges=0 " not in out


@pytest.mark.skipif(_n_gpus() < 2, reason="needs two GPUs")
def test_two_rank_ppo_nccl_gather():
    assert "peer=False" in _run(29652, PPO_BACKEND="nccl", B200RL_PEER="0")


@pytest.mark.skipif(_n_gpus() < 1, reason="needs a GPU")
def test_two_rank_ppo_gloo_one_gpu():
    assert "peer=False" in _run(29653, PPO_BACKEND="gloo")
