"""Two-rank CEM (tests/cem_peer_worker.py under torchrun): the members sharded over two ranks give cur_mean, cur_std and the
policy bit-identical to the single-rank run, and identical on both ranks.  Over both multi-GPU transports (peer memory and
the NCCL all-gather; skipped on a box with fewer than two GPUs) and over gloo with both ranks on one GPU."""
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
           "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tests", "cem_peer_worker.py")]
    e = dict(os.environ)
    e.update(env)
    out = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=600, env=e)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-4000:]
    assert "CEM_PEER_OK" in out.stdout, out.stdout[-2000:]
    print(out.stdout.strip().splitlines()[-1])
    return out.stdout


@pytest.mark.skipif(_n_gpus() < 2, reason="needs two GPUs")
def test_two_rank_cem_peer_memory():
    assert "peer=True" in _run(29651, CEM_BACKEND="nccl", B200RL_PEER="1")


@pytest.mark.skipif(_n_gpus() < 2, reason="needs two GPUs")
def test_two_rank_cem_nccl_gather():
    assert "peer=False" in _run(29652, CEM_BACKEND="nccl", B200RL_PEER="0")


@pytest.mark.skipif(_n_gpus() < 1, reason="needs a GPU")
def test_two_rank_cem_gloo_one_gpu():
    _run(29653, CEM_BACKEND="gloo")
