"""Worker of tests/test_gpu_cem_peer.py (one process per rank under torchrun): CEM with the members sharded over the ranks
against the same CEM on one rank.

Every rank runs CEM twice from the same seed: once sharded with the communicator, then single-rank (a Comm-like object
with world_size 1) with the key the sharded run used.  Checks: cur_mean, cur_std and the policy of the sharded run are
bit-identical to the single-rank run and identical on all ranks (a member's row and episodes depend only on its global index; the elites are regenerated
locally from the gathered fitness).  Cases: n_samples; batch_size (waves of members); no seed given, with np.random
seeded differently on every rank (the ranks must agree one key); and fewer members than ranks in Swimmer (an empty
shard in an env whose diagnostics gather the episodes' observations).

Environment: CEM_BACKEND = "nccl" (default; B200RL_PEER=0 selects the NCCL all-gather transport instead of peer memory)
or "gloo" (every rank on cuda:0, for a box with a single GPU)."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


class _Single(object):
    world_size, rank, active = 1, 0, False

    def shard(self, n_total):
        return n_total, 0


def run(comm, env_name="cartpole", **kw):
    from rllab_b200.algos.cem import CEM
    from rllab_b200.envs.normalized_env import normalize
    from rllab_b200.policies.gaussian_mlp_policy import GaussianMLPPolicy
    if env_name == "swimmer":
        from rllab_b200.envs.mujoco.swimmer_env import SwimmerEnv as E
    else:
        from rllab_b200.envs.box2d.cartpole_env import CartpoleEnv as E
    env = normalize(E())
    pol = GaussianMLPPolicy(env.spec, hidden_sizes=(32, 32), seed=3)
    kw.setdefault("max_path_length", 100)
    algo = CEM(env, pol, n_itr=3, comm=comm, **kw)
    algo.train()
    torch.cuda.synchronize()
    return torch.cat([algo.cur_mean, algo.cur_std, pol.theta64]), algo.last["M"], algo.seed


def main():
    from rllab_b200.misc import logger
    from rllab_b200.parallel import Comm
    logger.set_quiet(True)
    backend = os.environ.get("CEM_BACKEND", "nccl")
    comm = Comm(backend=backend)
    if backend == "gloo":
        torch.cuda.set_device(0)
    assert comm.active
    W = comm.world_size
    out = []
    cases = (
        dict(seed=31, n_samples=301, best_frac=0.05, n_evals=2),
        dict(seed=31, n_samples=40, batch_size=5000, best_frac=0.1),
        # no seed: every rank draws its own key from its own np.random (seeded differently per rank here); train()
        # must agree one key over the ranks before any rank regenerates another rank's elite rows
        dict(seed=None, n_samples=97, best_frac=0.1),
        # fewer members than ranks: one rank's shard is empty, in an env whose diagnostics gather observations
        dict(seed=31, env_name="swimmer", n_samples=1, best_frac=0.5, max_path_length=20),
    )
    for kw in cases:
        kw = dict(kw)
        if kw["seed"] is None:
            np.random.seed(1000 + comm.rank)
        sharded, m_sharded, seed = run(comm, **kw)
        kw["seed"] = seed                       # the agreed key, to rerun on one rank
        single, m_single, _ = run(_Single(), **kw)
        assert m_single == m_sharded, (m_single, m_sharded)
        assert torch.equal(single, sharded), "sharded run differs from the single-rank run"
        g = [torch.empty_like(sharded) for _ in range(W)]
        comm.dist.all_gather(g, sharded)
        assert all(torch.equal(g[0], q) for q in g), "ranks disagree"
        out.append(m_sharded)
    if comm.rank == 0:
        print("CEM_PEER_OK backend=%s peer=%s members=%s collectives=%d exchanges=%d" %
              (backend, comm.peer, out, comm.n_collectives, comm.n_peer_exchanges))
    comm.close()


if __name__ == "__main__":
    main()
