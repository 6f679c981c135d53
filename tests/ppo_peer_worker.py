"""Worker of tests/test_gpu_ppo_peer.py (one process per rank under torchrun): PPO updates on lanes sharded over the ranks
against the same updates of the whole batch on one rank.

Every rank builds two PPO algos with the same policy initialisation and sampler seed: one sharded (its LaneSampler takes
this rank's block of the lanes, the advantage statistics and the baseline's normal equations are reduced over the ranks,
and every L-BFGS evaluation exchanges the [gradient | loss, sum KL | max KL] vector of its pass), one on the whole batch
with a single-rank communicator.  The Philox streams are indexed by the global lane, so a shard holds exactly the
corresponding lanes of the whole batch.  Two iterations each, so the second update starts from the carried penalty.
Checks: theta and the carried penalty are bit-identical on all ranks; every iteration tries the same penalties as the
single-rank run; theta is within PPO_TOL (relative to max |theta|) of the single-rank run.  With N = 384 lanes per rank (a
multiple of the 128-sample tile) every tile of a shard holds the same samples as the corresponding tile of the whole batch;
what differs is the float64 order of the block sums and, through the reduced advantage statistics, the last bits of
the centred advantages: measured 5.7e-15 with the same penalties (gloo, two ranks on one H100).

Environment: PPO_BACKEND = "nccl" (default; B200RL_PEER=0 selects the NCCL all-gather transport instead of peer memory) or
"gloo" (every rank on cuda:0, for a box with a single GPU)."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PPO_TOL = 1e-4


def _local_comm():
    """A single-rank communicator inside the torchrun job (it reads WORLD_SIZE / RANK at construction)."""
    from rllab_b200.parallel import Comm
    saved = {k: os.environ.get(k) for k in ("WORLD_SIZE", "RANK")}
    os.environ["WORLD_SIZE"], os.environ["RANK"] = "1", "0"
    try:
        c = Comm()
    finally:
        for k, v in saved.items():
            os.environ[k] = v
    assert not c.active
    return c


def main():
    import bench
    from rllab_b200.algos.ppo import PPO
    from rllab_b200.baselines.linear_feature_baseline import LinearFeatureBaseline
    from rllab_b200.misc import logger
    from rllab_b200.parallel import Comm
    from rllab_b200.policies.gaussian_mlp_policy import GaussianMLPPolicy
    logger.set_quiet(True)
    backend = os.environ.get("PPO_BACKEND", "nccl")
    comm = Comm(backend=backend)
    if backend == "gloo":
        torch.cuda.set_device(0)
    dev = torch.device("cuda", torch.cuda.current_device())
    want_peer = backend == "nccl" and os.environ.get("B200RL_PEER", "1") != "0"
    assert comm.active and comm.peer == want_peer, (comm.active, comm.peer, want_peer)
    dist, W = comm.dist, comm.world_size
    N, T = 384, 100

    def algo(c):
        env = bench.make_env("cartpole")
        policy = GaussianMLPPolicy(env.spec, hidden_sizes=(32, 32), seed=3)
        return PPO(env=env, policy=policy, baseline=LinearFeatureBaseline(env.spec), batch_size=N * W * T,
                   max_path_length=T, n_itr=2, discount=0.99, sampler_args=dict(n_envs=N * W, seed=7, comm=c))

    single, sharded = algo(_local_comm()), algo(comm)
    for a in (single, sharded):
        a.start_worker()
        a.init_opt()
    assert sharded.sampler.batch.N == N and single.sampler.batch.N == N * W
    res = []
    for itr in range(2):
        single.train_itr(itr)
        sharded.train_itr(itr)
        res.append((list(single.optimizer.tried_penalties), list(sharded.optimizer.tried_penalties)))
    torch.cuda.synchronize()
    th = sharded.policy.get_param_values()
    state = torch.tensor(np.concatenate([th, [float(sharded.optimizer._penalty)]]), dtype=torch.float64, device=dev)
    g = [torch.empty_like(state) for _ in range(W)]
    dist.all_gather(g, state)
    assert all(torch.equal(g[0], q) for q in g), "ranks disagree"
    for p_single, p_sharded in res:
        assert p_single == p_sharded, (p_single, p_sharded)
    assert float(sharded.optimizer._penalty) == float(single.optimizer._penalty)
    ref = single.policy.get_param_values()
    rel = float(np.max(np.abs(th - ref)) / np.max(np.abs(ref)))
    assert rel < PPO_TOL, rel
    if comm.rank == 0:
        print("PPO_PEER_OK backend=%s peer=%s penalties=%s theta_rel=%.3g evals=%d exchanges=%d collectives=%d" %
              (backend, comm.peer, res, rel, sharded._objective.n_evals, comm.n_peer_exchanges, comm.n_collectives))
    comm.close()


if __name__ == "__main__":
    main()
