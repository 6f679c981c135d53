"""Worker of tests/test_gpu_reps_peer.py (one process per rank under torchrun): REPS updates on lanes sharded over the
ranks against the same updates of the whole batch on one rank.

Every rank builds two REPS algos with the same policy initialisation, sampler seed and initial v: one sharded (its
LaneSampler takes this rank's block of the lanes; the dual's maximum and sums and every policy gradient pass are reduced
over the ranks), one on the whole batch with a single-rank communicator.  Two iterations each, so the second dual solve
starts from the first one's eta and v.  Both L-BFGS runs are capped at REPS_MAX_OPT_ITR iterations: the policy objective
is float32-grade, and over the default 50 iterations the line searches of two runs whose gradients differ in the last
bits (the summation order) part ways, so a longer run measures L-BFGS, not the sharding.  Checks: theta, eta and v are
bit-identical on all ranks; eta and v are within REPS_DUAL_TOL and theta within REPS_THETA_TOL (relative to the largest
entry) of the single-rank run.  With N = 384 lanes
per rank what differs from the single-rank run is the float64 order of the block sums.

Environment: REPS_BACKEND = "nccl" (default; B200RL_PEER=0 selects the NCCL all-gather transport instead of peer memory)
or "gloo" (every rank on cuda:0, for a box with a single GPU)."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

REPS_DUAL_TOL = 1e-6
REPS_THETA_TOL = 1e-4
REPS_MAX_OPT_ITR = 5


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
    from rllab_b200.algos.reps import REPS
    from rllab_b200.baselines.linear_feature_baseline import LinearFeatureBaseline
    from rllab_b200.misc import logger
    from rllab_b200.parallel import Comm
    from rllab_b200.policies.gaussian_mlp_policy import GaussianMLPPolicy
    logger.set_quiet(True)
    backend = os.environ.get("REPS_BACKEND", "nccl")
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
        return REPS(env=env, policy=policy, baseline=LinearFeatureBaseline(env.spec), batch_size=N * W * T,
                    max_path_length=T, n_itr=2, discount=0.99, max_opt_itr=REPS_MAX_OPT_ITR,
                    sampler_args=dict(n_envs=N * W, seed=7, comm=c))

    single, sharded = algo(_local_comm()), algo(comm)
    for a in (single, sharded):
        a.start_worker()
        np.random.seed(11)                   # the same initial v for both runs
        a.init_opt()
    assert sharded.sampler.batch.N == N and single.sampler.batch.N == N * W
    for itr in range(2):
        single.train_itr(itr)
        sharded.train_itr(itr)
    torch.cuda.synchronize()
    th = sharded.policy.get_param_values()
    state = torch.tensor(np.concatenate([th, [sharded.param_eta], sharded.param_v]), dtype=torch.float64, device=dev)
    g = [torch.empty_like(state) for _ in range(W)]
    dist.all_gather(g, state)
    assert all(torch.equal(g[0], q) for q in g), "ranks disagree"
    ref = single.policy.get_param_values()
    rel_th = float(np.max(np.abs(th - ref)) / np.max(np.abs(ref)))
    rel_eta = abs(sharded.param_eta - single.param_eta) / abs(single.param_eta)
    rel_v = float(np.max(np.abs(sharded.param_v - single.param_v)) / np.max(np.abs(single.param_v)))
    if comm.rank == 0:
        print("REPS_PEER backend=%s peer=%s eta=%.6g eta_rel=%.3g v_rel=%.3g theta_rel=%.3g exchanges=%d collectives=%d"
              % (backend, comm.peer, sharded.param_eta, rel_eta, rel_v, rel_th, comm.n_peer_exchanges,
                 comm.n_collectives), flush=True)
    assert rel_eta < REPS_DUAL_TOL and rel_v < REPS_DUAL_TOL, (rel_eta, rel_v)
    assert rel_th < REPS_THETA_TOL, rel_th
    if comm.rank == 0:
        print("REPS_PEER_OK backend=%s peer=%s" % (backend, comm.peer), flush=True)
    comm.close()


if __name__ == "__main__":
    main()
