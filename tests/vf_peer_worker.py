"""Worker of tests/test_gpu_vf_peer.py (one process per rank under torchrun): a GaussianMLPBaseline fit on lanes sharded over
the ranks against the same fit of the whole batch on one rank.

Every rank rolls out the whole batch (the Philox stream is indexed by the global lane, so its shard is bit-identical to the
corresponding lanes of the whole batch) and fits twice: once on its own shard with the communicator (the fit of every
sharded run: all-reduced normalisation statistics, and per L-BFGS evaluation the exchanged [gradient | NLL, KL, max KL]
vector), once on the whole batch without it.  Two fits in a row, so the second starts from the persisted penalty.
Checks: theta, the normalisation constants and the penalty are bit-identical on all ranks; the penalty sequence equals the
single-rank one; theta is within VF_TOL (relative to max |theta|) of the single-rank fit.  With N = 384 lanes per rank
(a multiple of the 128-sample tile) every tile of a shard holds the same samples as the corresponding tile of the whole
batch, so only the float64 order of the block sums differs: measured 1.8e-14 (gloo, two ranks on one H100).  A grouping
that puts different samples into the tiles moves theta by up to ~4e-4 (test_host_api_matches_lane_hooks); VF_TOL sits
between the two.

Environment: VF_BACKEND = "nccl" (default; B200RL_PEER=0 selects the NCCL all-gather transport instead of peer memory) or
"gloo" (every rank on cuda:0, for a box with a single GPU)."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

VF_TOL = 1e-4


def main():
    from rllab_b200 import ops
    from rllab_b200 import _lib as L
    from rllab_b200.misc import logger
    from rllab_b200.optimizers.penalty_lbfgs_optimizer import PenaltyLbfgsOptimizer
    from rllab_b200.parallel import Comm
    from rllab_b200.regressors.gaussian_mlp_regressor import GaussianMLPRegressor
    logger.set_quiet(True)
    backend = os.environ.get("VF_BACKEND", "nccl")
    comm = Comm(backend=backend)
    if backend == "gloo":
        torch.cuda.set_device(0)
    dev = torch.device("cuda", torch.cuda.current_device())
    want_peer = backend == "nccl" and os.environ.get("B200RL_PEER", "1") != "0"
    assert comm.active and comm.peer == want_peer, (comm.active, comm.peer, want_peer)
    dist, W = comm.dist, comm.world_size
    O, A, N, T = 4, 1, 384, 100
    theta_pol = np.random.RandomState(1).uniform(-0.3, 0.3, 4 * 32 + 32 + 32 * 32 + 32 + 32 + 1 + 1)
    th32 = torch.tensor(theta_pol, dtype=torch.float32, device=dev)

    def make_batch(n, lane0):
        b = ops.LaneBatch(O, A, n, T, dev)
        ops.rollout(L.ENV_CARTPOLE, th32, 32, 32, 1e-6, b, T, None, None, 3, 0, lane0)
        ops.process_samples(b, None, 0.99, 1.0, drop_cut_paths=True)      # cut paths masked: the count is exercised
        return b

    full = make_batch(N * W, 0)
    mine = make_batch(N, comm.rank * N)

    def regressor():
        np.random.seed(5)
        return GaussianMLPRegressor((O,), 1, name="vf", optimizer=PenaltyLbfgsOptimizer(max_opt_itr=20))

    single, sharded = regressor(), regressor()
    res = []
    for _ in range(2):
        single.fit_device(full.obs, full.ret.view(-1), full.flags.view(-1), None)
        sharded.fit_device(mine.obs, mine.ret.view(-1), mine.flags.view(-1), comm)
        res.append((list(single._optimizer.tried_penalties), list(sharded._optimizer.tried_penalties)))
    torch.cuda.synchronize()
    th = sharded.get_param_values()
    state = torch.tensor(np.concatenate([th, sharded.get_stats(), [float(sharded._optimizer._penalty)]]), device=dev)
    g = [torch.empty_like(state) for _ in range(W)]
    dist.all_gather(g, state)
    assert all(torch.equal(g[0], q) for q in g), "ranks disagree"
    for p_single, p_sharded in res:
        assert p_single == p_sharded, (p_single, p_sharded)
    np.testing.assert_allclose(sharded.get_stats(), single.get_stats(), rtol=1e-12)
    ref = single.get_param_values()
    rel = float(np.max(np.abs(th - ref)) / np.max(np.abs(ref)))
    assert rel < VF_TOL, rel
    if comm.rank == 0:
        print("VF_PEER_OK backend=%s peer=%s penalties=%s theta_rel=%.3g exchanges=%d collectives=%d" %
              (backend, comm.peer, res, rel, comm.n_peer_exchanges, comm.n_collectives))
    comm.close()


if __name__ == "__main__":
    main()
