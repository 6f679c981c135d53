"""gym CartPole-v0 with CategoricalGRUPolicy (hidden 32, one-hot previous action in the input): CUDA-event timings
(median of --reps after a warm-up, with the min and max to show the spread) of the categorical GRU rollout, loss/KL,
BPTT gradient, Fisher-vector product (activation cache) and one TRPO update (optimize_policy: gradient, 10 CG
iterations, line search), at --lanes x --steps and at the example's 4000 samples (20 lanes x 200 steps).  Reads the
card name and power limit in the same call and prints one JSON line.

    python scripts/categorical_gru_bench.py [--lanes 65536] [--steps 200] [--reps 5]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import categorical_gru_oracle as C  # noqa: E402
from gru_bench import card, timed  # noqa: E402
from rllab_b200 import _lib as L, ops  # noqa: E402


def passes(N, T, reps):
    dev = torch.device("cuda:0")
    dims = ops.CategoricalGRUDims(4, 32, 2, True)
    th = torch.tensor(C.init_params(C.CatGruDims(4, 32, 2, True), np.random.RandomState(3)), dtype=torch.float32,
                      device=dev)
    b = ops.LaneBatch(4, 2, N, T, dev)
    b.recurrent = b.categorical = True
    P_ = th.numel()
    out = torch.zeros(3, dtype=torch.float64, device=dev)
    g = torch.zeros(P_, dtype=torch.float64, device=dev)
    Hx = torch.zeros_like(g)
    x = torch.tensor(np.random.RandomState(1).randn(P_), device=dev)
    hc = b.hcache(32, 0)
    w = torch.zeros(2 * b.O + 4, dtype=torch.float64, device=dev)
    r = dict()
    r["rollout_s"] = timed(lambda i: ops.gru_rollout(dims, th, b, T, L.ENV_GYM_CARTPOLE, None, None, 1, i, 0), reps)
    ops.process_samples(b, w, 0.99, 1.0, drop_cut_paths=True)
    r["loss_kl_s"] = timed(lambda i: ops.loss_kl(L.LOSS_TRPO, th, dims, None, b, out), reps)
    r["grad_s"] = timed(lambda i: ops.grad(L.LOSS_TRPO, th, dims, None, b, g, out, hc), reps)
    r["fvp_cached_s"] = timed(lambda i: ops.fvp(th, dims, None, b, x, 1e-5, 1.0, Hx, hc), reps)
    return r


def trpo_update(N, T, reps):
    from rllab_b200.algos.trpo import TRPO
    from rllab_b200.baselines.linear_feature_baseline import LinearFeatureBaseline
    from rllab_b200.envs.gym_env import GymEnv
    from rllab_b200.envs.normalized_env import normalize
    from rllab_b200.policies.categorical_gru_policy import CategoricalGRUPolicy
    env = normalize(GymEnv("CartPole-v0"))
    pol = CategoricalGRUPolicy(env_spec=env.spec, seed=3)
    algo = TRPO(env=env, policy=pol, baseline=LinearFeatureBaseline(env_spec=env.spec), batch_size=N * T,
                max_path_length=T, n_itr=1, discount=0.99, step_size=0.01, sampler_args=dict(n_envs=N, seed=7))
    algo.start_worker()
    algo.init_opt()
    sd = algo.sampler.process_samples(0, algo.sampler.obtain_samples(0))
    theta0 = pol.get_param_values()

    def step(i):
        pol.set_param_values(theta0)
        algo.optimize_policy(0, sd)
    return timed(step, reps)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lanes", type=int, default=65536)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    L.load()
    from rllab_b200.misc import logger
    logger.set_quiet(True)
    res = dict(what="categorical_gru_cartpole_v0", card=card(), lanes=a.lanes, steps=a.steps)
    for tag, (N, T) in (("big", (a.lanes, a.steps)), ("example", (20, 200))):
        r = passes(N, T, a.reps)
        r["trpo_optimize_s"] = trpo_update(N, T, a.reps)
        res.update({"%s_%s" % (tag, k): v for k, v in r.items()})
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
