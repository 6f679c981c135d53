"""How confident does CartPole-v0 TRPO training make CategoricalMLPPolicy?  Runs the reference example's configuration
(examples/trpo_gym_cartpole.py: TRPO, CategoricalMLPPolicy (32, 32), LinearFeatureBaseline, batch 4000,
max_path_length 200, discount 0.99, step_size 0.01) for the iterations of tests/golden/oracle_cartpole_v0_trpo_curve.json
and prints, per iteration, AverageReturn and the fraction of valid samples whose logit gap |z0 - z1| at theta_old
exceeds 8, 12, 16 and 20 (float64 logits of the sampled observations), then one JSON line with the whole table.

    python scripts/categorical_regime.py [--seed 7]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402

import categorical_oracle as C  # noqa: E402

THRESHOLDS = (8, 12, 16, 20)
CURVE = os.path.join(ROOT, "tests", "golden", "oracle_cartpole_v0_trpo_curve.json")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seed", type=int, default=7)
    a = ap.parse_args()
    from rllab_b200.algos.trpo import TRPO
    from rllab_b200.baselines.linear_feature_baseline import LinearFeatureBaseline
    from rllab_b200.envs.gym_env import GymEnv
    from rllab_b200.envs.normalized_env import normalize
    from rllab_b200.misc import logger
    from rllab_b200.policies.categorical_mlp_policy import CategoricalMLPPolicy
    logger.set_quiet(True)
    n_itr = len(next(iter(json.load(open(CURVE))["AverageReturn"].values())))
    env = normalize(GymEnv("CartPole-v0"))
    policy = CategoricalMLPPolicy(env_spec=env.spec, hidden_sizes=(32, 32), seed=3)
    algo = TRPO(env=env, policy=policy, baseline=LinearFeatureBaseline(env_spec=env.spec), batch_size=4000,
                max_path_length=200, n_itr=n_itr, discount=0.99, step_size=0.01, sampler_args=dict(seed=a.seed))
    dims = C.CatDims(4, (32, 32), 2)
    rows = []
    optimize = algo.optimize_policy

    def optimize_and_record(itr, sd):
        b = sd.lane_batch
        keep = b.valid_mask().reshape(-1)
        obs = b.obs.cpu().numpy().reshape(4, -1).T[keep].astype(np.float64)
        z, _ = C.forward(policy.get_param_values(), obs, dims)
        gap = np.abs(z[:, 0] - z[:, 1])
        rows.append(dict(itr=itr, samples=int(keep.sum()), max_gap=float(gap.max()),
                         **{"frac_gap_gt_%d" % t: float(np.mean(gap > t)) for t in THRESHOLDS}))
        return optimize(itr, sd)

    algo.optimize_policy = optimize_and_record
    algo.start_worker()
    algo.init_opt()
    for itr in range(n_itr):
        algo.train_itr(itr)
        rows[-1]["AverageReturn"] = float(logger.get_last_table()["AverageReturn"])
        r = rows[-1]
        print("itr %3d  return %6.1f  samples %5d  max gap %6.2f  " % (itr, r["AverageReturn"], r["samples"], r["max_gap"])
              + "  ".join(">%d: %.4f" % (t, r["frac_gap_gt_%d" % t]) for t in THRESHOLDS))
    print(json.dumps(dict(what="categorical_regime", seed=a.seed, rows=rows)))


if __name__ == "__main__":
    main()
