"""GPU side of north_star's Swimmer learning check: TRPO on the device with the configuration of
tests/golden/oracle_swimmer_trpo_curve.json (same lanes, horizon, Philox seed, policy seed), AverageReturn per iteration
printed next to the float64 oracle's curve.  Run on an H100:  python scripts/swimmer_curve_gpu.py [n_itr] [swimmer|hopper]

Iteration 0 sees the same initial policy and the same noise as the oracle run, so its AverageReturn must agree to the
planar-dynamics tolerance; later iterations are two independent stochastic-optimisation trajectories of the same
algorithm, to be compared at matched sample count (north_star: within +-5 %)."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main(n_itr, env_name="swimmer", precision="f32", seed=None, policy_seed=None):
    from rllab_b200.algos.trpo import TRPO
    from rllab_b200.baselines.linear_feature_baseline import LinearFeatureBaseline
    from rllab_b200.envs.mujoco.hopper_env import HopperEnv
    from rllab_b200.envs.mujoco.swimmer_env import SwimmerEnv
    from rllab_b200.envs.normalized_env import normalize
    from rllab_b200.misc import logger
    from rllab_b200.policies.gaussian_mlp_policy import GaussianMLPPolicy
    gold = json.load(open(os.path.join(ROOT, "tests", "golden", "oracle_%s_trpo_curve.json" % env_name)))
    cfg, curve = gold["config"], gold["curve"]
    logger.set_quiet(True)
    env = normalize(HopperEnv() if env_name == "hopper" else SwimmerEnv())
    policy = GaussianMLPPolicy(env.spec, hidden_sizes=tuple(cfg["hidden"]),
                               seed=cfg["policy_seed"] if policy_seed is None else policy_seed)
    algo = TRPO(env=env, policy=policy, baseline=LinearFeatureBaseline(env.spec), batch_size=cfg["lanes"] * cfg["horizon"],
                max_path_length=cfg["horizon"], n_itr=n_itr, discount=cfg["discount"], gae_lambda=cfg["gae_lambda"],
                step_size=cfg["step_size"], optimizer_args=dict(cg_iters=cfg["cg_iters"], precision=precision),
                sampler_args=dict(n_envs=cfg["lanes"], seed=cfg["seed"] if seed is None else seed))
    algo.start_worker()
    algo.init_opt()
    rows = []
    for itr in range(min(n_itr, len(curve))):
        with logger.prefix("itr #%d | " % itr):
            algo.train_itr(itr)
        tab = logger.get_last_table()
        ref = curve[itr]
        rows.append((itr, tab["AverageReturn"], ref["AverageReturn"], tab["MeanKL"], ref["MeanKL"]))
        print("itr %3d  AverageReturn gpu %9.3f  oracle %9.3f   MeanKL gpu %.5f oracle %.5f"
              % rows[-1], flush=True)
    tail = rows[-5:]
    g, o = np.mean([r[1] for r in tail]), np.mean([r[2] for r in tail])
    print("mean AverageReturn over the last %d iterations: gpu %.3f oracle %.3f  (ratio %.3f)" % (len(tail), g, o, g / o))


if __name__ == "__main__":
    main(int(sys.argv[1]) if len(sys.argv) > 1 else 40, sys.argv[2] if len(sys.argv) > 2 else "swimmer",
         sys.argv[3] if len(sys.argv) > 3 else "f32", int(sys.argv[4]) if len(sys.argv) > 4 else None,
         int(sys.argv[5]) if len(sys.argv) > 5 else None)
