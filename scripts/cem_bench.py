"""Time CEM's population rollout (b200rl_population_rollout) and one whole CEM iteration; print one JSON line per case.

  cartpole   CartPole (32,32), 65 536 members x max_path_length 200, n_evals 1, init_std 1
  swimmer    Swimmer (32,32), 16 384 members x max_path_length 500, n_evals 1, init_std 1

The population rollout is CUDA-event timed over at least a second after warm-up on the rows of iteration 0; the rate is
EXECUTED env-steps per second (the sum of the episode lengths over the time: episodes end at done or max_path_length).
The whole iteration (sample rows, rollout, gather, top-k, regenerate the elites, mean / std, the table's readback) is timed
as CEM.train with n_itr = 3 minus n_itr = 1, halved.  For context the same process times the lane rollout (b200rl_rollout,
every lane runs all T steps with auto-reset) of as many lanes x T.  Card name and power limit are read with nvidia-smi in
the same run.

Usage:  python scripts/cem_bench.py [--out FILE]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from vf_bench import card, timed  # noqa: E402


def _algo(env_name, M, T, n_itr):
    from rllab_b200.algos.cem import CEM
    from rllab_b200.envs.normalized_env import normalize
    from rllab_b200.policies.gaussian_mlp_policy import GaussianMLPPolicy
    if env_name == "cartpole":
        from rllab_b200.envs.box2d.cartpole_env import CartpoleEnv as E
    else:
        from rllab_b200.envs.mujoco.swimmer_env import SwimmerEnv as E
    env = normalize(E())
    pol = GaussianMLPPolicy(env.spec, hidden_sizes=(32, 32), seed=1)
    return CEM(env, pol, n_itr=n_itr, n_samples=M, max_path_length=T, init_std=1.0, best_frac=0.05, seed=5), pol


def run(cfg, env_name, M, T):
    import torch
    from rllab_b200 import _lib as L
    from rllab_b200 import ops
    algo, pol = _algo(env_name, M, T, 1)
    kind = L.ENV_KINDS[env_name]
    dev = pol.theta64.device
    P = pol.n_params
    mean = pol.theta64.clone()
    std = torch.ones(P, dtype=torch.float64, device=dev)
    rows = torch.empty((M, P), dtype=torch.float64, device=dev)
    ops.population_sample(mean, std, 1.0, 5, 0, rows)
    res = ops.PopulationResult(M, 1, pol.obs_dim, dev, keep_obs=False)

    def pop():
        ops.population_rollout(kind, rows, 32, 32, pol.min_std, 1, T, 0.99, 5, 0, 0, res)
    ms_pop = timed(pop)
    steps = int(res.len.sum().item())
    b = ops.LaneBatch(pol.obs_dim, pol.action_dim, M, T, dev)

    def lanes():
        ops.rollout(kind, pol.theta32, 32, 32, pol.min_std, b, T, None, None, 5, 0, 0)
    ms_lane = timed(lanes)

    def train(n):
        a, _ = _algo(env_name, M, T, n)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        a.train()
        torch.cuda.synchronize()
        return time.perf_counter() - t0
    train(1)
    t1 = min(train(1) for _ in range(2))
    t3 = min(train(3) for _ in range(2))
    name, power = card()
    return dict(cfg=cfg, env=env_name, members=M, max_path_length=T, hidden=32, gpu=name, power_limit=power,
                pop_rollout_ms=ms_pop, executed_steps=steps, mean_episode_len=steps / M,
                pop_executed_steps_per_s=steps / (ms_pop * 1e-3), lane_rollout_ms=ms_lane,
                lane_steps_per_s=M * T / (ms_lane * 1e-3),
                pop_over_lane_rate=(steps / ms_pop) / (M * T / ms_lane), cem_iteration_ms=(t3 - t1) / 2 * 1e3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from rllab_b200.misc import logger
    logger.set_quiet(True)
    res = [run("cartpole", "cartpole", 65536, 200), run("swimmer", "swimmer", 16384, 500)]
    for r in res:
        print(json.dumps(r))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
