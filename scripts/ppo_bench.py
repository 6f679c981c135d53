"""Time PPO's penalised gradient pass (b200rl_grad_penalized) against the plain gradient pass (b200rl_grad) and one whole
PPO iteration; print one JSON line per batch.

  cfg2     CartPole 65 536 lanes x 200 steps, (32,32)     cfg3     Swimmer 16 384 lanes x 500 steps, (32,32)
  hopper   Hopper 4 096 lanes x 500 steps, (64,64)

For each batch (one rollout of the PPO sampler at a seeded policy), the two passes at a theta off the sampling policy
(KL > 0, penalty 1) are CUDA-event timed over at least a second each after warm-up, alternating plain / penalised /
plain / penalised, and the faster repetition of each is reported.  cfg2 and cfg3 then run one PPO policy update with the
default PenaltyLbfgsOptimizer on that batch: wall time (host clock around work that ends in a device synchronise),
penalties tried, L-BFGS evaluations per try, and the host time per evaluation (wall time per evaluation minus the
measured penalised pass).  Card name and power limit are read with nvidia-smi in the same run.

Usage:  python scripts/ppo_bench.py [--out FILE]
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


def run(cfg, env_name, n_envs, T, hidden, iteration):
    import numpy as np
    import torch
    import bench
    from rllab_b200 import _lib as L
    from rllab_b200 import ops
    from rllab_b200.algos.ppo import PPO
    from rllab_b200.baselines.linear_feature_baseline import LinearFeatureBaseline
    from rllab_b200.policies.gaussian_mlp_policy import GaussianMLPPolicy
    env = bench.make_env(env_name)
    policy = GaussianMLPPolicy(env.spec, hidden_sizes=(hidden, hidden), seed=1)
    algo = PPO(env=env, policy=policy, baseline=LinearFeatureBaseline(env.spec), batch_size=n_envs * T,
               max_path_length=T, n_itr=1, discount=0.99, sampler_args=dict(n_envs=n_envs, seed=7))
    algo.start_worker()
    algo.init_opt()
    paths = algo.sampler.obtain_samples(0)
    sd = algo.sampler.process_samples(0, paths)
    b = sd.lane_batch
    theta0 = policy.get_param_values()
    th = torch.tensor(theta0 + 0.01 * np.random.RandomState(3).randn(theta0.size), dtype=torch.float32,
                      device=b.device)
    g = torch.zeros(policy.n_params, dtype=torch.float64, device=b.device)
    tri = torch.zeros(3, dtype=torch.float64, device=b.device)
    plain = lambda: ops.grad(L.LOSS_TRPO, th, policy.dims, policy.min_std, b, g, tri)             # noqa: E731
    pen = lambda: ops.grad_penalized(L.LOSS_TRPO, 1.0, th, policy.dims, policy.min_std, b, g, tri)  # noqa: E731
    t_plain, t_pen = [], []
    for _ in range(2):
        t_plain.append(timed(plain))
        t_pen.append(timed(pen))
    t_plain, t_pen = min(t_plain), min(t_pen)
    ops.grad_penalized(L.LOSS_TRPO, 1.0, th, policy.dims, policy.min_std, b, g, tri)
    mean_kl = float(tri[1].item())
    name, power = card()
    out = dict(cfg=cfg, env=env_name, lanes=n_envs, steps=T, hidden=hidden, samples=b.B, gpu=name, power_limit=power,
               grad_ms=round(t_plain, 4), grad_penalized_ms=round(t_pen, 4),
               penalized_over_plain=round(t_pen / t_plain, 4), mean_kl_at_timed_theta=mean_kl)
    if iteration:
        policy.set_param_values(theta0)
        ob = algo._objective
        n0 = ob.n_evals
        torch.cuda.synchronize()
        w0 = time.perf_counter()
        algo.optimize_policy(0, sd)
        after = ob.eval_lazy(sd)
        kl_after = after[1]                          # blocks: the iteration ends with its last pass read back
        wall = time.perf_counter() - w0
        n_evals = ob.n_evals - n0
        opt = algo.optimizer
        out.update(iteration_s=round(wall, 3), penalties=opt.tried_penalties,
                   evals_per_try=[t[2] for t in opt.terminations], terminations=[t[1] for t in opt.terminations],
                   evals=n_evals, wall_ms_per_eval=round(wall * 1e3 / max(n_evals, 1), 3),
                   host_ms_per_eval=round(wall * 1e3 / max(n_evals, 1) - t_pen, 3), mean_kl_after=kl_after)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from rllab_b200.misc import logger
    logger.set_quiet(True)
    res = [run("cfg2", "cartpole", 65536, 200, 32, True), run("cfg3", "swimmer", 16384, 500, 32, True),
           run("hopper", "hopper", 4096, 500, 64, False)]
    for r in res:
        print(json.dumps(r))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
