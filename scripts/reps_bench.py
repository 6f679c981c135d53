"""Time REPS's dual evaluation (b200rl_reps_delta_max + b200rl_reps_dual_sums) and one whole REPS policy update; print
one JSON line per batch.

  cfg2     CartPole 65 536 lanes x 200 steps, (32,32)     cfg3     Swimmer 16 384 lanes x 500 steps, (32,32)

For each batch (one rollout of the REPS sampler at a seeded policy):
  * the dual evaluation at the initial (eta, v) is CUDA-event timed over at least a second after warm-up, without and with
    the weights written; the report gives its algorithmic bytes per sample (4 O + 7 read per pass, two passes, + 4 written
    for w) and the achieved share of the H100 SXM's 3.35 TB/s data-sheet HBM bandwidth;
  * one optimize_policy with the default settings: wall time (host clock around work that ends in a device synchronise),
    the number of dual and policy evaluations, the device time of those passes (evaluations x the timed pass), and the
    host share of the wall time.
Card name and power limit are read with nvidia-smi in the same run.

Usage:  python scripts/reps_bench.py [--out FILE]
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

HBM_BYTES_PER_S = 3.35e12


def run(cfg, env_name, n_envs, T, hidden):
    import numpy as np
    import torch
    import bench
    from rllab_b200 import _lib as L
    from rllab_b200 import ops
    from rllab_b200.algos.reps import REPS
    from rllab_b200.baselines.linear_feature_baseline import LinearFeatureBaseline
    from rllab_b200.policies.gaussian_mlp_policy import GaussianMLPPolicy
    np.random.seed(1)
    env = bench.make_env(env_name)
    policy = GaussianMLPPolicy(env.spec, hidden_sizes=(hidden, hidden), seed=1)
    algo = REPS(env=env, policy=policy, baseline=LinearFeatureBaseline(env.spec), batch_size=n_envs * T,
                max_path_length=T, n_itr=1, discount=0.99, sampler_args=dict(n_envs=n_envs, seed=7))
    algo.start_worker()
    algo.init_opt()
    paths = algo.sampler.obtain_samples(0)
    sd = algo.sampler.process_samples(0, paths)
    b = sd.lane_batch
    O, D = b.O, 2 * b.O + 4
    v = torch.tensor(algo.param_v, dtype=torch.float64, device=b.device)
    M = torch.zeros(1, dtype=torch.float64, device=b.device)
    sums = torch.zeros(D + 2, dtype=torch.float64, device=b.device)
    w = torch.zeros((b.T, b.N), dtype=torch.float32, device=b.device)

    def dual(w_out=None):
        ops.reps_delta_max(b, v, M)
        ops.reps_dual_sums(b, v, float(algo.param_eta), M, sums, w_out)

    t_dual = min(timed(dual) for _ in range(2))
    t_dual_w = min(timed(lambda: dual(w)) for _ in range(2))
    th = policy.theta32
    g = torch.zeros(policy.n_params, dtype=torch.float64, device=b.device)
    t_grad = min(timed(lambda: ops.grad(L.LOSS_VPG, th, policy.dims, policy.min_std, b, g)) for _ in range(2))
    bytes_dual = 2 * (4 * O + 7)
    name, power = card()
    out = dict(cfg=cfg, env=env_name, lanes=n_envs, steps=T, hidden=hidden, samples=b.B, gpu=name, power_limit=power,
               dual_ms=round(t_dual, 4), dual_with_weights_ms=round(t_dual_w, 4), dual_bytes_per_sample=bytes_dual,
               dual_hbm_share=round(bytes_dual * b.B / (t_dual * 1e-3) / HBM_BYTES_PER_S, 3),
               dual_with_weights_hbm_share=round((bytes_dual + 4) * b.B / (t_dual_w * 1e-3) / HBM_BYTES_PER_S, 3),
               policy_grad_ms=round(t_grad, 4))
    torch.cuda.synchronize()
    w0 = time.perf_counter()
    algo.optimize_policy(0, sd)
    torch.cuda.synchronize()
    wall = time.perf_counter() - w0
    dev_s = (algo.n_dual_evals * t_dual + algo.n_policy_evals * t_grad) * 1e-3
    out.update(iteration_s=round(wall, 3), dual_evals=algo.n_dual_evals, policy_evals=algo.n_policy_evals,
               device_s_estimate=round(dev_s, 3), host_share=round(max(0.0, 1.0 - dev_s / wall), 3),
               eta_after=float(algo.param_eta))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from rllab_b200.misc import logger
    logger.set_quiet(True)
    res = [run("cfg2", "cartpole", 65536, 200, 32), run("cfg3", "swimmer", 16384, 500, 32)]
    for r in res:
        print(json.dumps(r))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
