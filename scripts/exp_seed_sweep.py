"""Experiment (not product code): distribution of the Swimmer TRPO learning curve over sampler seeds for several update
precisions -- the curves are chaotic (a 1e-16 perturbation moves the iteration-40 return by several units), so single runs
say little.  Variants: f32 (shipped path), f64 (precision="f64" parity kernels), hilo (float32 kernels, CG direction split
into two float32 words, two kernel calls), f64cg6 (float64 kernels, 6 CG iterations), f32cg20 (float32, 20 CG iterations).
Usage: python scripts/exp_seed_sweep.py <n_seeds> [variants comma separated] [swimmer|hopper] -> results/seed_sweep_<env>.json"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def run(variant, seed, n_itr=40, env_name="swimmer"):
    import torch
    from rllab_b200.algos.trpo import TRPO
    from rllab_b200.baselines.linear_feature_baseline import LinearFeatureBaseline
    from rllab_b200.envs.mujoco.hopper_env import HopperEnv
    from rllab_b200.envs.mujoco.swimmer_env import SwimmerEnv
    from rllab_b200.envs.normalized_env import normalize
    from rllab_b200.misc import logger
    from rllab_b200.optimizers.conjugate_gradient_optimizer import ConjugateGradientOptimizer as CGO
    from rllab_b200.policies.gaussian_mlp_policy import GaussianMLPPolicy

    class HiLo(CGO):
        def _make_Hx(self, batch, b, hcache, tiles):
            inner = CGO._make_Hx(self, batch, b, hcache, tiles)
            lo_out = torch.zeros_like(b["z"])

            def Hx(vec, out):
                hi = vec.float().double()
                inner(hi, out)
                inner(vec - hi, lo_out)
                out.add_(lo_out)
            return Hx

    cfg = json.load(open(os.path.join(ROOT, "tests", "golden", "oracle_%s_trpo_curve.json" % env_name)))["config"]
    opt = dict(f32=lambda: CGO(cg_iters=10), f64=lambda: CGO(cg_iters=10, precision="f64"), hilo=lambda: HiLo(cg_iters=10),
               f64cg6=lambda: CGO(cg_iters=6, precision="f64"), f32cg20=lambda: CGO(cg_iters=20))[variant]()
    env = normalize(HopperEnv() if env_name == "hopper" else SwimmerEnv())
    policy = GaussianMLPPolicy(env.spec, hidden_sizes=tuple(cfg["hidden"]), seed=cfg["policy_seed"])
    algo = TRPO(env=env, policy=policy, baseline=LinearFeatureBaseline(env.spec), batch_size=cfg["lanes"] * cfg["horizon"],
                max_path_length=cfg["horizon"], n_itr=n_itr, discount=cfg["discount"], gae_lambda=cfg["gae_lambda"],
                step_size=cfg["step_size"], optimizer=opt, sampler_args=dict(n_envs=cfg["lanes"], seed=seed))
    algo.start_worker()
    algo.init_opt()
    rets = []
    for itr in range(n_itr):
        algo.train_itr(itr)
        rets.append(float(logger.get_last_table()["AverageReturn"]))
    algo.shutdown_worker()
    return rets


def main():
    from rllab_b200.misc import logger
    logger.set_quiet(True)
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 8
    variants = (sys.argv[2] if len(sys.argv) > 2 else "f32,f64,hilo,f64cg6,f32cg20").split(",")
    env_name = sys.argv[3] if len(sys.argv) > 3 else "swimmer"
    out = {}
    for v in variants:
        out[v] = {}
        for seed in range(101, 101 + n):
            r = run(v, seed, env_name=env_name)
            out[v][seed] = r
            print("%-8s seed %d: itr 9 %.2f  19 %.2f  29 %.2f  last-5 %.2f" % (v, seed, r[9], r[19], r[29], np.mean(r[-5:])),
                  flush=True)
        tails = np.array([np.mean(r[-5:]) for r in out[v].values()])
        print("== %-8s last-5 mean over %d seeds: %.2f +- %.2f  (min %.2f max %.2f)" %
              (v, n, tails.mean(), tails.std(), tails.min(), tails.max()), flush=True)
    os.makedirs(os.path.join(ROOT, "results"), exist_ok=True)
    json.dump(out, open(os.path.join(ROOT, "results", "seed_sweep_%s.json" % env_name), "w"))


if __name__ == "__main__":
    main()
