"""CartPole-v0 with CategoricalMLPPolicy (32, 32): CUDA-event timings (median of --reps after a warm-up) of the
categorical rollout, process_samples, loss/KL, gradient, Fisher-vector product (activation cache) and one TRPO update
(optimize_policy: gradient, 10 CG iterations, line search), and in the same run the Gaussian passes of the Box CartPole
on the same batch shape.  Reads the card name and power limit in the same call and prints one JSON line.

    python scripts/categorical_bench.py [--lanes 65536] [--steps 200] [--reps 5]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import categorical_oracle as C  # noqa: E402
from oracle import policy as P  # noqa: E402
from rllab_b200 import _lib as L, ops  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:   # noqa: BLE001
        out = ""
    return out or torch.cuda.get_device_name(0) + ", power limit unknown"


def timed(fn, reps):
    fn(0)
    torch.cuda.synchronize()
    ts = []
    for r in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn(r + 1)
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) / 1e3)
    return float(np.median(ts))


def passes(kind, th, dims, min_std, b, reps):
    P_ = th.numel()
    out = torch.zeros(3, dtype=torch.float64, device=th.device)
    g = torch.zeros(P_, dtype=torch.float64, device=th.device)
    Hx = torch.zeros_like(g)
    x = torch.tensor(np.random.RandomState(1).randn(P_), device=th.device)
    hc = b.hcache(32, 32)
    w = torch.zeros(2 * b.O + 4, dtype=torch.float64, device=th.device)
    r = dict()
    r["rollout_s"] = timed(lambda i: ops.rollout(kind, th, 32, 32, min_std, b, 200, None, None, 1, i, 0), reps)
    r["process_samples_s"] = timed(lambda i: ops.process_samples(b, w, 0.99, 1.0, drop_cut_paths=True), reps)
    r["loss_kl_s"] = timed(lambda i: ops.loss_kl(L.LOSS_TRPO, th, dims, min_std, b, out), reps)
    r["grad_s"] = timed(lambda i: ops.grad(L.LOSS_TRPO, th, dims, min_std, b, g, out, hc), reps)
    r["fvp_cached_s"] = timed(lambda i: ops.fvp(th, dims, min_std, b, x, 1e-5, 1.0, Hx, hc), reps)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lanes", type=int, default=65536)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    L.load()
    from rllab_b200.misc import logger
    logger.set_quiet(True)
    dev = torch.device("cuda:0")
    N, T = a.lanes, a.steps
    res = dict(what="categorical_cartpole_v0", card=card(), lanes=N, steps=T, samples=N * T)
    # categorical CartPole-v0
    th = torch.tensor(C.init_params(C.CatDims(4, (32, 32), 2), np.random.RandomState(3)), dtype=torch.float32,
                      device=dev)
    b = ops.LaneBatch(4, 2, N, T, dev)
    b.categorical = True
    cat = passes(L.ENV_GYM_CARTPOLE, th, ops.CategoricalDims(4, 32, 32, 2), None, b, a.reps)
    del b
    # Gaussian Box CartPole, same batch shape
    thg = torch.tensor(P.init_params(P.Dims(4, (32, 32), 1), np.random.RandomState(3)), dtype=torch.float32,
                       device=dev)
    bg = ops.LaneBatch(4, 1, N, T, dev)
    gau = passes(L.ENV_CARTPOLE, thg, (4, 32, 32, 1), 1e-6, bg, a.reps)
    del bg
    torch.cuda.empty_cache()
    # one TRPO update of the reference example's configuration at this batch size
    from rllab_b200.algos.trpo import TRPO
    from rllab_b200.baselines.linear_feature_baseline import LinearFeatureBaseline
    from rllab_b200.envs.gym_env import GymEnv
    from rllab_b200.envs.normalized_env import normalize
    from rllab_b200.policies.categorical_mlp_policy import CategoricalMLPPolicy
    env = normalize(GymEnv("CartPole-v0"))
    pol = CategoricalMLPPolicy(env_spec=env.spec, hidden_sizes=(32, 32), seed=3)
    algo = TRPO(env=env, policy=pol, baseline=LinearFeatureBaseline(env_spec=env.spec), batch_size=N * T,
                max_path_length=T, n_itr=1, discount=0.99, step_size=0.01, sampler_args=dict(n_envs=N, seed=7))
    algo.start_worker()
    algo.init_opt()
    sd = algo.sampler.process_samples(0, algo.sampler.obtain_samples(0))
    theta0 = pol.get_param_values()

    def trpo(i):
        pol.set_param_values(theta0)
        algo.optimize_policy(0, sd)
    cat["trpo_optimize_s"] = timed(trpo, a.reps)
    res.update({"categorical_" + k: v for k, v in cat.items()})
    res.update({"gaussian_" + k: v for k, v in gau.items()})
    res["categorical_rollout_env_steps_per_s"] = N * T / cat["rollout_s"]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
