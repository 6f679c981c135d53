"""CartpoleEnv with GaussianGRUPolicy (hidden 32): CUDA-event timings (median of --reps after a warm-up, with the min and
max to show the spread) of the GRU rollout, loss/KL, BPTT gradient, Fisher-vector product (activation cache) and one
TRPO update (optimize_policy: gradient, 10 CG iterations, line search), at --lanes x --steps and at the reference
example's 4000 samples (40 lanes x 100 steps), and in the same run the Gaussian MLP (32, 32) passes on the first batch
shape.  Reads the card name and power limit in the same call and prints one JSON line.

    python scripts/gru_bench.py [--lanes 65536] [--steps 100] [--reps 5]
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

import gru_oracle as G  # noqa: E402
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
    return dict(median=float(np.median(ts)), min=float(np.min(ts)), max=float(np.max(ts)))


def gru_passes(N, T, reps):
    dev = torch.device("cuda:0")
    dims = ops.GRUDims(4, 32, 1, True)
    th = torch.tensor(G.init_params(G.GruDims(4, 32, 1, True), np.random.RandomState(3)), dtype=torch.float32,
                      device=dev)
    b = ops.LaneBatch(4, 1, N, T, dev)
    b.recurrent = True
    P_ = th.numel()
    out = torch.zeros(3, dtype=torch.float64, device=dev)
    g = torch.zeros(P_, dtype=torch.float64, device=dev)
    Hx = torch.zeros_like(g)
    x = torch.tensor(np.random.RandomState(1).randn(P_), device=dev)
    hc = b.hcache(32, 0)
    w = torch.zeros(2 * b.O + 4, dtype=torch.float64, device=dev)
    r = dict()
    r["rollout_s"] = timed(lambda i: ops.gru_rollout(dims, th, b, T, L.ENV_CARTPOLE, None, None, 1, i, 0), reps)
    ops.process_samples(b, w, 0.99, 1.0, drop_cut_paths=True)
    r["loss_kl_s"] = timed(lambda i: ops.loss_kl(L.LOSS_TRPO, th, dims, None, b, out), reps)
    r["grad_s"] = timed(lambda i: ops.grad(L.LOSS_TRPO, th, dims, None, b, g, out, hc), reps)
    r["fvp_cached_s"] = timed(lambda i: ops.fvp(th, dims, None, b, x, 1e-5, 1.0, Hx, hc), reps)
    return r


def gaussian_passes(N, T, reps):
    dev = torch.device("cuda:0")
    th = torch.tensor(P.init_params(P.Dims(4, (32, 32), 1), np.random.RandomState(3)), dtype=torch.float32, device=dev)
    b = ops.LaneBatch(4, 1, N, T, dev)
    dims = (4, 32, 32, 1)
    out = torch.zeros(3, dtype=torch.float64, device=dev)
    g = torch.zeros(th.numel(), dtype=torch.float64, device=dev)
    Hx = torch.zeros_like(g)
    x = torch.tensor(np.random.RandomState(1).randn(th.numel()), device=dev)
    hc = b.hcache(32, 32)
    w = torch.zeros(2 * b.O + 4, dtype=torch.float64, device=dev)
    r = dict()
    r["rollout_s"] = timed(lambda i: ops.rollout(L.ENV_CARTPOLE, th, 32, 32, 1e-6, b, T, None, None, 1, i, 0), reps)
    ops.process_samples(b, w, 0.99, 1.0, drop_cut_paths=True)
    r["loss_kl_s"] = timed(lambda i: ops.loss_kl(L.LOSS_TRPO, th, dims, 1e-6, b, out), reps)
    r["grad_s"] = timed(lambda i: ops.grad(L.LOSS_TRPO, th, dims, 1e-6, b, g, out, hc), reps)
    r["fvp_cached_s"] = timed(lambda i: ops.fvp(th, dims, 1e-6, b, x, 1e-5, 1.0, Hx, hc), reps)
    return r


def trpo_update(N, T, reps):
    from rllab_b200.algos.trpo import TRPO
    from rllab_b200.baselines.linear_feature_baseline import LinearFeatureBaseline
    from rllab_b200.envs.box2d.cartpole_env import CartpoleEnv
    from rllab_b200.envs.normalized_env import normalize
    from rllab_b200.policies.gaussian_gru_policy import GaussianGRUPolicy
    env = normalize(CartpoleEnv())
    pol = GaussianGRUPolicy(env_spec=env.spec, seed=3)
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
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    L.load()
    from rllab_b200.misc import logger
    logger.set_quiet(True)
    res = dict(what="gru_cartpole", card=card(), lanes=a.lanes, steps=a.steps)
    for tag, (N, T) in (("big", (a.lanes, a.steps)), ("example", (40, 100))):
        r = gru_passes(N, T, a.reps)
        r["trpo_optimize_s"] = trpo_update(N, T, a.reps)
        res.update({"gru_%s_%s" % (tag, k): v for k, v in r.items()})
        torch.cuda.empty_cache()
    res.update({"gaussian_big_" + k: v for k, v in gaussian_passes(a.lanes, a.steps, a.reps).items()})
    print(json.dumps(res))


if __name__ == "__main__":
    main()
