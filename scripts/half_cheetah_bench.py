"""HalfCheetah timings, with CUDA events after warm-up; prints the card name and power limit of the same run, and one
JSON line per measurement:
  * b200rl_rollout at 16 384 lanes x 500 steps, hidden 32 and 64 (env-steps/s);
  * b200rl_grad and b200rl_fvp (with the activation cache) at (obs 20, act 6) against (20, 3) on the same batch size;
  * one TRPO iteration (sampling, process_samples, baseline fit, optimize_policy) on 16 384 x 500 samples.

    python scripts/half_cheetah_bench.py [--lanes 16384] [--steps 500] [--reps 5]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import policy as P  # noqa: E402
from rllab_b200 import _lib as L, ops  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:   # noqa: BLE001
        out = ""
    return out or torch.cuda.get_device_name(0) + ", power limit unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lanes", type=int, default=16384)
    ap.add_argument("--steps", type=int, default=500)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    L.load()
    dev = torch.device("cuda:0")
    print("card:", card())
    for H in (32, 64):
        dims = P.Dims(20, (H, H), 6)
        th = torch.tensor(P.init_params(dims, np.random.RandomState(H)), dtype=torch.float32, device=dev)
        b = ops.LaneBatch(20, 6, a.lanes, a.steps, dev)
        ops.rollout(L.ENV_HALF_CHEETAH, th, H, H, 1e-6, b, 1000, None, None, 1, 0, 0)   # warm-up
        torch.cuda.synchronize()
        times = []
        for r in range(a.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            ops.rollout(L.ENV_HALF_CHEETAH, th, H, H, 1e-6, b, 1000, None, None, 1, r + 1, 0)
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1) / 1e3)
        t = float(np.median(times))
        print(json.dumps(dict(what="half_cheetah_rollout", hidden=H, lanes=a.lanes, steps=a.steps, seconds=t,
                              env_steps_per_s=a.lanes * a.steps / t, min_s=min(times), max_s=max(times))))
    # policy passes: the same batch size at act_dim 6 (HalfCheetah) and 3 (Hopper), rollout data of each env
    for H in (32, 64):
        for kind, A in ((L.ENV_HALF_CHEETAH, 6), (L.ENV_HOPPER, 3)):
            dims = P.Dims(20, (H, H), A)
            th = torch.tensor(P.init_params(dims, np.random.RandomState(H)), dtype=torch.float32, device=dev)
            b = ops.LaneBatch(20, A, a.lanes, a.steps, dev)
            ops.rollout(kind, th, H, H, 1e-6, b, 1000, None, None, 1, 0, 0)
            ops.process_samples(b, None, 0.99, 1.0)
            ops.center_advantages(b, True, False)
            dd = (20, H, H, A)
            g = torch.zeros(dims.P, dtype=torch.float64, device=dev)
            hc = torch.empty((2 * H, a.lanes * a.steps), dtype=torch.float32, device=dev)
            x = torch.tensor(np.random.RandomState(2).randn(dims.P), dtype=torch.float64, device=dev)
            Hx = torch.zeros_like(g)
            runs = dict(grad=lambda: ops.grad(L.LOSS_TRPO, th, dd, 1e-6, b, g, None, hc),
                        fvp=lambda: ops.fvp(th, dd, 1e-6, b, x, 1e-5, 1.0, Hx, hc))
            for name, fn in runs.items():
                fn()
                torch.cuda.synchronize()
                times = []
                for r in range(a.reps):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    fn()
                    e1.record()
                    torch.cuda.synchronize()
                    times.append(e0.elapsed_time(e1))
                print(json.dumps(dict(what="b200rl_" + name, obs_dim=20, act_dim=A, hidden=H, samples=a.lanes * a.steps,
                                      ms=float(np.median(times)), min_ms=min(times), max_ms=max(times))))
    # one TRPO iteration after a warm-up iteration
    import time
    from rllab_b200.algos.trpo import TRPO
    from rllab_b200.baselines.linear_feature_baseline import LinearFeatureBaseline
    from rllab_b200.envs.mujoco.half_cheetah_env import HalfCheetahEnv
    from rllab_b200.envs.normalized_env import normalize
    from rllab_b200.policies.gaussian_mlp_policy import GaussianMLPPolicy
    for H in (32, 64):
        env = normalize(HalfCheetahEnv())
        algo = TRPO(env=env, policy=GaussianMLPPolicy(env.spec, hidden_sizes=(H, H), seed=1),
                    baseline=LinearFeatureBaseline(env.spec), batch_size=a.lanes * a.steps, max_path_length=a.steps,
                    n_itr=1, discount=0.99, sampler_args=dict(n_envs=a.lanes, seed=1))
        algo.start_worker()
        algo.init_opt()
        walls = []
        for itr in range(3):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            sd = algo.sampler.process_samples(itr, algo.sampler.obtain_samples(itr))
            algo.optimize_policy(itr, sd)
            torch.cuda.synchronize()
            walls.append(time.perf_counter() - t0)
        print(json.dumps(dict(what="trpo_iteration", hidden=H, samples=a.lanes * a.steps, seconds=float(np.median(walls[1:])),
                              warmup_s=walls[0])))


if __name__ == "__main__":
    main()
