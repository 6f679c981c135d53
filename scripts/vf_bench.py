"""Time the GaussianMLPBaseline passes (csrc/vf.cu) on the bench batches and print one JSON line per batch.

  cfg2   CartPole 65 536 lanes x 200 steps      cfg3   Swimmer 16 384 lanes x 500 steps

For each batch, after warm-up, with CUDA events over at least a second of repeated work: one forward pass, one
loss+gradient pass (trust region on), the normalisation-statistics pass, and b200rl_grad of the policy on the same batch
for context; the FP32 peak measured in the same run (b200rl_bench_ffma2); one whole default fit (wall time, device
passes, the host time between them).  Card name and power limit are read with nvidia-smi in the same run.

Usage:  python scripts/vf_bench.py [--out FILE]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=20).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in q.split(",")]
        return name, power
    except Exception:
        return None, None


def timed(fn, min_s=1.0):
    import torch
    fn()
    torch.cuda.synchronize()
    reps = 1
    while True:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1)
        if ms >= min_s * 1e3:
            return ms / reps
        reps *= 2 if ms < 100 else max(2, int(min_s * 1e3 / ms) + 1)


def run(cfg, env_name, n_envs, T):
    import numpy as np
    import torch
    import bench
    from rllab_b200 import _lib as L
    from rllab_b200 import ops
    from rllab_b200.algos.trpo import TRPO
    from rllab_b200.baselines.gaussian_mlp_baseline import GaussianMLPBaseline
    from rllab_b200.policies.gaussian_mlp_policy import GaussianMLPPolicy
    env = bench.make_env(env_name)
    policy = GaussianMLPPolicy(env.spec, hidden_sizes=(32, 32), seed=1)
    np.random.seed(2)
    baseline = GaussianMLPBaseline(env.spec)
    algo = TRPO(env=env, policy=policy, baseline=baseline, batch_size=n_envs * T, max_path_length=T, n_itr=1,
                discount=0.99, sampler_args=dict(n_envs=n_envs, seed=7))
    algo.start_worker()
    algo.init_opt()
    paths = algo.sampler.obtain_samples(0)
    algo.sampler.process_samples(0, paths)           # predict + fit once (warm-up, normalisation constants set)
    torch.cuda.synchronize()
    b = paths.lane_batch
    reg = baseline.regressor
    d = reg._ensure_device()
    O, B, P = b.O, b.B, reg.n_params
    flags = b.flags.view(-1)
    y = b.ret.view(-1)
    mu = torch.empty(B, dtype=torch.float32, device=b.device)
    g = torch.zeros(P, dtype=torch.float64, device=b.device)
    lo = torch.zeros(3, dtype=torch.float64, device=b.device)
    acc = torch.zeros(2 * O + 3, dtype=torch.float64, device=b.device)
    st = torch.zeros(2 * O + 2, dtype=torch.float64, device=b.device)
    ops.vf_norm_stats(O, B, b.obs, y, flags, ops.VF_STATS_ALL, acc, st)
    cnt = acc[O + 1:O + 2]
    ops.vf_forward(d["theta32"], O, B, b.obs, st, mu, False)

    t_fwd = timed(lambda: ops.vf_forward(d["theta32"], O, B, b.obs, st, mu, False))
    t_grad = timed(lambda: ops.vf_loss_grad(d["theta32"], O, B, b.obs, y, flags, st, mu, 0.0, 1.0, True, 1.0, cnt, g,
                                            lo))
    t_loss = timed(lambda: ops.vf_loss_grad(d["theta32"], O, B, b.obs, y, flags, st, mu, 0.0, 1.0, True, 1.0, cnt, None,
                                            lo))
    t_stats = timed(lambda: ops.vf_norm_stats(O, B, b.obs, y, flags, ops.VF_STATS_ALL, acc, st))
    pg = torch.zeros(policy.n_params, dtype=torch.float64, device=b.device)
    t_pgrad = timed(lambda: ops.grad(L.LOSS_TRPO, policy.theta32, policy.dims, policy.min_std, b, pg, lo))
    sink = torch.zeros(4, dtype=torch.float32, device=b.device)
    fma = ctypes.c_longlong(0)
    t_ffma = timed(lambda: L.call("b200rl_bench_ffma2", 4096, L.ptr(sink), ctypes.byref(fma),
                                  ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), 0.5)
    peak = 2.0 * fma.value / (t_ffma * 1e-3) / 1e12

    # one whole default fit (penalty state as after the warm-up fit)
    torch.cuda.synchronize()
    w0 = time.perf_counter()
    reg.fit_device(b.obs, y, flags, None)
    torch.cuda.synchronize()
    fit_s = time.perf_counter() - w0
    n_evals = reg.last_fit["n_evals"]
    n_grad = sum(t[2] for t in reg._optimizer.terminations)
    n_loss = n_evals - n_grad
    dev_s = (n_grad * t_grad + n_loss * t_loss + t_stats + t_fwd) * 1e-3
    Fh = 2.0 * (O * 32 + 32 * 32 + 32)                       # flops of one forward per sample
    Fg = 2 * Fh + 2.0 * (32 + 32 * 32)                       # + backward (d2, d1) and the weight-gradient Gram products
    n_valid = float(acc[O + 1].item())
    name, power = card()
    return dict(cfg=cfg, env=env_name, lanes=n_envs, steps=T, samples=B, valid_samples=n_valid, gpu=name,
                power_limit=power, fp32_peak_tflops=round(peak, 2),
                forward_ms=round(t_fwd, 4), forward_tflops=round(Fh * B / t_fwd / 1e9, 2),
                loss_ms=round(t_loss, 4),
                loss_grad_ms=round(t_grad, 4), loss_grad_tflops=round(Fg * B / t_grad / 1e9, 2),
                loss_grad_peak_share=round(Fg * B / t_grad / 1e9 / peak, 3),
                flops_per_sample=dict(forward=Fh, loss_grad=Fg),
                stats_ms=round(t_stats, 4), policy_grad_ms=round(t_pgrad, 4),
                fit_s=round(fit_s, 3), fit_passes=dict(grad=n_grad, loss=n_loss),
                fit_device_s_est=round(dev_s, 3), fit_host_s_est=round(fit_s - dev_s, 3),
                penalties=reg._optimizer.tried_penalties)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from rllab_b200.misc import logger
    logger.set_quiet(True)
    res = [run("cfg2", "cartpole", 65536, 200), run("cfg3", "swimmer", 16384, 500)]
    for r in res:
        print(json.dumps(r))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
