"""Times one 1000-step DDPG epoch (b200rl_ddpg_train, float32 nets) on CartPole at the example's configuration, with the
pool already above min_pool_size, for n_runs = 1, #SMs and 2 x #SMs runs in one launch.  CUDA events, median of 5 after
a warm-up; prints the card's name and power limit from the same run, and steps + updates per second per run and in
aggregate (one update per step, so steps + updates = 2 x steps).

    python scripts/ddpg_bench.py [--steps 1000] [--reps 5] [--f64]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from rllab_b200 import _lib as L  # noqa: E402
from rllab_b200 import ops  # noqa: E402
from rllab_b200.policies.deterministic_mlp_policy import init_values  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--f64", action="store_true")
    args = ap.parse_args()
    L.load()
    dev = torch.device("cuda:0")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    hp = ops.ddpg_hparams(n_updates_per_sample=1, max_path_length=100, min_pool_size=1000, replay_pool_size=1000000,
                          include_horizon_terminal_transitions=0, es_kind=L.ES_OU, discount=0.99, scale_reward=0.01,
                          soft_target_tau=0.001, qf_weight_decay=0.0, qf_learning_rate=1e-3, policy_weight_decay=0.0,
                          policy_learning_rate=1e-4, ou_mu=0.0, ou_theta=0.15, ou_sigma=0.3, gs_max_sigma=1.0,
                          gs_min_sigma=0.1, gs_decay_period=1e6)
    out = dict(card=card, sms=sms, steps=args.steps, f64=args.f64, results=[])
    for n_runs in (1, sms, 2 * sms):
        rng = np.random.RandomState(0)
        H = 32
        th = np.concatenate([init_values([(4, H), (H,), (H, H), (H,), (H, 1), (1,)], rng),
                             init_values([(4, H), (H,), (H + 1, H), (H,), (H, 1), (1,)], rng)])
        nets = np.tile(np.stack([th, 0 * th, 0 * th, th])[None], (n_runs, 1, 1))
        runs = ops.DdpgRuns(L.ENV_CARTPOLE, 4, 1, n_runs, hp, nets, 1, dev, f64=args.f64, es_cap=1)
        runs.train(1000)                # fill the pool to min_pool_size (training starts at the last of these steps)
        runs.train(args.steps)          # warm-up epoch
        runs.take_stats()
        times = []
        for _ in range(args.reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            runs.train(args.steps)
            b.record()
            torch.cuda.synchronize()
            times.append(a.elapsed_time(b) / 1e3)
            runs.take_stats()
        t = float(np.median(times))
        per_run = 2 * args.steps / t
        out["results"].append(dict(n_runs=n_runs, epoch_s=t, steps_updates_per_s_per_run=per_run,
                                   steps_updates_per_s_total=per_run * n_runs, times=times))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
