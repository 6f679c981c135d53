"""Generate tests/golden/oracle_cartpole_ddpg_curve.json: the float64 ORACLE's DDPG learning curves for the
configuration of examples/ddpg_cartpole.py -- normalize(CartpoleEnv()), DeterministicMLPPolicy and
ContinuousMLPQFunction (32, 32), OUStrategy defaults, batch 32, epoch_length 1000, min_pool_size 10000, max_path_length
100, discount 0.99, scale_reward 0.01, learning rates 1e-3 (Q) / 1e-4 (policy), soft_target_tau 0.001, one update per
step -- with a reduced n_epochs, over five seeds.  AverageReturn is recorded for every epoch that evaluates (the pool
has min_pool_size samples), from noise-free lanes as DDPG.evaluate samples them: ceil(10000 / 100) lanes of 100 steps,
whole paths only.

The seed sets the initial networks (np.random.RandomState(seed)) and the reset draws; the exploration noise and the
minibatch indices come from the Philox streams of include/b200rl.h keyed by the seed (tests/ddpg_oracle.py).  The GPU
trajectories diverge from these after a few steps (float32 env, chaotic dynamics), so the GPU test compares with the band
of these curves, not value by value.

Run (CPU only):  python tests/golden/make_cartpole_ddpg_curve.py [n_epochs] [seeds...]
"""
import json
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

import ddpg_oracle as K  # noqa: E402
from oracle import envs as E  # noqa: E402

HP = dict(n_updates_per_sample=1, max_path_length=100, min_pool_size=10000, replay_pool_size=1000000,
          include_horizon_terminal_transitions=0, es_kind=0, discount=0.99, scale_reward=0.01, soft_target_tau=0.001,
          qf_weight_decay=0.0, qf_learning_rate=1e-3, policy_weight_decay=0.0, policy_learning_rate=1e-4, ou_mu=0.0,
          ou_theta=0.15, ou_sigma=0.3, gs_max_sigma=1.0, gs_min_sigma=0.1, gs_decay_period=1e6)
EPOCH_LENGTH, EVAL_SAMPLES = 1000, 10000
OUT = os.path.join(HERE, "oracle_cartpole_ddpg_curve.json")


def evaluate(env, d, theta_p, rng, T=100):
    """Noise-free lanes with auto-reset; the returns of the whole paths (a lane's path cut by the buffer is dropped)."""
    N = -(-EVAL_SAMPLES // T)
    s = env.reset(rng.rand(4, N).astype(np.float32))
    plen = np.zeros(N, np.int64)
    ret = np.zeros(N)
    returns = []
    for _ in range(T):
        _, _, mu = K.pi_forward(d, theta_p, env.obs(s).T.astype(np.float64))
        u = env.scale_action(mu.T.astype(np.float32))
        s, r, done = env.step(s, u)
        ret += r
        plen += 1
        end = done | (plen >= T)
        returns.extend(ret[end].tolist())
        if end.any():
            fresh = env.reset(rng.rand(4, N).astype(np.float32))
            s[:, end] = fresh[:, end]
            plen[end] = 0
            ret[end] = 0.0
    return float(np.mean(returns))


def run(seed, n_epochs):
    d = K.Dims(4, 1)
    rng = np.random.RandomState(seed)
    th = np.concatenate([K.init_params(d.pshapes, rng), K.init_params(d.qshapes, rng)])
    env = E.make("cartpole", np.float32)
    rows = HP["replay_pool_size"]
    n_pool = n_epochs * EPOCH_LENGTH
    st = dict(nets=np.stack([th, 0 * th, 0 * th, th]), env_state=None, obs=None, ou=np.zeros(1), path_return=0.0,
              path_length=0, terminal=2, itr=0, adam_t=0, top=0, bottom=0, size=0,
              pool=dict(obs=np.zeros((n_pool, 4), np.float32), act=np.zeros((n_pool, 1), np.float32),
                        rew=np.zeros(n_pool, np.float32), term=np.zeros(n_pool, np.uint8)))
    assert n_pool <= rows

    def env_reset(itr):
        s = env.reset(rng.rand(4, 1).astype(np.float32))[:, 0]
        return s, env.obs(s)

    def env_step(s, act):
        s2, r, done = env.step(s, env.scale_action(act.reshape(1, 1))[:, 0])
        return s2, env.obs(s2), float(r), bool(done)

    hp = dict(HP, replay_pool_size=n_pool)   # the pool never wraps within n_epochs: same draws as a 1e6-row pool
    curve = {}
    for epoch in range(n_epochs):
        for _ in range(EPOCH_LENGTH):
            K.train_step(d, st, hp, seed, 0, env_reset, env_step)
        if st["size"] >= HP["min_pool_size"]:
            curve[epoch] = evaluate(env, d, st["nets"][0][:d.PP], rng)
    return curve


def main(n_epochs, seeds):
    from multiprocessing import Pool
    t0 = time.time()
    with Pool(len(seeds)) as pool:          # one process per seed: the seeds are independent
        res = pool.starmap(run, [(seed, n_epochs) for seed in seeds])
    curves = {str(seed): c for seed, c in zip(seeds, res)}
    for seed in seeds:
        print(seed, {k: round(v, 1) for k, v in curves[str(seed)].items()}, flush=True)
    print("%.0f s" % (time.time() - t0))
    with open(OUT, "w") as f:
        json.dump(dict(config=dict(HP, epoch_length=EPOCH_LENGTH, eval_samples=EVAL_SAMPLES, batch_size=32,
                                   env="normalize(CartpoleEnv())", n_epochs=n_epochs,
                                   arithmetic="float64 NumPy oracle (tests/ddpg_oracle.py), float32 env"),
                       AverageReturn=curves), f, indent=1)


if __name__ == "__main__":
    main(int(sys.argv[1]) if len(sys.argv) > 1 else 20, [int(s) for s in sys.argv[2:]] or [1, 2, 3, 4, 5])
