"""Generate tests/golden/oracle_cartpole_v0_gru_trpo_curve.json: the float64 ORACLE's TRPO learning curves on
normalize(GymEnv("CartPole-v0")) with CategoricalGRUPolicy (hidden 32, one-hot previous action in the input),
LinearFeatureBaseline, batch 4000 = 20 lanes x 200 steps, max_path_length 200, discount 0.99, GAE lambda 1, step_size
0.01, cg_iters 10, whole paths only, over five seeds.  The seed sets the initial policy and the np.random streams of
the action and reset draws, which are not the GPU's Philox streams: the GPU test compares its curve with the band of
these curves, not value by value.

Run (CPU only):  python tests/golden/make_cartpole_v0_gru_curve.py [n_itr] [seeds...]
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

import categorical_gru_oracle as C  # noqa: E402
from oracle import sampler as S  # noqa: E402

N, T = 20, 200
DISCOUNT, GAE_LAMBDA, STEP_SIZE, CG_ITERS = 0.99, 1.0, 0.01, 10
OUT = os.path.join(HERE, "oracle_cartpole_v0_gru_trpo_curve.json")


def run(seed, n_itr):
    dims = C.CatGruDims(4, 32, 2, True)
    rng = np.random.RandomState(seed)
    theta = C.init_params(dims, rng)
    coeffs = None
    rets = []
    for itr in range(n_itr):
        traj = C.rollout_cartpole_v0(theta, dims, N, T, T, rng.rand(T, N), rng.rand(T + 1, 4, N))
        out = S.process_samples_lanes(traj, coeffs, DISCOUNT, GAE_LAMBDA, center_adv=True, drop_cut=True)
        valid = out["valid"]
        coeffs = S.lfb_fit_lanes(traj["obs"], traj["tstep"], out["ret"], valid=valid)
        lanes = dict(obs=traj["obs"], act=traj["act"], tstep=traj["tstep"], adv=out["adv"], old_prob=traj["mean"],
                     valid=valid)
        theta, _ = C.trpo_step(theta, lanes, dims, STEP_SIZE, CG_ITERS)
        rets.append(float(out["stats"]["AverageReturn"]))
    return rets


def main(n_itr, seeds):
    curves = {}
    for seed in seeds:
        t0 = time.time()
        curves[str(seed)] = run(seed, n_itr)
        print(seed, "%.0f s" % (time.time() - t0), [round(r, 1) for r in curves[str(seed)]], flush=True)
    with open(OUT, "w") as f:
        json.dump(dict(config=dict(env="GymEnv('CartPole-v0') (normalized)", lanes=N, horizon=T, hidden=32,
                                   state_include_action=True, discount=DISCOUNT, gae_lambda=GAE_LAMBDA,
                                   step_size=STEP_SIZE, cg_iters=CG_ITERS, baseline="LinearFeatureBaseline",
                                   whole_paths=True, hvp="Gauss-Newton J^T M J x (tests/categorical_gru_oracle.py)",
                                   arithmetic="float64 NumPy oracle (tests/categorical_gru_oracle.py, oracle/optim.py)"),
                       AverageReturn=curves), f, indent=1)


if __name__ == "__main__":
    main(int(sys.argv[1]) if len(sys.argv) > 1 else 20, [int(s) for s in sys.argv[2:]] or [1, 2, 3, 4, 5])
