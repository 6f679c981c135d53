"""Generate tests/golden/reference_vf_golden.npz: the reference's own PenaltyLbfgsOptimizer.optimize and
LbfgsOptimizer.optimize (rllab/optimizers/penalty_lbfgs_optimizer.py, lbfgs_optimizer.py), run verbatim through
oracle/ref_shims.py with the float64 callables of tests/vf_oracle.py injected into _opt_fun / _target (the Theano
functions they would compile), on small fixed datasets.

Per case <name>: <name>_theta0, _xs, _ys (inputs), _penalty0 (the penalty before the fit), _penalties (tried, in
order; recorded by wrapping fmin_l_bfgs_b), _theta (final), _penalty (persisted), _loss (before, after), _kl (after).

Run:  python tests/golden/make_vf_golden.py        (needs the reference tree; the tests only read the committed file)
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

from oracle import ref_shims  # noqa: E402
import vf_oracle as V  # noqa: E402

# name: (obs_dim, n, optimizer kind, optimizer kwargs, learn_std, initial log_std, y scale, penalty0)
CASES = {
    "pen_decrease": (4, 400, "penalty", dict(), True, 0.0, 1.0, 100.0),
    "pen_increase": (3, 300, "penalty", dict(), True, 0.0, 10.0, 1e-2),
    "pen_maxitr": (4, 300, "penalty", dict(max_penalty_itr=3), True, 0.0, 10.0, 1e-2),
    "pen_noadapt": (6, 250, "penalty", dict(adapt_penalty=False), True, 0.3, 3.0, 1.0),
    "pen_fixedstd": (2, 300, "penalty", dict(), False, 0.0, 5.0, 1.0),
    "lbfgs20": (4, 300, "lbfgs", dict(max_opt_itr=20), True, 0.0, 3.0, None),
    "lbfgs3": (13, 200, "lbfgs", dict(max_opt_itr=3), True, 0.0, 3.0, None),
}


def dataset(O, n, y_scale, seed):
    rng = np.random.RandomState(seed)
    xs = rng.randn(n, O) * (1.0 + 0.5 * np.arange(O)) + np.arange(O)
    ys = np.sin(xs[:, 0]) * y_scale + 0.3 * xs[:, -1] * y_scale + rng.randn(n) * 0.2 * y_scale + 1.0
    return xs, ys


def main():
    ref_shims.install()
    import scipy.optimize
    import rllab.optimizers.penalty_lbfgs_optimizer as plo
    import rllab.optimizers.lbfgs_optimizer as lo

    out = {}
    for i, (name, (O, n, kind, kw, learn_std, ls0, y_scale, pen0)) in enumerate(sorted(CASES.items())):
        xs, ys = dataset(O, n, y_scale, 100 + i)
        theta0 = V.init_params(O, np.random.RandomState(200 + i))
        theta0[-1] = ls0
        tried = []
        orig = scipy.optimize.fmin_l_bfgs_b

        def recording(func, x0, **k):
            cells = dict(zip(func.__code__.co_freevars, func.__closure__))   # gen_f_opt(penalty)'s closure
            tried.append(float(cells["penalty"].cell_contents))
            return orig(func, x0, **k)
        if kind == "penalty":
            opt = plo.PenaltyLbfgsOptimizer(initial_penalty=pen0, **kw)
            plo.scipy.optimize.fmin_l_bfgs_b = recording
        else:
            opt = lo.LbfgsOptimizer(**kw)
        try:
            th, stats, info = V.fit(theta0, xs, ys, O, opt, use_trust_region=(kind == "penalty"), learn_std=learn_std)
        finally:
            plo.scipy.optimize.fmin_l_bfgs_b = orig
        out[name + "_theta0"] = theta0
        out[name + "_xs"] = xs
        out[name + "_ys"] = ys
        out[name + "_theta"] = th
        out[name + "_loss"] = np.array([info["LossBefore"], info["LossAfter"]])
        if kind == "penalty":
            out[name + "_penalty0"] = np.array(pen0)
            out[name + "_penalties"] = np.array(tried)
            out[name + "_penalty"] = np.array(float(opt._penalty))
            out[name + "_kl"] = np.array(info["MeanKL"])
        print(name, tried, info)
    path = os.path.join(HERE, "reference_vf_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path)


if __name__ == "__main__":
    main()
