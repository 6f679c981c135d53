"""Generate tests/golden/reference_reps_golden.npz: the reference's own REPS.optimize_policy (rllab/algos/reps.py), run
verbatim through oracle/ref_shims.py on a fixed small set of paths, two iterations per case (the second warm-started from
the first's eta and v, as the reference's train loop does).

Stand-ins, since the reference's Theano graph cannot be built here:
  * opt_info (f_dual, f_dual_grad, f_loss, f_loss_grad, f_kl) are float64 NumPy callables from tests/reps_oracle.py and
    oracle/policy.py, with the reference's argument lists;
  * the policy is a NumPy GaussianMLPPolicy stand-in (flat float64 parameters, oracle/policy.py forward);
  * the optimizer is scipy.optimize.fmin_l_bfgs_b wrapped to drop `disp` (scipy >= 1.18 no longer takes it);
  * init_opt's draws are restated (param_eta = 15, param_v = np.random.rand(2 O + 4)) after a fixed seed.

Recorded per case <c> (keys "<c>/..."): the paths (obs_flat, act_flat, rew_flat, mean_flat, path_len), log_std, theta0,
hidden sizes, the constructor arguments (args_*), and per iteration <i>: feat_diff (as the reference built it), eta_before,
v_before, eta_after, v_after, theta_after and the tabular values (tab_<key>).

Run:  python tests/golden/make_reps_golden.py        (needs the reference tree; the tests only read the committed file)
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

import reps_oracle as K  # noqa: E402
from oracle import policy as OP  # noqa: E402
from oracle import ref_shims  # noqa: E402

O, A, HIDDEN = 4, 1, (8, 8)
PATH_LENS = (37, 12, 50, 1, 28, 9)
CASES = {
    "defaults": dict(),
    "regularized": dict(epsilon=0.1, L2_reg_dual=1e-3, L2_reg_loss=1e-2, max_opt_itr=10),
}
KEYS = ("LossBefore", "LossAfter", "DualBefore", "DualAfter", "MeanKL")


class _Dist(object):
    dist_info_keys = ["mean", "log_std"]


class NumpyGaussianMLPPolicy(object):
    """The surface REPS.optimize_policy uses."""
    recurrent = False
    state_info_keys = []
    distribution = _Dist()

    def __init__(self, dims, theta):
        self.dims = dims
        self.theta = np.array(theta, np.float64)

    def get_param_values(self, **tags):
        return self.theta.copy()

    def set_param_values(self, flat, **tags):
        self.theta = np.array(flat, np.float64).reshape(-1)


def make_paths(rng, dims, theta):
    paths = []
    for n in PATH_LENS:
        obs = rng.randn(n, O) * 3.0
        big = rng.rand(n, O) < 0.1
        obs[big] = np.sign(rng.randn(int(big.sum()))) * rng.uniform(10.0, 15.0, int(big.sum()))  # beyond the clip
        mean, log_std = OP.forward(theta, obs, dims)
        act = mean + np.exp(log_std) * rng.randn(n, A)
        paths.append(dict(observations=obs, actions=act, rewards=rng.rand(n) * 2.0 - 0.5,
                          agent_infos=dict(mean=mean, log_std=np.tile(log_std, (n, 1)))))
    return paths


def opt_info(algo, dims):
    """Oracle-backed callables with the argument lists of the compiled functions of reps.py:133-197."""
    pol = algo.policy

    def batch(obs, act, mean=None, log_std=None):
        return dict(obs=obs, actions=act, old_mean=mean, old_log_std=log_std)

    def f_dual(rew, fd, eta, v):
        return np.float64(K.dual(eta, v, rew, fd, algo.epsilon, algo.L2_reg_dual))

    def f_dual_grad(rew, fd, eta, v):
        g = K.dual_grad(eta, v, rew, fd, algo.epsilon, algo.L2_reg_dual)
        return [g[0], g[1:]]

    def f_loss(rew, obs, fd, act, eta, v):
        w = K.weights(eta, v, rew, fd)
        return np.float64(K.policy_loss(pol.theta, batch(obs, act), w, dims, algo.L2_reg_loss))

    def f_loss_grad(rew, obs, fd, act, eta, v):
        w = K.weights(eta, v, rew, fd)
        return [K.policy_grad(pol.theta, batch(obs, act), w, dims, algo.L2_reg_loss)]

    def f_kl(obs, act, old_mean, old_log_std):
        mean, log_std = OP.forward(pol.theta, obs, dims)
        return np.float64(np.mean(OP.kl(old_mean, old_log_std, mean, log_std * np.ones_like(mean))))

    return dict(f_dual=f_dual, f_dual_grad=f_dual_grad, f_loss=f_loss, f_loss_grad=f_loss_grad, f_kl=f_kl)


def run_case(name, kw, seed):
    import scipy.optimize
    import rllab.algos.reps as reps
    import rllab.misc.logger as rlogger

    def lbfgs(**k):
        k.pop("disp", None)
        return scipy.optimize.fmin_l_bfgs_b(**k)

    rng = np.random.RandomState(seed)
    dims = OP.Dims(O, HIDDEN, A)
    theta0 = OP.init_params(dims, rng)
    theta0[-A:] = -0.3
    paths = make_paths(rng, dims, theta0)
    policy = NumpyGaussianMLPPolicy(dims, theta0)
    algo = reps.REPS(env=None, policy=policy, baseline=None, optimizer=lbfgs, **kw)
    np.random.seed(seed)
    algo.param_eta = 15.                                    # init_opt, reps.py:55-57
    algo.param_v = np.random.rand(O * 2 + 4)
    algo.opt_info = opt_info(algo, dims)
    samples_data = dict(
        rewards=np.concatenate([p["rewards"] for p in paths]),
        actions=np.vstack([p["actions"] for p in paths]),
        observations=np.vstack([p["observations"] for p in paths]),
        agent_infos=dict(mean=np.vstack([p["agent_infos"]["mean"] for p in paths]),
                         log_std=np.vstack([p["agent_infos"]["log_std"] for p in paths])),
        paths=paths)
    out = {}
    p = name + "/"
    out[p + "obs_flat"] = samples_data["observations"]
    out[p + "act_flat"] = samples_data["actions"]
    out[p + "rew_flat"] = samples_data["rewards"]
    out[p + "mean_flat"] = samples_data["agent_infos"]["mean"]
    out[p + "log_std"] = paths[0]["agent_infos"]["log_std"][0]
    out[p + "path_len"] = np.array(PATH_LENS)
    out[p + "theta0"] = theta0
    out[p + "hidden"] = np.array(HIDDEN)
    for k, v in sorted(dict(epsilon=algo.epsilon, L2_reg_dual=algo.L2_reg_dual, L2_reg_loss=algo.L2_reg_loss,
                            max_opt_itr=algo.max_opt_itr).items()):
        out[p + "args_" + k] = np.array(v)
    orig_rec = rlogger.record_tabular
    for it in range(2):
        q = "%s%d/" % (p, it)
        tab, seen = {}, {}
        f_dual = algo.opt_info["f_dual"]

        def spy(rew, fd, eta, v, f_dual=f_dual):
            seen.setdefault("fd", np.array(fd))
            return f_dual(rew, fd, eta, v)
        algo.opt_info["f_dual"] = spy
        out[q + "eta_before"] = np.array(algo.param_eta)
        out[q + "v_before"] = np.array(algo.param_v)
        rlogger.record_tabular = lambda key, val: tab.__setitem__(key, val)
        try:
            algo.optimize_policy(it, samples_data)
        finally:
            rlogger.record_tabular = orig_rec
            algo.opt_info["f_dual"] = f_dual
        out[q + "feat_diff"] = seen["fd"]
        out[q + "eta_after"] = np.array(algo.param_eta)
        out[q + "v_after"] = np.array(algo.param_v)
        out[q + "theta_after"] = policy.get_param_values()
        for key in KEYS:
            out[q + "tab_" + key] = np.array(tab[key])
    return out


def main():
    ref_shims.install()
    if not hasattr(np, "float"):
        np.float = float                  # reps.py:262 (removed from NumPy 1.24)
    out = {}
    for i, (name, kw) in enumerate(sorted(CASES.items())):
        out.update(run_case(name, kw, 20 + i))
        print(name, [(float(out["%s/%d/eta_after" % (name, j)]), float(out["%s/%d/tab_LossAfter" % (name, j)]))
                     for j in range(2)])
    path = os.path.join(HERE, "reference_reps_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path)


if __name__ == "__main__":
    main()
