"""Generate tests/golden/reference_cem_golden.npz: the reference's own CEM.train (rllab/algos/cem.py), run verbatim
through oracle/ref_shims.py on normalize(PointEnv()) with a float64 NumPy GaussianMLPPolicy stand-in built from
oracle/policy.py, in one process (n_parallel = 1).

Recorded per case <c> and iteration <i> (keys "<c>/<i>/..."): xs (the members' parameter rows, from a wrapped
run_collect), fs (fitness), ustat (undiscounted-return statistic), rewards of every episode (ragged: rew_flat + rew_len,
member-major then eval), cur_mean / cur_std (the snapshot of save_itr_params), best_x (the policy's row at the snapshot) and
the CEM tabular values (tab_<key>).  Per case: n_itr, n_best, n_evals, discount, the constructor arguments (args_*).

Run:  python tests/golden/make_cem_golden.py        (needs the reference tree; the tests only read the committed file)
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import policy as OP  # noqa: E402
from oracle import ref_shims  # noqa: E402

# name: CEM keyword arguments (every case: n_itr = 3, hidden (8, 8))
CASES = {
    "evals1_decay": dict(n_samples=20, n_evals=1, best_frac=0.2, max_path_length=30, extra_std=0.5,
                         extra_decay_time=2, init_std=0.7),
    "evals3_best1": dict(n_samples=15, n_evals=3, best_frac=0.05, max_path_length=25, discount=0.9),
    "batch": dict(n_samples=30, batch_size=200, n_evals=2, best_frac=0.1, max_path_length=25, extra_decay_time=4),
}
KEYS = ("Iteration", "CurStdMean", "AverageReturn", "StdReturn", "MaxReturn", "MinReturn", "AverageDiscountedReturn",
        "NumTrajs", "AvgTrajLen", "AveragePolicyStd")


class NumpyGaussianMLPPolicy(object):
    """The surface CEM and rollout() use: get_action, get/set_param_values, reset, terminate, log_diagnostics."""

    def __init__(self, dims, theta):
        self.dims = dims
        self.theta = np.array(theta, np.float64)

    def get_param_values(self, **tags):
        return self.theta.copy()

    def set_param_values(self, flat, **tags):
        self.theta = np.array(flat, np.float64).reshape(-1)

    def reset(self, dones=None):
        pass

    def terminate(self):
        pass

    def get_action(self, observation):
        mean, log_std = OP.forward(self.theta, np.asarray(observation)[None], self.dims)
        rnd = np.random.normal(size=mean.shape)
        action = rnd * np.exp(log_std) + mean           # gaussian_mlp_policy.py:125-130
        return action[0], dict(mean=mean[0], log_std=log_std)

    def log_diagnostics(self, paths):
        # every step of every path carries the (state-independent) log_std of its member
        from rllab.misc import logger
        stds = np.exp(np.concatenate([np.asarray(p["agent_infos"]["log_std"]) for p in paths]))
        logger.record_tabular('AveragePolicyStd', float(stds.mean()))


def run_case(name, kw, seed):
    import rllab.algos.cem as cem
    import rllab.misc.logger as rlogger
    from rllab.envs.normalized_env import normalize
    from rllab.sampler import stateful_pool
    from examples.point_env import PointEnv

    np.random.seed(seed)
    env = normalize(PointEnv())
    dims = OP.Dims(2, (8, 8), 2)
    policy = NumpyGaussianMLPPolicy(dims, OP.init_params(dims, np.random.RandomState(seed + 1)))
    rec = {"collect": [], "snap": [], "tab": []}
    pool = stateful_pool.singleton_pool
    orig_collect, orig_save, orig_rec = pool.run_collect, rlogger.save_itr_params, rlogger.record_tabular

    def collect(*a, **k):
        out = orig_collect(*a, **k)
        rec["collect"].append(out)
        return out

    def save(itr, params):
        # the policy holds best_x here: cem.py sets it right before the snapshot (the workers of a one-process pool set
        # every member's row into the same policy object, so set_param_values itself is not a record of best_x)
        rec["snap"].append((np.array(params["cur_mean"]), np.array(params["cur_std"]),
                            params["policy"].get_param_values()))

    def record(key, val):
        if key == "Iteration":
            rec["tab"].append({})
        rec["tab"][-1][key] = val
        orig_rec(key, val)

    pool.run_collect, rlogger.save_itr_params, rlogger.record_tabular = collect, save, record
    try:
        algo = cem.CEM(env=env, policy=policy, n_itr=3, **kw)
        algo.train()
    finally:
        pool.run_collect, rlogger.save_itr_params, rlogger.record_tabular = orig_collect, orig_save, orig_rec
    out = {}
    p = name + "/"
    out[p + "n_itr"] = np.array(3)
    out[p + "n_best"] = np.array(max(1, int(algo.n_samples * algo.best_frac)))
    out[p + "n_evals"] = np.array(algo.n_evals)
    out[p + "discount"] = np.array(algo.discount)
    for k, v in sorted(kw.items()):
        out[p + "args_" + k] = np.array(v)
    for i in range(3):
        infos = rec["collect"][i]
        q = "%s%d/" % (p, i)
        out[q + "xs"] = np.asarray([info[0] for info in infos])
        out[q + "fs"] = np.array([info[1]["returns"][0] for info in infos])
        out[q + "ustat"] = np.array([info[1]["undiscounted_return"] for info in infos])
        rews = [pa["rewards"] for info in infos for pa in info[1]["full_paths"]]
        out[q + "rew_flat"] = np.concatenate(rews)
        out[q + "rew_len"] = np.array([len(r) for r in rews])
        out[q + "cur_mean"], out[q + "cur_std"], out[q + "best_x"] = rec["snap"][i]
        for key in KEYS:
            out[q + "tab_" + key] = np.array(rec["tab"][i][key])
    return out


def main():
    ref_shims.install()
    from rllab.sampler import stateful_pool
    stateful_pool.singleton_pool.initialize(1)
    out = {}
    for i, (name, kw) in enumerate(sorted(CASES.items())):
        out.update(run_case(name, kw, 10 + i))
        print(name, [out["%s/%d/tab_AverageReturn" % (name, j)] for j in range(3)])
    path = os.path.join(HERE, "reference_cem_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path)


if __name__ == "__main__":
    main()
