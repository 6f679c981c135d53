"""CPU: the REPS oracle (tests/reps_oracle.py) against the reference's own REPS.optimize_policy
(tests/golden/reference_reps_golden.npz, made by tests/golden/make_reps_golden.py), the REPS surface against
tests/golden/reference_api_reps.json, the lane form of feat_diff against the path form, and the dual gradient against
finite differences."""
import ast
import importlib
import inspect
import json
import os
import pickle

import numpy as np
import pytest
import scipy.optimize

import reps_oracle as K
from oracle import policy as P

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(os.path.join(HERE, "golden", "reference_reps_golden.npz")))


def _cases(g):
    return sorted({k.split("/")[0] for k in g})


def _paths(g, c):
    lens = g[c + "/path_len"]
    cuts = np.concatenate([[0], np.cumsum(lens)])
    obs = g[c + "/obs_flat"]
    return [dict(observations=obs[cuts[i]:cuts[i + 1]]) for i in range(len(lens))]


def _batch(g, c):
    return dict(obs=g[c + "/obs_flat"], actions=g[c + "/act_flat"], old_mean=g[c + "/mean_flat"],
                old_log_std=g[c + "/log_std"])


def _dims(g, c):
    return P.Dims(g[c + "/obs_flat"].shape[1], tuple(int(h) for h in g[c + "/hidden"]), g[c + "/act_flat"].shape[1])


def _args(g, c):
    return {k.split("args_")[1]: g[k][()] for k in g if k.startswith(c + "/args_")}


def lanes_from_paths(paths, N, T):
    """Lay whole paths out on N lanes of T steps, in order; every lane's tail is filled by a path cut at T - 1.
    Returns obs [O][T][N], flags, tstep [T][N] and the (t, n) cell of every path sample in path order."""
    O = paths[0]["observations"].shape[1]
    obs = np.zeros((O, T, N))
    flags = np.zeros((T, N), np.uint8)
    tstep = np.zeros((T, N), np.uint16)
    cells, n, t = [], 0, 0
    rng = np.random.RandomState(5)
    for p in paths:
        L = len(p["observations"])
        if t + L > T:
            n, t = n + 1, 0
        for i in range(L):
            obs[:, t + i, n] = p["observations"][i]
            tstep[t + i, n] = i
            cells.append((t + i, n))
        flags[t + L - 1, n] = K.FLAG_END
        t += L
    for m in range(N):                                       # tails: filler paths cut by the end of the buffer
        used = max([c[0] + 1 for c in cells if c[1] == m] + [0])
        if used < T:
            obs[:, used:, m] = rng.randn(O, T - used) * 20.0
            tstep[used:, m] = np.arange(T - used)
            flags[T - 1, m] = K.FLAG_END | 4
    return obs, flags, tstep, cells


def test_golden_covers_the_cases(golden):
    cases = _cases(golden)
    assert cases == ["defaults", "regularized"]
    a = _args(golden, "regularized")
    assert a["L2_reg_dual"] > 0 and a["L2_reg_loss"] > 0
    assert 1 in golden["defaults/path_len"]
    assert np.abs(golden["defaults/obs_flat"]).max() > 10          # the clip is exercised
    assert float(golden["defaults/1/eta_after"]) < 1.0             # eta moves far from its start of 15


def test_feat_diff_path_form_matches_reference(golden):
    for c in _cases(golden):
        fd = K.feat_diff_paths(_paths(golden, c))
        for it in range(2):
            assert np.array_equal(fd, golden["%s/%d/feat_diff" % (c, it)])


def test_feat_diff_lane_form_equals_path_form(golden):
    paths = _paths(golden, "defaults")
    ref = K.feat_diff_paths(paths)
    for N, T in ((3, 64), (6, 50), (2, 100)):
        obs, flags, tstep, cells = lanes_from_paths(paths, N, T)
        fd = K.feat_diff_lanes(obs, flags, tstep)
        got = np.array([fd[t, n] for t, n in cells])
        assert np.array_equal(got, ref), (N, T)
        # a cut filler path ends with phi(next) = 0 like a whole one
        assert np.array_equal(fd[T - 1, N - 1], -K.features(obs[:, T - 1, N - 1][None], [tstep[T - 1, N - 1]])[0])


def test_dual_gradient_matches_finite_differences(golden):
    c = "defaults"
    rew = golden[c + "/rew_flat"]
    fd = K.feat_diff_paths(_paths(golden, c))
    rng = np.random.RandomState(3)
    for eta, l2 in ((0.3, 0.0), (1.0, 0.0), (15.0, 0.0), (2.0, 1e-3), (50.0, 0.1)):
        v = rng.randn(fd.shape[1])
        x = np.concatenate([[eta], v])
        g = K.dual_grad(eta, v, rew, fd, 0.5, l2)
        num = np.zeros_like(x)
        for i in range(len(x)):
            h = 1e-6 * max(1.0, abs(x[i]))
            xp, xm = x.copy(), x.copy()
            xp[i] += h
            xm[i] -= h
            num[i] = (K.dual(xp[0], xp[1:], rew, fd, 0.5, l2) - K.dual(xm[0], xm[1:], rew, fd, 0.5, l2)) / (2 * h)
        err = np.max(np.abs(num - g)) / np.max(np.abs(g))
        assert err < 1e-6, (eta, l2, err)


def test_optimize_policy_restatement_matches_reference(golden):
    for c in _cases(golden):
        a = _args(golden, c)
        rew = golden[c + "/rew_flat"]
        fd = K.feat_diff_paths(_paths(golden, c))
        batch, dims = _batch(golden, c), _dims(golden, c)
        theta = golden[c + "/theta0"]
        for it in range(2):
            q = "%s/%d/" % (c, it)
            r = K.optimize_policy(float(golden[q + "eta_before"]), golden[q + "v_before"], theta, batch, rew, fd, dims,
                                  epsilon=float(a["epsilon"]), l2_reg_dual=float(a["L2_reg_dual"]),
                                  l2_reg_loss=float(a["L2_reg_loss"]), max_opt_itr=int(a["max_opt_itr"]))
            assert abs(r["eta"] - golden[q + "eta_after"]) <= 1e-10 * abs(golden[q + "eta_after"]), (c, it)
            v_ref, th_ref = golden[q + "v_after"], golden[q + "theta_after"]
            assert np.max(np.abs(r["v"] - v_ref)) <= 1e-10 * np.max(np.abs(v_ref)), (c, it)
            assert np.max(np.abs(r["theta"] - th_ref)) <= 1e-10 * np.max(np.abs(th_ref)), (c, it)
            for key in ("LossBefore", "LossAfter", "DualBefore", "DualAfter", "MeanKL"):
                assert r[key] == pytest.approx(float(golden[q + "tab_" + key]), rel=1e-10, abs=1e-12), (c, it, key)
            theta = th_ref


def _api():
    return json.load(open(os.path.join(HERE, "golden", "reference_api_reps.json")))["REPS"]


def test_reps_signature_matches_reference():
    d = _api()
    mod, cls = d["mirror"].rsplit(".", 1)
    C = getattr(importlib.import_module(mod), cls)
    params = inspect.signature(C.__init__).parameters
    assert [p for p in params if p not in ("self", "kwargs")] == [a["name"] for a in d["init"]["args"]]
    for a in d["init"]["args"]:
        want = a["default"]["literal"] if "literal" in a["default"] else eval(a["default"]["source"], {"scipy": scipy})
        assert params[a["name"]].default == want, a["name"]
    assert any(p.kind == inspect.Parameter.VAR_KEYWORD for p in params.values()) == d["init"]["kwargs"]
    for base in d["bases"]:
        assert base in [b.__name__ for b in C.__mro__[1:]], base
    for m in d["methods"] + d["properties"]:
        assert hasattr(C, m), m


def test_reps_records_the_reference_tabular_keys():
    tree = ast.parse(open(os.path.join(ROOT, "rllab_b200", "algos", "reps.py")).read())
    keys = [n.args[0].value for n in ast.walk(tree)
            if isinstance(n, ast.Call) and isinstance(n.func, ast.Attribute) and n.func.attr == "record_tabular"
            and n.args and isinstance(n.args[0], ast.Constant)]
    assert sorted(keys) == sorted(_api()["tabular"])


def test_dual_from_sums_equals_oracle(golden):
    """The host half of the device dual (rllab_b200.algos.reps.dual_from_sums) on sums formed in NumPy."""
    from rllab_b200.algos.reps import dual_from_sums
    rew = golden["defaults/rew_flat"]
    fd = K.feat_diff_paths(_paths(golden, "defaults"))
    rng = np.random.RandomState(4)
    for eta, l2 in ((1e-2, 0.0), (1.0, 0.0), (15.0, 1e-3), (1e3, 0.0)):
        v = rng.rand(fd.shape[1])
        d = K.delta(rew, fd, v)
        M = d.max()
        e = np.exp((d - M) / eta)
        sums = np.concatenate([[e.sum(), (e * (d - M)).sum()], e @ fd])
        g, grad = dual_from_sums(eta, M, sums, len(d), 0.5, l2)
        assert g == pytest.approx(K.dual(eta, v, rew, fd, 0.5, l2), rel=1e-12)
        np.testing.assert_allclose(grad, K.dual_grad(eta, v, rew, fd, 0.5, l2), rtol=1e-12, atol=1e-12)


def test_reps_rejects_plot_and_pickles_dual_variables():
    from rllab_b200.algos.reps import REPS
    with pytest.raises(NotImplementedError):
        REPS(env=None, policy=None, baseline=None, plot=True)
    algo = REPS(env=None, policy=None, baseline=None, epsilon=0.2, max_opt_itr=7)
    algo.param_eta, algo.param_v = 3.5, np.arange(12.0)
    back = pickle.loads(pickle.dumps(algo))
    assert (back.epsilon, back.max_opt_itr, back.param_eta) == (0.2, 7, 3.5)
    assert np.array_equal(back.param_v, algo.param_v)
    assert back.optimizer is scipy.optimize.fmin_l_bfgs_b
