"""CPU: GaussianMLPBaseline's oracle (tests/vf_oracle.py) and host optimizers.

- the oracle's hand-written gradient against torch.autograd (float64) and central finite differences
- the host PenaltyLbfgsOptimizer / LbfgsOptimizer, driven by the oracle's callables, against the reference's own
  optimizers run on the same callables (tests/golden/reference_vf_golden.npz, tests/golden/make_vf_golden.py)
- the API surface and tabular keys against tests/golden/reference_api_vf.json; rejected options; construction
  without a GPU
"""
import importlib
import inspect
import json
import os

import numpy as np
import pytest

import vf_oracle as V

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def _problem(O=3, n=50, seed=0):
    rng = np.random.RandomState(seed)
    th = V.init_params(O, rng)
    th[O * 32:O * 32 + 32] = 0.1 * rng.randn(32)
    th[-1] = 0.25
    nx = rng.randn(n, O)
    ny = rng.randn(n)
    mu_old = V.forward(th + 0.05 * rng.randn(th.size), nx, O)[0]
    return th, nx, ny, mu_old, -0.1


def _objective_torch(th, nx, ny, O, penalty, mu_old, ls_old, w):
    import torch
    t = torch.tensor(th, dtype=torch.float64, requires_grad=True)
    X = torch.tensor(nx)
    i = 0
    parts = []
    for s in [(O, 32), (32,), (32, 32), (32,), (32, 1), (1,), (1,)]:
        k = int(np.prod(s))
        parts.append(t[i:i + k].reshape(s))
        i += k
    W0, b0, W1, b1, Wo, bo, ls = parts
    h1 = torch.relu(X @ W0 + b0)
    h2 = torch.relu(h1 @ W1 + b1)
    mu = (h2 @ Wo + bo).reshape(-1)
    y = torch.tensor(ny)
    var = torch.exp(2 * ls)
    nll = ls + 0.5 * (y - mu) ** 2 / var + V.HALF_LOG_2PI
    ww = torch.tensor(w)
    f = (nll * ww).sum() / ww.sum()
    if mu_old is not None:
        mo = torch.tensor(mu_old)
        kl = ((mo - mu) ** 2 + np.exp(2 * ls_old) - var) / (2 * var + 1e-8) + ls - ls_old
        f = f + penalty * (kl * ww).sum() / ww.sum()
    f.backward()
    return t.grad.numpy()


@pytest.mark.parametrize("trust", [True, False])
@pytest.mark.parametrize("learn_std", [True, False])
def test_oracle_gradient_matches_autograd_and_finite_differences(trust, learn_std):
    pytest.importorskip("torch")
    O = 3
    th, nx, ny, mu_old, ls_old = _problem(O)
    w = np.ones(len(ny))
    w[::7] = 0.0                                      # masked samples
    pen = 3.0 if trust else 0.0
    mo, lo = (mu_old, ls_old) if trust else (None, None)
    _, _, _, g = V.loss_grad(th, nx, ny, O, pen, mo, lo, learn_std, w)
    ref = _objective_torch(th, nx, ny, O, pen, mo, lo, w)
    if not learn_std:
        ref[-1] = 0.0
    np.testing.assert_allclose(g, ref, rtol=1e-9, atol=1e-12)

    def f(t):
        nll, kl, _, _ = V.loss_grad(t, nx, ny, O, pen, mo, lo, learn_std, w)
        return nll + pen * kl
    eps = 1e-6
    idx = list(range(0, th.size, 37)) + [th.size - 2, th.size - 1]
    for i in idx:
        if i == th.size - 1 and not learn_std:
            continue
        e = np.zeros_like(th)
        e[i] = eps
        fd = (f(th + e) - f(th - e)) / (2 * eps)
        assert abs(fd - g[i]) <= 1e-9 + 1e-7 * abs(g[i]), (i, fd, g[i])


def _golden():
    return np.load(os.path.join(HERE, "golden", "reference_vf_golden.npz"))


GOLDEN_CASES = ["lbfgs20", "lbfgs3", "pen_decrease", "pen_fixedstd", "pen_increase", "pen_maxitr", "pen_noadapt"]


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_host_optimizers_reproduce_reference_golden(name):
    """The restated optimizers on the oracle callables follow the reference's own optimizers step for step."""
    from rllab_b200.misc import logger
    from rllab_b200.optimizers.lbfgs_optimizer import LbfgsOptimizer
    from rllab_b200.optimizers.penalty_lbfgs_optimizer import PenaltyLbfgsOptimizer
    logger.set_quiet(True)
    import sys
    sys.path.insert(0, os.path.join(HERE, "golden"))
    import make_vf_golden as C
    O, n, kind, kw, learn_std, ls0, y_scale, pen0 = C.CASES[name]
    G = _golden()
    xs, ys, theta0 = G[name + "_xs"], G[name + "_ys"], G[name + "_theta0"]
    if kind == "penalty":
        opt = PenaltyLbfgsOptimizer(initial_penalty=pen0, **kw)
    else:
        opt = LbfgsOptimizer(**kw)
    th, _, info = V.fit(theta0, xs, ys, O, opt, use_trust_region=(kind == "penalty"), learn_std=learn_std)
    np.testing.assert_allclose(th, G[name + "_theta"], rtol=1e-12, atol=1e-12 * np.abs(G[name + "_theta"]).max())
    np.testing.assert_allclose([info["LossBefore"], info["LossAfter"]], G[name + "_loss"], rtol=1e-12)
    if kind == "penalty":
        assert opt.tried_penalties == list(G[name + "_penalties"])
        assert float(opt._penalty) == float(G[name + "_penalty"])
        np.testing.assert_allclose(info["MeanKL"], G[name + "_kl"], rtol=1e-12, atol=1e-15)
        assert len(opt.terminations) == len(opt.tried_penalties)
    else:
        assert opt.termination is not None


def test_golden_covers_the_penalty_paths():
    G = _golden()
    dec, inc, mx = G["pen_decrease_penalties"], G["pen_increase_penalties"], G["pen_maxitr_penalties"]
    assert len(dec) >= 2 and (np.diff(dec) < 0).all()           # decreasing until the constraint is violated
    assert len(inc) >= 2 and (np.diff(inc) > 0).all()           # increasing from a violated start
    assert len(mx) == 3                                          # ran out of max_penalty_itr
    assert len(G["pen_noadapt_penalties"]) == 1


def test_api_surface_and_tabular_keys_match_reference():
    api = json.load(open(os.path.join(HERE, "golden", "reference_api_vf.json")))
    tab = api.pop("__tabular__")
    for rel, d in tab.items():
        src = "".join(open(os.path.join(ROOT, m)).read() for m in d["mirrors"])
        assert d["prefixed_keys"] == ["LossBefore", "LossAfter", "dLoss", "MeanKL"]
        for key in d["prefixed_keys"] + d["keys"]:
            assert "'%s'" % key in src or '"%s"' % key in src, key
    exempt = {"GaussianMLPRegressor": {"log_likelihood_sym"}}
    assert set(api) == {"GaussianMLPBaseline", "GaussianMLPRegressor", "PenaltyLbfgsOptimizer", "LbfgsOptimizer"}
    for name, d in api.items():
        mod, cls = d["mirror"].rsplit(".", 1)
        C = getattr(importlib.import_module(mod), cls)
        params = inspect.signature(C.__init__).parameters
        for a in d["init"]["args"]:
            assert a["name"] in params, (name, a["name"])
            if a["default"] and "literal" in a["default"]:
                mine = params[a["name"]].default
                mine = list(mine) if isinstance(mine, tuple) else mine
                assert mine == a["default"]["literal"], (name, a["name"])
        for m in d["methods"] + d["properties"]:
            if m in exempt.get(name, ()):
                assert not hasattr(C, m)
                continue
            assert hasattr(C, m), (name, m)
    from rllab_b200.baselines.gaussian_mlp_baseline import GaussianMLPBaseline
    assert hasattr(GaussianMLPBaseline, "log_diagnostics")


def _spec():
    import bench
    return bench.make_env("cartpole").spec


@pytest.mark.parametrize("kw", [dict(adaptive_std=True), dict(std_share_network=True), dict(mean_network=object()),
                                dict(hidden_sizes=(64, 64)), dict(hidden_sizes=(32,)), dict(hidden_nonlinearity="tanh"),
                                dict(batchsize=100), dict(subsample_factor=0.5), dict(optimizer=object())])
def test_rejected_options(kw):
    from rllab_b200.baselines.gaussian_mlp_baseline import GaussianMLPBaseline
    with pytest.raises(NotImplementedError):
        GaussianMLPBaseline(_spec(), regressor_args=kw)


def test_unknown_keywords_and_seq_inputs():
    from rllab_b200.baselines.gaussian_mlp_baseline import GaussianMLPBaseline
    from rllab_b200.optimizers.penalty_lbfgs_optimizer import PenaltyLbfgsOptimizer
    from rllab_b200.regressors.gaussian_mlp_regressor import GaussianMLPRegressor
    with pytest.raises(TypeError):
        GaussianMLPBaseline(_spec(), regressor_args=dict(no_such_option=1))
    with pytest.raises(TypeError):
        GaussianMLPRegressor((4,), 1, no_such_option=1)
    with pytest.raises(TypeError):
        PenaltyLbfgsOptimizer(no_such_option=1)
    with pytest.raises(NotImplementedError):
        GaussianMLPBaseline(_spec(), num_seq_inputs=2)


def test_construction_without_gpu():
    import pickle
    from rllab_b200.baselines.gaussian_mlp_baseline import GaussianMLPBaseline
    from rllab_b200.optimizers.lbfgs_optimizer import LbfgsOptimizer
    np.random.seed(4)
    b = GaussianMLPBaseline(_spec(), subsample_factor=1.0)
    P = V.num_params(4)
    th = b.get_param_values()
    assert th.shape == (P,) and th[-1] == 0.0 and (th[4 * 32:4 * 32 + 32] == 0).all()
    assert np.abs(th[:4 * 32]).max() <= np.sqrt(6.0 / 36)
    reg = b.regressor
    np.testing.assert_array_equal(reg.get_stats(), np.concatenate([np.zeros(4), np.ones(4), [0.0, 1.0]]))
    b2 = pickle.loads(pickle.dumps(b))
    np.testing.assert_array_equal(b2.get_param_values(), th)
    r = GaussianMLPBaseline(_spec(), regressor_args=dict(use_trust_region=False, learn_std=False, init_std=2.0))
    assert isinstance(r.regressor._optimizer, LbfgsOptimizer)
    assert r.regressor.get_param_values(trainable=True).shape == (P - 1,)
    assert r.get_param_values()[-1] == np.log(2.0)
