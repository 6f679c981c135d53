"""CPU: PPO and ERWR without a device.

- the float64 gradient of mean KL (tests/ppo_oracle.py) against torch.autograd and a central finite difference
- PPO / ERWR signatures and defaults against tests/golden/reference_api_ppo.json (tests/golden/make_api_ppo_golden.py)
- the optimizers the constructors build (NPO's default PenaltyLbfgsOptimizer, optimizer_args forwarded) and the options
  that stay rejected
- optimizer snapshots keep the carried penalty and drop the bound callables
"""
import importlib
import inspect
import json
import os
import pickle

import numpy as np
import pytest
import torch

import ppo_oracle as K
from oracle import policy as P

HERE = os.path.dirname(os.path.abspath(__file__))


def _problem(seed, O, H, A, B, min_std_clamp=False):
    rng = np.random.RandomState(seed)
    dims = P.Dims(O, H, A)
    theta = P.init_params(dims, rng) + 0.05 * rng.randn(dims.P)
    theta[-A:] = rng.uniform(-0.7, 0.3, size=A)
    obs = rng.randn(B, O)
    old_mean, old_log_std = P.forward(theta, obs, dims)
    actions = old_mean + np.exp(old_log_std) * rng.randn(B, A)
    batch = dict(obs=obs, actions=actions, adv=rng.randn(B), old_mean=old_mean, old_log_std=old_log_std)
    th = theta + 0.1 * rng.randn(dims.P)                       # off theta_old: KL > 0
    if min_std_clamp:
        th[-A] = np.log(1e-3) - 1.0
    return dims, th, batch


def _mean_kl_torch(th, batch, dims, min_std):
    t = torch.tensor(th, dtype=torch.float64, requires_grad=True)
    k, ts = 0, []
    for s in dims.shapes:
        n = int(np.prod(s))
        ts.append(t[k:k + n].reshape(s))
        k += n
    h = torch.tensor(batch["obs"])
    nl = len(dims.H)
    for i in range(nl):
        h = torch.tanh(h @ ts[2 * i] + ts[2 * i + 1])
    mu = h @ ts[2 * nl] + ts[2 * nl + 1]
    ls = torch.maximum(ts[-1], torch.tensor(np.log(min_std), dtype=torch.float64))
    om = torch.tensor(batch["old_mean"])
    ols = torch.tensor(np.asarray(batch["old_log_std"], dtype=np.float64))
    num = (om - mu) ** 2 + torch.exp(2 * ols) - torch.exp(2 * ls)
    kl = (num / (2 * torch.exp(2 * ls) + 1e-8) + ls - ols).sum(dim=-1)
    kl.mean().backward()
    return t.grad.numpy()


@pytest.mark.parametrize("O,H,A,clamp", [(4, (32, 32), 1, False), (13, (64, 64), 2, False), (6, (32, 32), 3, True)])
def test_grad_mean_kl_matches_autograd_and_finite_differences(O, H, A, clamp):
    min_std = 1e-3 if clamp else 1e-6
    dims, th, batch = _problem(3, O, H, A, 40, clamp)
    g = K.grad_mean_kl(th, batch, dims, min_std)
    assert P.kl_stats(th, batch, dims, min_std)[0] > 1e-3
    ref = _mean_kl_torch(th, batch, dims, min_std)
    np.testing.assert_allclose(g, ref, rtol=1e-9, atol=1e-9 * np.abs(ref).max())
    if clamp:
        assert g[dims.P - A] == 0.0
    rng = np.random.RandomState(5)
    idx = np.concatenate([rng.choice(dims.P - A, 12, replace=False), np.arange(dims.P - A, dims.P)])
    eps = 1e-6
    # float64 rounding of the two KL values over 2 eps: matters where a component clamped at min_std = 1e-3 makes the
    # mean KL large
    f0 = P.kl_stats(th, batch, dims, min_std)[0]
    for i in idx:
        e = np.zeros(dims.P)
        e[i] = eps
        fd = (P.kl_stats(th + e, batch, dims, min_std)[0] - P.kl_stats(th - e, batch, dims, min_std)[0]) / (2 * eps)
        assert abs(fd - g[i]) <= 1e-9 + 1e-6 * abs(g[i]) + 1e-15 * f0 / eps, (i, fd, g[i], f0)


def test_penalized_gradient_is_surrogate_plus_penalty_times_kl():
    dims, th, batch = _problem(4, 4, (32, 32), 1, 30)
    for kind in ("trpo", "vpg"):
        g0 = K.grad_penalized(th, batch, dims, kind, 0.0)
        np.testing.assert_array_equal(g0, P.grad_surr(th, batch, dims, kind))
        g = K.grad_penalized(th, batch, dims, kind, 7.0)
        np.testing.assert_allclose(g, g0 + 7.0 * K.grad_mean_kl(th, batch, dims), rtol=1e-14, atol=1e-14)
        f, loss, mkl = K.penalized_loss(th, batch, dims, kind, 7.0)
        assert f == loss + 7.0 * mkl


def test_api_matches_reference():
    api = json.load(open(os.path.join(HERE, "golden", "reference_api_ppo.json")))
    assert set(api) == {"PPO", "ERWR"}
    for name, d in api.items():
        mod, cls = d["mirror"].rsplit(".", 1)
        C = getattr(importlib.import_module(mod), cls)
        params = inspect.signature(C.__init__).parameters
        assert [p for p in params if p not in ("self", "kwargs")] == [a["name"] for a in d["init"]["args"]], name
        for a in d["init"]["args"]:
            assert params[a["name"]].default == a["default"]["literal"], (name, a["name"])
        assert any(p.kind == inspect.Parameter.VAR_KEYWORD for p in params.values()) == d["init"]["kwargs"]
        base = d["bases"][0]
        assert base in [b.__name__ for b in C.__mro__[1:]], (name, base)
        for m in d["methods"] + d["properties"]:
            assert hasattr(C, m), (name, m)


def _env_policy():
    from rllab_b200.envs.box2d.cartpole_env import CartpoleEnv
    from rllab_b200.envs.normalized_env import normalize
    from rllab_b200.policies.gaussian_mlp_policy import GaussianMLPPolicy
    from rllab_b200.baselines.zero_baseline import ZeroBaseline
    env = normalize(CartpoleEnv())
    return env, GaussianMLPPolicy(env.spec, hidden_sizes=(32, 32), seed=1), ZeroBaseline(env.spec)


def test_constructors_build_the_reference_optimizers():
    from rllab_b200.algos.erwr import ERWR
    from rllab_b200.algos.npo import NPO
    from rllab_b200.algos.ppo import PPO
    from rllab_b200.algos.vpg import VPG
    from rllab_b200.optimizers.first_order_optimizer import FirstOrderOptimizer
    from rllab_b200.optimizers.lbfgs_optimizer import LbfgsOptimizer
    from rllab_b200.optimizers.penalty_lbfgs_optimizer import PenaltyLbfgsOptimizer
    env, pol, base = _env_policy()
    a = NPO(env=env, policy=pol, baseline=base)
    assert isinstance(a.optimizer, PenaltyLbfgsOptimizer) and a.optimizer._max_opt_itr == 20 and a.step_size == 0.01
    a = NPO(env=env, policy=pol, baseline=base, optimizer_args=dict(max_opt_itr=7, initial_penalty=3.0), step_size=0.05)
    assert a.optimizer._max_opt_itr == 7 and a.optimizer._penalty == 3.0 and a.step_size == 0.05
    a = PPO(env=env, policy=pol, baseline=base, optimizer_args=dict(max_penalty_itr=4))
    assert isinstance(a.optimizer, PenaltyLbfgsOptimizer) and a.optimizer._max_penalty_itr == 4
    mine = PenaltyLbfgsOptimizer(max_opt_itr=3)
    assert PPO(env=env, policy=pol, baseline=base, optimizer=mine).optimizer is mine
    e = ERWR(env=env, policy=pol, baseline=base, optimizer_args=dict(max_opt_itr=9))
    assert isinstance(e.optimizer, LbfgsOptimizer) and e.optimizer._max_opt_itr == 9
    assert e.positive_adv is True and e.center_adv is True
    assert ERWR(env=env, policy=pol, baseline=base, positive_adv=False).positive_adv is False
    assert isinstance(VPG(env=env, policy=pol, baseline=base).optimizer, FirstOrderOptimizer)
    assert isinstance(VPG(env=env, policy=pol, baseline=base, optimizer=LbfgsOptimizer()).optimizer, LbfgsOptimizer)


def test_rejected_options():
    from rllab_b200.algos.npo import NPO
    from rllab_b200.algos.ppo import PPO
    env, pol, base = _env_policy()
    for C in (NPO, PPO):
        with pytest.raises(NotImplementedError):
            C(env=env, policy=pol, baseline=base, truncate_local_is_ratio=2.0)
    with pytest.raises(TypeError):
        PPO(env=env, policy=pol, baseline=base, optimizer_args=dict(no_such_option=1))


def test_optimizer_snapshot_keeps_penalty_and_drops_callables():
    from rllab_b200.optimizers.lbfgs_optimizer import LbfgsOptimizer
    from rllab_b200.optimizers.penalty_lbfgs_optimizer import PenaltyLbfgsOptimizer
    opt = PenaltyLbfgsOptimizer(max_opt_itr=5)
    f = lambda *a: 0.0                                    # noqa: E731  (a lambda does not pickle)
    opt.update_opt(loss=f, target=object(), leq_constraint=(f, 0.01), f_opt=f, f_penalized_loss=f)
    opt._penalty = 0.25
    o2 = pickle.loads(pickle.dumps(opt))
    assert o2._penalty == 0.25 and o2._max_opt_itr == 5 and o2._opt_fun is None and o2._target is None
    assert opt._opt_fun is not None                       # the live optimizer keeps its binding
    lb = LbfgsOptimizer(max_opt_itr=4)
    lb.update_opt(loss=f, target=object(), f_opt=f)
    l2 = pickle.loads(pickle.dumps(lb))
    assert l2._max_opt_itr == 4 and l2._opt_fun is None
