"""CPU: the DDPG oracle (tests/ddpg_oracle.py) against torch.autograd, its replay-pool and exploration draws, and the host
API of DDPG, DeterministicMLPPolicy, ContinuousMLPQFunction and the exploration strategies (constructor surfaces,
rejections, pickling) -- no GPU needed."""
import pickle

import numpy as np
import pytest
import torch

import ddpg_oracle as K
from rllab_b200 import _lib as L


def _nets(d, seed):
    rng = np.random.RandomState(seed)
    th = np.concatenate([K.init_params(d.pshapes, rng), K.init_params(d.qshapes, rng)])
    th = th + 0.1 * rng.randn(d.P)   # move the output layers off their tiny init so every gradient entry is non-trivial
    return np.stack([th, 1e-3 * rng.randn(d.P), 1e-6 * rng.rand(d.P), th + 0.05 * rng.randn(d.P)])


def _batch(d, seed):
    rng = np.random.RandomState(seed)
    return dict(s=rng.randn(32, d.O), a=rng.uniform(-1, 1, (32, d.A)), r=0.1 * rng.randn(32),
                term=(rng.rand(32) < 0.3).astype(np.float64), s2=rng.randn(32, d.O))


def _torch_grads(d, nets, batch, hp):
    """Critic and actor gradients of do_training by torch.autograd in float64."""
    def split(t, shapes):
        out, k = [], 0
        for s in shapes:
            n = int(np.prod(s))
            out.append(t[k:k + n].reshape(s))
            k += n
        return out

    def pi(tp, obs):
        W0, b0, W1, b1, W2, b2 = split(tp, d.pshapes)
        return torch.tanh(torch.relu(torch.relu(obs @ W0 + b0) @ W1 + b1) @ W2 + b2)

    def qf(tq, obs, act):
        W0, b0, W1, b1, W2, b2 = split(tq, d.qshapes)
        x = torch.cat([torch.relu(obs @ W0 + b0), act], 1)
        return (torch.relu(x @ W1 + b1) @ W2 + b2)[:, 0]

    T = {k: torch.tensor(v) for k, v in batch.items()}
    th, tg = torch.tensor(nets[0]), torch.tensor(nets[3])
    y = T["r"] + (1 - T["term"]) * hp["discount"] * qf(tg[d.PP:], T["s2"], pi(tg[:d.PP], T["s2"]))
    tq = th[d.PP:].clone().requires_grad_(True)
    wq = torch.tensor(d.weight_mask()[d.PP:])
    loss = torch.mean((y - qf(tq, T["s"], T["a"])) ** 2) + 0.5 * hp["qf_weight_decay"] * torch.sum(wq * tq ** 2)
    gq, = torch.autograd.grad(loss, tq)
    return y.numpy(), gq.numpy(), pi, qf, T


def test_oracle_backward_matches_autograd():
    d = K.Dims(4, 1)
    hp = dict(discount=0.99, qf_weight_decay=0.01, policy_weight_decay=0.02, qf_learning_rate=1e-3,
              policy_learning_rate=1e-4, soft_target_tau=0.001)
    nets = _nets(d, 1)
    batch = _batch(d, 2)
    new, info = K.do_training(d, nets, batch, hp, 5)
    y, gq, pi, qf, T = _torch_grads(d, nets, batch, hp)
    np.testing.assert_allclose(info["y"], y, rtol=0, atol=1e-12)
    np.testing.assert_allclose(info["grad"][d.PP:], gq, rtol=0, atol=1e-10)
    # actor: surrogate with the UPDATED critic
    tq_new = torch.tensor(new[0][d.PP:])
    tp = torch.tensor(nets[0][:d.PP]).requires_grad_(True)
    wp = torch.tensor(d.weight_mask()[:d.PP])
    surr = -torch.mean(qf(tq_new, T["s"], pi(tp, T["s"]))) + 0.5 * hp["policy_weight_decay"] * torch.sum(wp * tp ** 2)
    gp, = torch.autograd.grad(surr, tp)
    np.testing.assert_allclose(info["grad"][:d.PP], gp.numpy(), rtol=0, atol=1e-10)
    assert np.abs(gp.numpy()).max() > 1e-4 and np.abs(gq).max() > 1e-4
    # soft update over both nets after the two Adam steps
    np.testing.assert_allclose(new[3], nets[3] * (1 - 0.001) + new[0] * 0.001, rtol=0, atol=1e-15)


def test_random_batch_rejects_size_minus_one_including_the_full_pool():
    # not full: bottom 0, size 40 of 150 rows -> indices in [0, 40) minus 39
    idx = np.concatenate([K.draw_indices(3, itr, 0, 0, 0, 40, 150) for itr in range(200)])
    assert idx.min() >= 0 and idx.max() <= 38 and len(set(idx.tolist())) == 39
    # full: bottom 70, indices cover every row but size - 1 = 149, which is not the newest sample (row 69)
    idx = np.concatenate([K.draw_indices(3, itr, 0, 0, 70, 150, 150) for itr in range(400)])
    assert 149 not in set(idx.tolist()) and 69 in set(idx.tolist()) and len(set(idx.tolist())) == 149


def test_explore_normals_are_standard_normal():
    n = np.array([K.explore_normals(5, itr, 0, 2) for itr in range(20000)])
    assert abs(n.mean()) < 0.02 and abs(n.std() - 1.0) < 0.02


class _Spec(object):
    def __init__(self, O, A):
        from rllab_b200.spaces import Box
        self.observation_space = Box(-np.inf, np.inf, shape=(O,))
        self.action_space = Box(-1.0, 1.0, shape=(A,))


def _spec(O=4, A=1):
    return _Spec(O, A)


def _lib_or_skip():
    import os
    if not os.path.exists(L.LIB_PATH):
        pytest.skip("library not built")


def test_policy_and_qf_surface_and_pickling():
    _lib_or_skip()
    from rllab_b200.policies.deterministic_mlp_policy import DeterministicMLPPolicy
    from rllab_b200.q_functions.continuous_mlp_q_function import ContinuousMLPQFunction
    spec = _spec()
    pol = DeterministicMLPPolicy(spec, seed=1)
    qf = ContinuousMLPQFunction(spec, seed=2)
    assert pol.get_param_values().size == 1249 and qf.get_param_values().size == 1281
    assert [s for s in pol.get_param_shapes()] == [(4, 32), (32,), (32, 32), (32,), (32, 1), (1,)]
    assert [s for s in qf.get_param_shapes()] == [(4, 32), (32,), (33, 32), (32,), (32, 1), (1,)]
    assert pol.get_param_values(regularizable=True).size == 4 * 32 + 32 * 32 + 32
    W0 = pol.flat_to_params(pol.get_param_values())[0]
    assert np.abs(W0).max() <= np.sqrt(3.0 / 4) and np.all(pol.flat_to_params(pol.get_param_values())[1] == 0)
    assert np.abs(qf.flat_to_params(qf.get_param_values())[4]).max() <= 3e-3
    for obj in (pol, qf):
        back = pickle.loads(pickle.dumps(obj))
        np.testing.assert_array_equal(back.get_param_values(), obj.get_param_values())


@pytest.mark.parametrize("kw", [dict(bn=True), dict(hidden_sizes=(64, 64)), dict(hidden_nonlinearity="tanh")])
def test_nets_reject_what_is_not_built(kw):
    _lib_or_skip()
    from rllab_b200.policies.deterministic_mlp_policy import DeterministicMLPPolicy
    from rllab_b200.q_functions.continuous_mlp_q_function import ContinuousMLPQFunction
    for cls in (DeterministicMLPPolicy, ContinuousMLPQFunction):
        with pytest.raises(NotImplementedError):
            cls(_spec(), **kw)
    with pytest.raises(NotImplementedError):
        ContinuousMLPQFunction(_spec(), action_merge_layer=0)


def test_exploration_strategies_host_semantics():
    from rllab_b200.exploration_strategies.gaussian_strategy import GaussianStrategy
    from rllab_b200.exploration_strategies.ou_strategy import OUStrategy

    class Pol(object):
        def get_action(self, obs):
            return np.array([0.9]), {}

    np.random.seed(0)
    ou = OUStrategy(_spec(), mu=0.1, theta=0.15, sigma=0.3)
    np.testing.assert_array_equal(ou.state, [0.1])
    n = np.random.RandomState(0).randn(1)
    a = ou.get_action(0, None, Pol())
    np.testing.assert_allclose(ou.state, 0.1 + 0.3 * n)
    np.testing.assert_allclose(a, np.clip(0.9 + ou.state, -1, 1))
    ou.reset()
    np.testing.assert_array_equal(ou.state, [0.1])
    back = pickle.loads(pickle.dumps(ou))
    assert back.mu == 0.1 and back.sigma == 0.3
    gs = GaussianStrategy(_spec(), max_sigma=1.0, min_sigma=0.1, decay_period=100)
    assert gs.sigma(0) == 1.0 and abs(gs.sigma(50) - 0.55) < 1e-15 and abs(gs.sigma(500) - 0.1) < 1e-15
    assert pickle.loads(pickle.dumps(gs)).sigma(50) == gs.sigma(50)


def test_ddpg_rejections():
    _lib_or_skip()
    from rllab_b200.algos.ddpg import DDPG
    from rllab_b200.envs.box2d.cartpole_env import CartpoleEnv
    from rllab_b200.envs.normalized_env import normalize
    from rllab_b200.exploration_strategies.ou_strategy import OUStrategy
    from rllab_b200.policies.deterministic_mlp_policy import DeterministicMLPPolicy
    from rllab_b200.q_functions.continuous_mlp_q_function import ContinuousMLPQFunction
    env = normalize(CartpoleEnv())
    args = dict(env=env, policy=DeterministicMLPPolicy(env.spec), qf=ContinuousMLPQFunction(env.spec),
                es=OUStrategy(env.spec))
    DDPG(**args)
    for kw in (dict(plot=True), dict(qf_update_method='sgd'), dict(policy_update_method='sgd'), dict(batch_size=64)):
        with pytest.raises(NotImplementedError):
            DDPG(**dict(args, **kw))
    with pytest.raises(ValueError):
        DDPG(min_pool_size=32, **args)

    with pytest.raises(TypeError):                     # the kernel applies NormalizedEnv's action map
        DDPG(**dict(args, env=CartpoleEnv()))
    from rllab_b200.envs.gym_env import GymEnv
    from rllab_b200.envs.mujoco.swimmer_env import SwimmerEnv
    for other in (normalize(SwimmerEnv()), normalize(GymEnv("CartPole-v0"))):   # planar, Discrete
        with pytest.raises(NotImplementedError):
            DDPG(**dict(args, env=other))

    class Active(object):
        active = True
    with pytest.raises(NotImplementedError):
        DDPG(comm=Active(), **args)
