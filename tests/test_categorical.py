"""CPU: the float64 categorical oracle against torch.autograd, gym CartPole-v0 steps against hand-computed values, and the
host API of the discrete-action path (Discrete, Categorical, CategoricalMLPPolicy, GymEnv("CartPole-v0"))."""
import os
import pickle

import numpy as np
import pytest

import categorical_oracle as C

torch = pytest.importorskip("torch")

DIMS = C.CatDims(4, (32, 32), 2)


def _batch(rng, B=57, theta_old=None):
    obs = rng.randn(B, 4)
    theta_old = C.init_params(DIMS, rng) if theta_old is None else theta_old
    old_p = C.prob(theta_old, obs, DIMS)
    acts = C.weighted_sample_n(old_p, rng.rand(B))
    return dict(obs=obs, actions=np.eye(2)[acts], adv=rng.randn(B), old_prob=old_p), theta_old


def _torch_prob(theta, obs):
    ts, k = [], 0
    for s in DIMS.shapes:
        n = int(np.prod(s))
        ts.append(theta[k:k + n].reshape(s))
        k += n
    h = torch.tanh(torch.tanh(obs @ ts[0] + ts[1]) @ ts[2] + ts[3])
    return torch.softmax(h @ ts[4] + ts[5], dim=-1)


def _torch_terms(theta, batch, kind):
    obs = torch.tensor(batch["obs"])
    x = torch.tensor(batch["actions"])
    q = torch.tensor(batch["old_prob"])
    adv = torch.tensor(batch["adv"])
    p = _torch_prob(theta, obs)
    if kind == "trpo":       # categorical.py: likelihood_ratio_sym
        w = ((p * x).sum(-1) + C.TINY) / ((q * x).sum(-1) + C.TINY)
    else:                    # log_likelihood_sym
        w = torch.log((p * x).sum(-1) + C.TINY)
    kl = (q * (torch.log(q + C.TINY) - torch.log(p + C.TINY))).sum(-1)     # kl_sym
    return -(w * adv).mean(), kl.mean()


@pytest.mark.parametrize("kind", ["trpo", "vpg"])
@pytest.mark.parametrize("penalty", [0.0, 3.0])
def test_oracle_gradient_matches_autograd(kind, penalty):
    rng = np.random.RandomState(3)
    batch, th_old = _batch(rng)
    theta = th_old + 0.05 * rng.randn(DIMS.P)              # off theta_old: ratio != 1, KL > 0
    t = torch.tensor(theta, requires_grad=True)
    loss, kl = _torch_terms(t, batch, kind)
    (g,) = torch.autograd.grad(loss + penalty * kl, t)
    ours = C.grad_surr(theta, batch, DIMS, kind, penalty)
    np.testing.assert_allclose(ours, g.numpy(), rtol=1e-10, atol=1e-13 * np.abs(ours).max())
    assert abs(C.surr_loss(theta, batch, DIMS, kind) - loss.item()) < 1e-13
    assert abs(C.kl_stats(theta, batch, DIMS)[0] - kl.item()) < 1e-13


def test_oracle_fvp_matches_double_backward():
    """The oracle's product is torch's double backward through the reference's KL expression (float64), the O(TINY)
    curvature term of the logits included."""
    rng = np.random.RandomState(5)
    batch, theta = _batch(rng, B=91)
    x = rng.randn(DIMS.P)
    t = torch.tensor(theta, requires_grad=True)
    _, kl = _torch_terms(t, batch, "trpo")
    (g,) = torch.autograd.grad(kl, t, create_graph=True)
    (hx,) = torch.autograd.grad(g @ torch.tensor(x), t)
    ours = C.fvp(theta, batch, x, DIMS, reg_coeff=0.0)
    err = np.abs(ours - hx.numpy()).max() / np.abs(hx.numpy()).max()
    assert err < 1e-12, err
    # the closed-form logit Hessian itself is exact: against autograd's Hessian of kl(q || softmax(z)) in z
    z = rng.randn(6, 2)
    q = C.softmax(z)
    for i in range(6):
        zt = torch.tensor(z[i], requires_grad=True)
        qt = torch.tensor(q[i])
        f = lambda zz: (qt * (torch.log(qt + C.TINY) - torch.log(torch.softmax(zz, -1) + C.TINY))).sum()
        H = torch.autograd.functional.hessian(f, zt).numpy()
        np.testing.assert_allclose(C.logit_hessian(q[i:i + 1])[0], H, rtol=1e-12, atol=1e-16)


def test_oracle_ratio_one_and_kl_zero_at_theta_old():
    rng = np.random.RandomState(7)
    batch, theta = _batch(rng)
    p = C.prob(theta, batch["obs"], DIMS)
    assert np.all(C.likelihood_ratio(batch["actions"], batch["old_prob"], p) == 1.0)
    assert C.kl_stats(theta, batch, DIMS) == (0.0, 0.0)


GAPS = (4, 8, 12, 16, 20, 30, 60)          # logit gaps |z0 - z1| of the saturated buckets


def _mp_reference(theta, batch, x, kind, penalty):
    """(surrogate + penalty KL gradient, KL gradient, Fisher-vector product at theta_old = theta with q = p) in 50-digit
    arithmetic, by the textbook formulas (dz = -c p (x - pa), M = diag(R p - s) + s p^T + p s^T - (R + S) p p^T): at
    this precision their cancellation costs nothing."""
    mp = pytest.importorskip("mpmath")
    with mp.workdps(50):
        f = np.vectorize(lambda v: mp.mpf(float(v)), otypes=[object])
        tanh = np.vectorize(mp.tanh, otypes=[object])
        exp = np.vectorize(mp.exp, otypes=[object])
        E = mp.mpf(C.TINY)
        W0, b0, W1, b1, Wo, bo = (f(t) for t in C.unpack(theta, DIMS))
        V0, c0, V1, c1, Vo, co = (f(t) for t in C.unpack(x, DIMS))
        X, xa, q, adv = (f(batch[k]) for k in ("obs", "actions", "old_prob", "adv"))
        B = X.shape[0]
        h1 = tanh(X @ W0 + b0)
        h2 = tanh(h1 @ W1 + b1)
        z = h2 @ Wo + bo
        e = exp(z - np.max(z, axis=1, keepdims=True))
        p = e / np.sum(e, axis=1, keepdims=True)

        def backward(dz):
            d2 = (dz @ Wo.T) * (1 - h2 * h2)
            d1 = (d2 @ W1.T) * (1 - h1 * h1)
            return np.concatenate([(X.T @ d1).reshape(-1), d1.sum(0), (h1.T @ d2).reshape(-1), d2.sum(0),
                                   (h2.T @ dz).reshape(-1), dz.sum(0)]) / B

        pa = np.sum(p * xa, axis=1)
        c = adv / (np.sum(q * xa, axis=1) + E) if kind == "trpo" else adv / (pa + E)
        r = q * p / (p + E)
        gkl = -r + p * np.sum(r, axis=1, keepdims=True)
        g = backward(-c[:, None] * p * (xa - pa[:, None]) + penalty * gkl)
        g_kl = backward(gkl)
        # Fisher-vector product at q = p: J^T M J x + sum_j g_j (d^2 z_j)[x], as tests/categorical_oracle.py:fvp
        d1h, d2h = 1 - h1 * h1, 1 - h2 * h2
        t1 = d1h * (X @ V0 + c0)
        t2 = d2h * (t1 @ W1 + h1 @ V1 + c1)
        tz = t2 @ Wo + h2 @ Vo + co
        pe = p + E
        R = np.sum(p * p / pe, axis=1)[:, None]
        s = E * p * p / (pe * pe)
        S = np.sum(s, axis=1)[:, None]
        ptz = np.sum(p * tz, axis=1)[:, None]
        stz = np.sum(s * tz, axis=1)[:, None]
        mz = (R * p - s) * tz + s * ptz + p * stz - (R + S) * p * ptz
        rr = p * p / pe
        gg = -rr + p * np.sum(rr, axis=1, keepdims=True)
        d2g = (gg @ Wo.T) * d2h
        D2 = (mz @ Wo.T) * d2h + (gg @ Vo.T) * d2h - 2 * (gg @ Wo.T) * h2 * t2
        D1 = (D2 @ W1.T + d2g @ V1.T) * d1h - 2 * (d2g @ W1.T) * h1 * t1
        hx = np.concatenate([(X.T @ D1).reshape(-1), D1.sum(0), (h1.T @ D2 + t1.T @ d2g).reshape(-1), D2.sum(0),
                             (h2.T @ mz + t2.T @ gg).reshape(-1), mz.sum(0)]) / B
        return tuple(np.array([float(v) for v in a]) for a in (g, g_kl, hx))


def _blocks():
    out, k = [], 0
    for s in DIMS.shapes:
        n = int(np.prod(s))
        out.append(slice(k, k + n))
        k += n
    return out


def saturated_batch(rng, gap, sign, B=8, n_unlikely=2):
    """A batch at theta_old = C.saturated_params(gap): actions drawn from the policy, the last n_unlikely forced to the
    unlikely action (q down to its probability, 1e-26 at gap 60)."""
    theta = C.saturated_params(DIMS, gap, rng, sign)
    obs = rng.randn(B, 4)
    p = C.prob(theta, obs, DIMS)
    acts = C.weighted_sample_n(p, rng.rand(B))
    acts[B - n_unlikely:] = np.argmin(p[B - n_unlikely:], axis=1)
    return dict(obs=obs, actions=np.eye(2)[acts], adv=rng.randn(B), old_prob=p), theta


@pytest.mark.parametrize("gap", GAPS)
def test_oracle_exact_at_saturated_softmax(gap):
    """The oracle's gradients (TRPO and VPG surrogates, with and without a KL penalty, off theta_old), KL gradient and
    Fisher-vector product (at theta_old, TINY terms included) within 1e-13 of 50-digit arithmetic, per parameter block,
    on a batch whose every logit gap is `gap`: no term of it may cancel when a probability nears 1."""
    rng = np.random.RandomState(gap)
    batch, theta_old = saturated_batch(rng, gap, 1.0 if gap % 8 else -1.0)
    p = C.prob(theta_old, batch["obs"], DIMS)
    assert np.all(np.abs(np.log(p[:, 0]) - np.log(p[:, 1])) > gap - 0.3)
    theta = theta_old + 0.01 * rng.randn(DIMS.P)
    x = rng.randn(DIMS.P)
    checks = []
    for kind, pen in (("trpo", 0.0), ("trpo", 2.5), ("vpg", 0.0), ("vpg", 2.5)):
        g_ref, gkl_ref, _ = _mp_reference(theta, batch, x, kind, pen)
        checks.append(("grad %s pen %g" % (kind, pen), C.grad_surr(theta, batch, DIMS, kind, pen), g_ref))
    checks.append(("kl grad", C.grad_kl(theta, batch, DIMS), gkl_ref))
    batch_old = dict(batch, old_prob=p)
    _, _, hx_ref = _mp_reference(theta_old, batch_old, x, "trpo", 0.0)
    checks.append(("fvp", C.fvp(theta_old, batch_old, x, DIMS, reg_coeff=0.0), hx_ref))
    for what, got, ref in checks:
        for i, sl in enumerate(_blocks()):
            err = np.abs(got[sl] - ref[sl]).max() / np.abs(ref[sl]).max()
            assert err <= 1e-13, "gap %g, %s, block %d: %.3g" % (gap, what, i, err)


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_categorical_golden.npz")


def test_distribution_functions_match_reference_golden():
    """Against the reference's own Categorical / special.weighted_sample_n / Discrete.flatten_n
    (tests/golden/make_categorical_golden.py)."""
    g = np.load(GOLDEN)
    p, q, onehot = g["p"], g["q"], g["onehot"]
    from rllab_b200.distributions.categorical import Categorical
    from rllab_b200.spaces import Discrete
    d = Categorical(int(g["n"]))
    assert d.dist_info_keys == ["prob"]
    for ours in (C.kl(q, p), d.kl(dict(prob=q), dict(prob=p))):
        np.testing.assert_allclose(ours, g["kl"], rtol=1e-12, atol=1e-15)
    for ours in (C.log_likelihood(onehot, p), d.log_likelihood(onehot, dict(prob=p))):
        np.testing.assert_allclose(ours, g["loglik"], rtol=1e-12, atol=1e-15)
    for ours in (C.entropy(p), d.entropy(dict(prob=p))):
        np.testing.assert_allclose(ours, g["entropy"], rtol=1e-12, atol=1e-15)
    np.testing.assert_array_equal(Discrete(int(g["n"])).flatten_n(g["idx"]), onehot)
    np.testing.assert_array_equal(C.weighted_sample_n(p, g["ws_u"]), g["ws_idx"])
    # the host API's weighted_sample draws np.random.rand() once per call, in order, like special.weighted_sample
    dsp = Discrete(int(g["n"]))
    np.random.seed(123)
    np.testing.assert_array_equal([dsp.weighted_sample(row) for row in p], g["ws_idx"])
    # clipping: a row summing below u picks the last index
    assert list(C.weighted_sample_n(np.array([[0.3, 0.3, 0.3999999]] * 2), [0.2, 0.99999999])) == [0, 2]


def test_cartpole_v0_step_matches_gym_formula():
    env = C.CartPoleV0()
    s = np.array([0.01, -0.02, 0.03, 0.04])
    ns, r, done = env.step(s, 1)
    # hand-computed from gym 0.7.4 cartpole.py with force +10
    x, xd, th, thd = s
    temp = (10.0 + 0.05 * thd * thd * np.sin(th)) / 1.1
    thacc = (9.8 * np.sin(th) - np.cos(th) * temp) / (0.5 * (4.0 / 3.0 - 0.1 * np.cos(th) ** 2 / 1.1))
    xacc = temp - 0.05 * thacc * np.cos(th) / 1.1
    np.testing.assert_allclose(ns, [x + 0.02 * xd, xd + 0.02 * xacc, th + 0.02 * thd, thd + 0.02 * thacc], rtol=1e-15)
    assert r == 1.0 and not done
    ns, r, done = env.step(np.array([0.0, 0.0, 0.2095, 0.0]), 0)
    assert done and r == 1.0                                                  # |theta| > 12 deg: terminal, reward 1
    ns, _, done = env.step(np.array([2.399, 0.1, 0.0, 0.0]), 1)
    assert done                                                               # x > 2.4
    np.testing.assert_allclose(env.reset([0.0, 0.5, 1.0, 0.25]), [-0.05, 0.0, 0.05, -0.025])


# ---------------------------------------------------------------- host API (no device)
def _lib_or_skip():
    from rllab_b200 import _lib as L
    if not os.path.exists(L.LIB_PATH):
        pytest.skip("library not built")
    return L


def test_discrete_space():
    from rllab_b200.spaces import Discrete
    d = Discrete(3)
    assert d.n == d.flat_dim == 3 and repr(d) == "Discrete(3)" and d == Discrete(3) and d != Discrete(2)
    np.testing.assert_array_equal(d.flatten(2), [0, 0, 1])
    np.testing.assert_array_equal(d.flatten_n([1, 0]), [[0, 1, 0], [1, 0, 0]])
    assert d.unflatten([0, 1, 0]) == 1
    assert list(d.unflatten_n(np.array([[0, 0, 1], [1, 0, 0]]))) == [2, 0]
    assert d.contains(np.int64(2)) and not d.contains(np.int64(3))
    np.random.seed(4)
    u = np.random.rand(50)
    np.random.seed(4)
    w = np.array([0.1, 0.6, 0.3])
    got = [d.weighted_sample(w) for _ in range(50)]
    assert got == list(C.weighted_sample_n(np.tile(w, (50, 1)), u))


def test_gym_cartpole_env_and_policy_shapes():
    L = _lib_or_skip()
    from rllab_b200.envs.gym_env import GymEnv
    from rllab_b200.envs.normalized_env import normalize
    from rllab_b200.policies.categorical_mlp_policy import CategoricalMLPPolicy
    from rllab_b200.spaces import Discrete
    from rllab_b200 import ops
    assert L.env_num_actions(L.ENV_GYM_CARTPOLE) == 2
    assert L.env_num_actions(L.ENV_CARTPOLE) == 0
    info = L.env_info(L.ENV_GYM_CARTPOLE)
    assert (info["obs_dim"], info["act_dim"], info["state_dim"], info["reset_dim"]) == (4, 1, 4, 4)
    env = normalize(GymEnv("CartPole-v0"))
    assert env.horizon == 200
    assert env.action_space == Discrete(2) and env.observation_space.flat_dim == 4
    pol = CategoricalMLPPolicy(env_spec=env, hidden_sizes=(32, 32), seed=1)
    P = 4 * 32 + 32 + 32 * 32 + 32 + 32 * 2 + 2
    assert pol.n_params == P == L.categorical_num_params(4, 32, 32, 2)
    assert pol.get_param_shapes() == [(4, 32), (32,), (32, 32), (32,), (32, 2), (2,)]
    assert ops.is_categorical(pol.dims) and tuple(pol.dims) == (4, 32, 32, 2)
    th = pol.get_param_values()
    W0, b0, W1, b1, Wo, bo = pol.flat_to_params(th)
    for W in (W0, W1, Wo):
        a = np.sqrt(6.0 / sum(W.shape))
        assert np.abs(W).max() <= a and np.abs(W).max() > 0.5 * a
    assert not (b0.any() or b1.any() or bo.any())
    np.testing.assert_array_equal(th, C.init_params(C.CatDims(4, (32, 32), 2), np.random.RandomState(1)))
    with pytest.raises(L.B200RLError):
        L.categorical_num_params(4, 64, 64, 2)


def test_policy_rejects_unsupported_arguments_and_pickles():
    _lib_or_skip()
    from rllab_b200.envs.gym_env import GymEnv
    from rllab_b200.envs.normalized_env import normalize
    from rllab_b200.policies.categorical_mlp_policy import CategoricalMLPPolicy
    from rllab_b200.algos.cem import CEM
    env = normalize(GymEnv("CartPole-v0"))
    for kw in (dict(prob_network=object()), dict(hidden_nonlinearity=np.tanh), dict(num_seq_inputs=2),
               dict(hidden_sizes=(64, 64))):
        with pytest.raises(NotImplementedError):
            CategoricalMLPPolicy(env_spec=env, **kw)
    pol = CategoricalMLPPolicy(env_spec=env, seed=2)
    pol.set_param_values(pol.get_param_values() + 1.0)
    back = pickle.loads(pickle.dumps(pol))
    np.testing.assert_array_equal(back.get_param_values(), pol.get_param_values())
    assert back.version == 1
    with pytest.raises(NotImplementedError):
        CEM(env, pol)
    with pytest.raises(NotImplementedError):
        GymEnv("MountainCar-v0")
