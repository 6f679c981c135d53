"""CPU: the float64 categorical GRU oracle (tests/categorical_gru_oracle.py) against torch.autograd in float64 -- loss /
KL, the BPTT gradients (surrogate, surrogate + KL penalty, KL alone) and the Gauss-Newton Fisher-vector product (the
logit block by double backward) -- on lanes whose paths restart mid-lane, with and without masked paths, for both values
of state_include_action; and the host-side CategoricalGRUPolicy / RecurrentCategorical surface."""
import numpy as np
import pytest

import categorical_gru_oracle as C
import gru_oracle as G

torch = pytest.importorskip("torch")


def _case(seed, masked, inc):
    dims = C.CatGruDims(4, 32, 2, inc)
    rng = np.random.RandomState(seed)
    theta = C.init_params(dims, rng) + 0.1 * rng.randn(dims.P)
    lanes = C.synthetic_lanes(dims, 6, 23, rng, theta, path_len=(1, 9), masked_frac=0.3 if masked else 0.0)
    return dims, theta, lanes


def _torch_logits(th, lanes, dims):
    p, k = {}, 0
    for name, s in zip(dims.names, dims.shapes):
        n = int(np.prod(s))
        p[name] = th[k:k + n].reshape(s)
        k += n
    T, N = lanes["tstep"].shape
    h = torch.zeros((N, dims.H), dtype=torch.float64)
    out = []
    for t in range(T):
        x, start = G.inputs(lanes, dims, t)
        h = torch.where(torch.tensor(start)[:, None], torch.zeros_like(h), h)
        x = torch.tensor(x)
        r = torch.sigmoid(x @ p["W_xr"] + h @ p["W_hr"] + p["b_r"])
        u = torch.sigmoid(x @ p["W_xu"] + h @ p["W_hu"] + p["b_u"])
        c = torch.tanh(x @ p["W_xc"] + r * (h @ p["W_hc"]) + p["b_c"])
        h = (1 - u) * h + u * c
        out.append(h @ p["W_out"] + p["b_out"])
    return torch.stack(out)


def _kl(q, z):
    return (q * (torch.log(q + 1e-8) - torch.log(torch.softmax(z, -1) + 1e-8))).sum(-1)


def _torch_terms(th, lanes, dims):
    z = _torch_logits(th, lanes, dims)
    pr = torch.softmax(z, -1)
    x = torch.tensor(np.moveaxis(lanes["act"], 0, -1).astype(np.float64))
    q = torch.tensor(np.moveaxis(lanes["old_prob"], 0, -1).astype(np.float64))
    adv = torch.tensor(lanes["adv"].astype(np.float64))
    v = torch.tensor(G.valid_of(lanes))
    trpo = -(((pr * x).sum(-1) + 1e-8) / ((q * x).sum(-1) + 1e-8) * adv)[v].mean()
    vpg = -(torch.log((pr * x).sum(-1) + 1e-8) * adv)[v].mean()
    kl = _kl(q, z)[v]
    return dict(trpo=trpo, vpg=vpg, kl=kl.mean(), kl_max=kl.max())


CASES = [(s, m, inc) for s, m in ((0, False), (1, True)) for inc in (True, False)]


@pytest.mark.parametrize("seed,masked,inc", CASES)
def test_loss_and_gradients_match_autograd(seed, masked, inc):
    dims, theta, lanes = _case(seed, masked, inc)
    th = torch.tensor(theta + 0.02 * np.random.RandomState(seed + 7).randn(dims.P), requires_grad=True)
    t = _torch_terms(th, lanes, dims)
    for kind in ("trpo", "vpg"):
        surr, kl, kl_max = C.loss_kl(th.detach().numpy(), lanes, dims, kind)
        np.testing.assert_allclose([surr, kl, kl_max], [t[kind].item(), t["kl"].item(), t["kl_max"].item()],
                                   rtol=0, atol=1e-12)
        for penalty in (0.0, 0.5):
            g_ref = torch.autograd.grad(t[kind] + penalty * t["kl"], th, retain_graph=True)[0].numpy()
            g = C.grad(th.detach().numpy(), lanes, dims, kind, penalty)
            assert np.max(np.abs(g - g_ref)) <= 1e-10 * max(1.0, np.max(np.abs(g_ref)))
    g_ref = torch.autograd.grad(t["kl"], th)[0].numpy()
    g = C.grad(th.detach().numpy(), lanes, dims, "kl")
    assert np.max(np.abs(g - g_ref)) <= 1e-10 * max(1.0, np.max(np.abs(g_ref)))


@pytest.mark.parametrize("seed,masked,inc", CASES)
def test_fvp_matches_gauss_newton_by_double_backward(seed, masked, inc):
    """J^T M J x with J x by forward mode (double-backward trick), M by double backward of the KL in the logits at
    q = p(theta_old), and J^T by backward; and its distance to the exact Hessian of mean KL, which adds O(TINY)."""
    dims, theta, lanes = _case(seed, masked, inc)
    lanes = dict(lanes, old_prob=np.moveaxis(C.forward(theta, lanes, dims)[0], -1, 0))   # theta_old exactly
    xv = np.random.RandomState(seed + 3).randn(dims.P)
    th = torch.tensor(theta, requires_grad=True)
    z = _torch_logits(th, lanes, dims)
    w = torch.zeros_like(z, requires_grad=True)
    tz = torch.autograd.grad(torch.autograd.grad(z, th, w, create_graph=True)[0], w, torch.tensor(xv))[0]
    zd = z.detach().requires_grad_(True)
    q = torch.softmax(zd, -1).detach()
    v = torch.tensor(G.valid_of(lanes))
    gz = torch.autograd.grad(_kl(q, zd)[v].sum(), zd, create_graph=True)[0]
    m = torch.autograd.grad(gz, zd, tz)[0] / v.sum()
    ref = torch.autograd.grad(z, th, m)[0].numpy() + 1e-5 * xv
    out = C.fvp(theta, lanes, dims, xv, 1e-5)
    assert np.max(np.abs(out - ref)) <= 1e-9 * np.max(np.abs(ref))
    kl = _kl(torch.tensor(np.moveaxis(lanes["old_prob"], 0, -1)), _torch_logits(th, lanes, dims))[v].mean()
    g = torch.autograd.grad(kl, th, create_graph=True)[0]
    exact = torch.autograd.grad(g, th, torch.tensor(xv))[0].numpy() + 1e-5 * xv
    assert np.max(np.abs(out - exact)) <= 1e-6 * np.max(np.abs(exact))


def test_trpo_step_satisfies_the_constraint():
    dims, theta, lanes = _case(5, True, True)
    lanes = dict(lanes, old_prob=np.moveaxis(C.forward(theta, lanes, dims)[0], -1, 0))
    new, _ = C.trpo_step(theta, lanes, dims, step_size=0.01)
    surr0 = C.loss_kl(theta, lanes, dims, "trpo")[0]
    surr, kl, _ = C.loss_kl(new, lanes, dims, "trpo")
    assert kl <= 0.01 * (1 + 1e-9) and surr < surr0


def test_rollout_resets_state_at_path_starts():
    dims = C.CatGruDims(4, 32, 2, True)
    rng = np.random.RandomState(2)
    theta = C.init_params(dims, rng)
    N, T = 5, 60
    lanes = C.rollout_cartpole_v0(theta, dims, N, T, 30, rng.rand(T, N), rng.rand(T + 1, 4, N))
    assert np.all(lanes["act"].sum(0) == 1.0)
    # the recorded probabilities are the forward pass of the recorded lanes (h / prev_action reset where tstep == 0)
    p, _, _ = C.forward(theta, lanes, dims)
    np.testing.assert_allclose(np.moveaxis(p, -1, 0), lanes["mean"], rtol=0, atol=1e-14)
    assert (lanes["tstep"] == 0).sum() > N


def test_recurrent_categorical_matches_the_flat_distribution():
    from rllab_b200.distributions.categorical import Categorical
    from rllab_b200.distributions.recurrent_categorical import RecurrentCategorical
    rng = np.random.RandomState(0)
    p = rng.dirichlet(np.ones(2), size=(3, 7))
    q = rng.dirichlet(np.ones(2), size=(3, 7))
    x = np.eye(2)[rng.randint(0, 2, size=(3, 7))]
    d, flat = RecurrentCategorical(2), Categorical(2)
    np.testing.assert_allclose(d.kl(dict(prob=p), dict(prob=q)),
                               flat.kl(dict(prob=p.reshape(-1, 2)), dict(prob=q.reshape(-1, 2))).reshape(3, 7))
    np.testing.assert_allclose(d.log_likelihood(x, dict(prob=p)),
                               flat.log_likelihood(x.reshape(-1, 2), dict(prob=p.reshape(-1, 2))).reshape(3, 7))
    np.testing.assert_allclose(d.entropy(dict(prob=p)), flat.entropy(dict(prob=p.reshape(-1, 2))).reshape(3, 7))
    assert d.dist_info_keys == ["prob"] and d.dim == 2


def test_policy_surface_without_a_gpu():
    from rllab_b200 import _lib as L
    from rllab_b200.envs.gym_env import GymEnv
    from rllab_b200.envs.normalized_env import normalize
    from rllab_b200.policies.categorical_gru_policy import CategoricalGRUPolicy
    from rllab_b200 import ops
    import os
    if not os.path.exists(L.LIB_PATH):
        pytest.skip("library not built")
    env = normalize(GymEnv("CartPole-v0"))
    for inc in (True, False):
        pol = CategoricalGRUPolicy(env.spec, state_include_action=inc)
        dims = C.CatGruDims(4, 32, 2, inc)
        assert pol.n_params == dims.P == sum(int(np.prod(s)) for s in pol.get_param_shapes())
        assert [tuple(s) for s in pol.get_param_shapes()] == [tuple(s) for s in dims.shapes]
        assert ops.is_gru(pol.dims) and ops.is_categorical(pol.dims) and pol.recurrent
        assert pol.state_info_keys == (["prev_action"] if inc else [])
    with pytest.raises(NotImplementedError):
        CategoricalGRUPolicy(env.spec, feature_network=object())
    with pytest.raises(NotImplementedError):
        CategoricalGRUPolicy(env.spec, hidden_nonlinearity=np.sin)
    with pytest.raises(L.B200RLError):
        CategoricalGRUPolicy(env.spec, hidden_dim=16)
