"""CPU: the float64 GRU oracle (tests/gru_oracle.py) against torch.autograd in float64 -- loss/KL, the BPTT gradients
(surrogate, KL, KL-penalised) and the Fisher-vector product by double backward -- on lanes whose paths restart mid-lane,
with and without masked paths; its forward against torch.nn.GRU; and the host-side GaussianGRUPolicy surface."""
import numpy as np
import pytest

import gru_oracle as G

torch = pytest.importorskip("torch")

DIMS = G.GruDims(4, 32, 1, True)


def _case(seed, masked, inc=True, N=6, T=23):
    dims = G.GruDims(4, 32, 1, inc)
    rng = np.random.RandomState(seed)
    theta = G.init_params(dims, rng) + 0.1 * rng.randn(dims.P)
    theta[-1] = -0.3
    lanes = G.synthetic_lanes(dims, N, T, rng, theta, path_len=(1, 9), masked_frac=0.3 if masked else 0.0)
    return dims, theta, lanes


def _torch_mean(th, lanes, dims):
    """The recurrent dist_info_sym in torch: mean [T][N][A] and log_std."""
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
        st = torch.tensor(start)[:, None]
        h = torch.where(st, torch.zeros_like(h), h)
        x = torch.tensor(x)
        r = torch.sigmoid(x @ p["W_xr"] + h @ p["W_hr"] + p["b_r"])
        u = torch.sigmoid(x @ p["W_xu"] + h @ p["W_hu"] + p["b_u"])
        c = torch.tanh(x @ p["W_xc"] + r * (h @ p["W_hc"]) + p["b_c"])
        h = (1 - u) * h + u * c
        out.append(h @ p["W_out"] + p["b_out"])
    return torch.stack(out), p["log_std"]


def _torch_terms(th, lanes, dims, old_mean=None):
    mu, ls = _torch_mean(th, lanes, dims)
    act = torch.tensor(np.moveaxis(lanes["act"], 0, -1).astype(np.float64))
    om = torch.tensor(np.moveaxis(lanes["old_mean"], 0, -1).astype(np.float64)) if old_mean is None else old_mean
    ls_old = torch.tensor(lanes["old_log_std"].astype(np.float64))
    z = (act - mu) / torch.exp(ls)
    zo = (act - om) / torch.exp(ls_old)
    logp = -ls.sum() - 0.5 * (z * z).sum(-1) - 0.5 * dims.A * np.log(2 * np.pi)
    logp_old = -ls_old.sum() - 0.5 * (zo * zo).sum(-1) - 0.5 * dims.A * np.log(2 * np.pi)
    num = (om - mu) ** 2 + torch.exp(2 * ls_old) - torch.exp(2 * ls)
    kl = (num / (2 * torch.exp(2 * ls) + 1e-8) + ls - ls_old).sum(-1)
    v = torch.tensor(G.valid_of(lanes))
    adv = torch.tensor(lanes["adv"].astype(np.float64))
    trpo = -(torch.exp(logp - logp_old) * adv)[v].mean()
    vpg = -(logp * adv)[v].mean()
    return trpo, vpg, kl[v].mean(), kl[v].max()


@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("inc", [True, False])
def test_loss_and_gradients_match_autograd(masked, inc):
    dims, theta, lanes = _case(1 + int(masked) + 2 * int(inc), masked, inc)
    th = torch.tensor(theta, requires_grad=True)
    trpo, vpg, mkl, xkl = _torch_terms(th, lanes, dims)
    for kind, ref in (("trpo", trpo), ("vpg", vpg)):
        lo = G.loss_kl(theta, lanes, dims, kind)
        np.testing.assert_allclose(lo, [ref.item(), mkl.item(), xkl.item()], rtol=1e-12, atol=1e-14)
        g_ref = torch.autograd.grad(ref, th, retain_graph=True)[0].numpy()
        np.testing.assert_allclose(G.grad(theta, lanes, dims, kind), g_ref, rtol=1e-10, atol=1e-13)
        gp_ref = torch.autograd.grad(ref + 0.7 * mkl, th, retain_graph=True)[0].numpy()
        np.testing.assert_allclose(G.grad(theta, lanes, dims, kind, penalty=0.7), gp_ref, rtol=1e-10, atol=1e-13)
    gk_ref = torch.autograd.grad(mkl, th)[0].numpy()
    np.testing.assert_allclose(G.grad(theta, lanes, dims, "kl"), gk_ref, rtol=1e-10, atol=1e-13)


@pytest.mark.parametrize("masked", [False, True])
def test_fisher_product_matches_double_backward(masked):
    dims, theta, lanes = _case(7 + int(masked), masked)
    mean, _ = G.forward(theta, lanes, dims)
    lanes["old_mean"] = mean                          # exactly theta_old
    lanes["old_log_std"] = G.unpack(theta, dims)["log_std"].copy()
    x = np.random.RandomState(3).randn(dims.P)
    th = torch.tensor(theta, requires_grad=True)
    mu_old = torch.tensor(np.moveaxis(mean, 0, -1))
    _, _, mkl, _ = _torch_terms(th, lanes, dims, old_mean=mu_old)
    (g,) = torch.autograd.grad(mkl, th, create_graph=True)
    (hx,) = torch.autograd.grad(g @ torch.tensor(x), th)
    np.testing.assert_allclose(G.fvp(theta, lanes, dims, x, reg_coeff=0.0), hx.numpy(), rtol=1e-9, atol=1e-12)


def test_tangent_matches_finite_difference():
    dims, theta, lanes = _case(11, False)
    x = np.random.RandomState(5).randn(dims.P)
    e = 1e-6
    fd = (G.forward(theta + e * x, lanes, dims)[0] - G.forward(theta - e * x, lanes, dims)[0]) / (2 * e)
    np.testing.assert_allclose(np.moveaxis(G.tangent_mean(theta, lanes, dims, x), -1, 0), fd, rtol=1e-6, atol=1e-8)


def test_forward_matches_torch_gru():
    """torch.nn.GRU runs this cell with W_z = -W_u, b_z = -b_u (z = 1 - u) and b_hn = 0 (one path per lane)."""
    dims, theta, lanes = _case(13, False, N=5, T=17)
    lanes["tstep"] = np.tile(np.arange(17, dtype=np.uint16)[:, None], (1, 5))
    p = G.unpack(theta, dims)
    gru = torch.nn.GRU(dims.I, dims.H).double()
    with torch.no_grad():
        gru.weight_ih_l0.copy_(torch.tensor(np.concatenate([p["W_xr"].T, -p["W_xu"].T, p["W_xc"].T])))
        gru.weight_hh_l0.copy_(torch.tensor(np.concatenate([p["W_hr"].T, -p["W_hu"].T, p["W_hc"].T])))
        gru.bias_ih_l0.copy_(torch.tensor(np.concatenate([p["b_r"], -p["b_u"], p["b_c"]])))
        gru.bias_hh_l0.zero_()
        xs = np.stack([G.inputs(lanes, dims, t)[0] for t in range(17)])
        hs, _ = gru(torch.tensor(xs))
    mean, _ = G.forward(theta, lanes, dims)
    ref = hs.numpy() @ p["W_out"] + p["b_out"]
    np.testing.assert_allclose(np.moveaxis(mean, 0, -1), ref, rtol=1e-12, atol=1e-13)


def test_path_restart_resets_hidden_and_prev_action():
    """Changing anything before a path start leaves the means from that start on unchanged."""
    dims, theta, lanes = _case(17, False, N=4, T=30)
    mean0, _ = G.forward(theta, lanes, dims)
    starts = np.argwhere(lanes["tstep"][1:] == 0) + [1, 0]
    t0, n0 = starts[len(starts) // 2]
    lanes2 = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in lanes.items()}
    lanes2["obs"][:, :t0, n0] += 1.0
    lanes2["act"][:, :t0, n0] -= 2.0
    mean1, _ = G.forward(theta, lanes2, dims)
    np.testing.assert_array_equal(mean1[:, t0:, n0], mean0[:, t0:, n0])
    assert np.abs(mean1[:, t0 - 1, n0] - mean0[:, t0 - 1, n0]).max() > 0


def test_param_layout():
    assert DIMS.P == 3 * (5 * 32 + 32 * 32 + 32) + 32 + 1 + 1 == 3682
    assert G.GruDims(4, 32, 1, False).P == 3 * (4 * 32 + 32 * 32 + 32) + 34


def test_policy_surface_without_gpu():
    from rllab_b200.envs.box2d.cartpole_env import CartpoleEnv
    from rllab_b200.envs.normalized_env import normalize
    from rllab_b200.policies.gaussian_gru_policy import GaussianGRUPolicy
    from rllab_b200 import _lib
    try:
        _lib.load()
    except _lib.B200RLError:
        pytest.skip("libb200rl.so not built")
    env = normalize(CartpoleEnv())
    pol = GaussianGRUPolicy(env_spec=env.spec)
    assert pol.recurrent and pol.state_info_keys == ["prev_action"] and pol.n_params == 3682
    assert [tuple(s) for s in pol.get_param_shapes()] == [tuple(s) for s in DIMS.shapes]
    vals = pol.get_param_values()
    assert vals.shape == (3682,) and np.all(vals[-1:] == 0.0)
    assert GaussianGRUPolicy(env_spec=env.spec, state_include_action=False).state_info_keys == []
    with pytest.raises(Exception):
        GaussianGRUPolicy(env_spec=env.spec, hidden_sizes=(64,))
    import pickle
    pol2 = pickle.loads(pickle.dumps(pol))
    np.testing.assert_array_equal(pol2.get_param_values(), vals)
