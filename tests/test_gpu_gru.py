"""GPU: GaussianGRUPolicy -- the fused recurrent rollout and get_actions, the loss/KL, BPTT gradient (+ KL penalty) and
Fisher-vector passes in float32, and the float64 parity passes, against the float64 oracle (tests/gru_oracle.py) on
lanes whose paths restart mid-lane, masked and unmasked; whole TRPO steps (float32, precision="f64",
FiniteDifferenceHvp), VPG / PPO / ERWR through the host API, the recurrent wire format, and the reference's
examples/trpo_cartpole_recurrent.py."""
import os

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import gru_oracle as G          # noqa: E402

DIMS = G.GruDims(4, 32, 1, True)
# float32 BPTT error bound per T, relative to the largest entry of the float64 result: the largest error an H100 80GB
# HBM3 measured over the passes, lane counts and mask settings of test_passes_match_oracle at that T (DESIGN.md
# section 5: 1.2e-6, 4.7e-6, 7.9e-7, 2.6e-6 at T = 1, 16, 100, 500; the T = 16 maximum is the 20000-lane case, whose
# penalised gradients sum the most samples) with a margin of about 4x.
F32_TOL = {1: 5e-6, 16: 2e-5, 100: 4e-6, 500: 1e-5}


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from rllab_b200 import _lib
    _lib.load()
    from rllab_b200.misc import logger
    logger.set_quiet(True)
    return torch.device("cuda:0")


def _L():
    from rllab_b200 import _lib
    return _lib


def _ops():
    from rllab_b200 import ops
    return ops


def _f32(a):
    return np.asarray(a, dtype=np.float32).astype(np.float64)


def _rel(a, b):
    return np.max(np.abs(a - b)) / np.max(np.abs(b))


def _theta(dims, seed, scale=0.2):
    rng = np.random.RandomState(seed)
    th = G.init_params(dims, rng) + scale * rng.randn(dims.P)
    th[-dims.A:] = -0.5
    return _f32(th)


def _rollout(dev, dims, th32, N, T, mpl, eps=None, rr=None, seed=3, it=0):
    ops = _ops()
    b = ops.LaneBatch(4, 1, N, T, dev)
    b.recurrent = True
    ops.gru_rollout(_ops().GRUDims(4, 32, 1, dims.inc), th32, b, mpl, _L().ENV_CARTPOLE, eps, rr, seed, it)
    return b


@pytest.mark.parametrize("N,T", [(1, 1), (77, 2), (77, 100), (37 * 128, 100), (40000, 7), (150000, 3)])
@pytest.mark.parametrize("inc", [True, False])
def test_rollout_against_oracle(dev, N, T, inc):
    """Each recorded mean is the oracle's GRU on the recorded lanes (h and prev_action reset at every path start), the
    action is mean + std eps, the env steps from the recorded obs; the Philox run is the injected-noise run bit for
    bit, and a replay reproduces it."""
    L = _L()
    dims = G.GruDims(4, 32, 1, inc)
    mpl = 13
    theta = _theta(dims, 2)
    th32 = torch.tensor(theta, dtype=torch.float32, device=dev)
    eps = torch.empty((T, 1, N), dtype=torch.float32, device=dev)
    rr = torch.empty((T + 1, 4, N), dtype=torch.float32, device=dev)
    L_ = _ops()
    L_.fill_noise(eps, T, 0, 1, N, 0, L.NOISE_NORMAL, 3, 0, 0)
    L_.fill_noise(rr, T + 1, 0, 4, N, 0, L.NOISE_UNIFORM, 3, 0, 1)
    b = _rollout(dev, dims, th32, N, T, mpl, eps, rr)
    t = b.to_numpy()
    lanes = dict(obs=t["obs"], act=t["act"], tstep=t["tstep"])
    mean_ref, _ = G.forward(theta, lanes, dims)
    np.testing.assert_allclose(t["mean"], mean_ref, rtol=0, atol=2e-5)
    np.testing.assert_allclose(t["act"], t["mean"] + np.exp(theta[-1]) * eps.cpu().numpy()[:, 0][None], rtol=0, atol=1e-5)
    assert t["log_std"][0] == np.float32(theta[-1])
    ends = (t["flags"] & L.FLAG_END) != 0
    assert np.all(t["tstep"][0] == 0)
    if T > 1:
        np.testing.assert_array_equal(t["tstep"][1:], np.where(ends[:-1], 0, t["tstep"][:-1] + 1))
        assert np.all(t["tstep"] < mpl)
        # dynamics of the continuing steps, from the recorded obs and action
        from oracle import envs as E
        env = E.make("cartpole", np.float64)
        for s in range(T - 1):
            ns, _, _ = env.step(t["obs"][:, s].astype(np.float64), env.scale_action(t["act"][:, s].astype(np.float64)))
            cont = ~ends[s]
            np.testing.assert_allclose(t["obs"][:, s + 1][:, cont], ns[:, cont], rtol=1e-4, atol=1e-4)
    bp = _rollout(dev, dims, th32, N, T, mpl)
    bq = _rollout(dev, dims, th32, N, T, mpl)
    tp, tq = bp.to_numpy(), bq.to_numpy()
    for k in ("obs", "act", "mean", "rew", "flags", "tstep"):
        np.testing.assert_array_equal(tp[k], t[k], err_msg=k)
        np.testing.assert_array_equal(tq[k], t[k], err_msg=k)


def test_get_actions_against_oracle_and_philox(dev):
    L, ops = _L(), _ops()
    n = 333
    rng = np.random.RandomState(4)
    theta = _theta(DIMS, 5, 0.3)
    th32 = torch.tensor(theta, dtype=torch.float32, device=dev)
    obs, pa, h = (rng.randn(4, n).astype(np.float32), rng.randn(1, n).astype(np.float32),
                  np.tanh(rng.randn(32, n)).astype(np.float32))
    obs_d, pa_d, h_d = (torch.tensor(a, device=dev) for a in (obs, pa, h))
    eps = torch.empty((1, 1, n), dtype=torch.float32, device=dev)
    ops.fill_noise(eps, 1, 5, 1, n, 9, L.NOISE_NORMAL, 11, 2, 0)
    outs = []
    for e in (eps.view(1, n), None):
        act, mean = (torch.empty((1, n), dtype=torch.float32, device=dev) for _ in range(2))
        h_out = torch.empty((32, n), dtype=torch.float32, device=dev)
        ls = torch.empty(1, dtype=torch.float32, device=dev)
        if e is None:
            L.call("b200rl_gru_get_actions", L.ptr(th32), 4, 32, 1, 1, L.ptr(obs_d), L.ptr(pa_d), L.ptr(h_d), n, None,
                   11, 2, 5, 9, L.ptr(act), L.ptr(mean), L.ptr(h_out), L.ptr(ls), ops._stream())
        else:
            ops.gru_get_actions(th32, ops.GRUDims(4, 32, 1, True), obs_d, pa_d, h_d, n, e, 0, 0, 0, 0, act, mean,
                                h_out, ls)
        outs.append([v.cpu().numpy() for v in (act, mean, h_out, ls)])
    for a, b in zip(*outs):
        np.testing.assert_array_equal(a, b)
    p = G.unpack(theta, DIMS)
    x = np.concatenate([obs.T, pa.T], axis=1).astype(np.float64)
    hn, _, _, _, _ = G.cell(p, x, h.T.astype(np.float64))
    np.testing.assert_allclose(outs[0][2], hn.T, rtol=0, atol=2e-6)
    np.testing.assert_allclose(outs[0][1], (hn @ p["W_out"] + p["b_out"]).T, rtol=0, atol=1e-5)


def test_loss_at_theta_old_is_exact(dev):
    """The loss pass recomputes the rollout's mean bit for bit: mean and max KL exactly 0, likelihood ratio exactly 1."""
    ops, L = _ops(), _L()
    N, T = 1000, 100
    theta = _theta(DIMS, 6)
    th32 = torch.tensor(theta, dtype=torch.float32, device=dev)
    b = _rollout(dev, DIMS, th32, N, T, 37)
    adv = np.random.RandomState(1).randn(T, N).astype(np.float32)
    b.adv.copy_(torch.tensor(adv))
    out = torch.empty(3, dtype=torch.float64, device=dev)
    dims = ops.GRUDims(4, 32, 1, True)
    ops.loss_kl(L.LOSS_TRPO, th32, dims, None, b, out)
    loss, mkl, xkl = out.cpu().numpy()
    assert mkl == 0.0 and xkl == 0.0
    np.testing.assert_allclose(loss, -adv.astype(np.float64).mean(), rtol=1e-12, atol=1e-14)
    g = torch.empty(DIMS.P, dtype=torch.float64, device=dev)
    tri = torch.empty(3, dtype=torch.float64, device=dev)
    ops.grad(L.LOSS_TRPO, th32, dims, None, b, g, tri)
    assert tri[1].item() == 0.0 and tri[2].item() == 0.0


def _lane_case(dev, N, T, masked, seed):
    """Synthetic lanes recorded at theta (paths of random lengths) as a LaneBatch, and the oracle's dict."""
    ops, L = _ops(), _L()
    rng = np.random.RandomState(seed)
    theta = _theta(DIMS, seed)
    lanes = G.synthetic_lanes(DIMS, N, T, rng, theta, path_len=(1, min(T, 60)), masked_frac=0.3 if masked else 0.0)
    b = ops.LaneBatch(4, 1, N, T, dev)
    b.recurrent = True
    for k, src in (("obs", "obs"), ("act", "act"), ("mean", "old_mean")):
        getattr(b, k).copy_(torch.tensor(lanes[src]))
    b.tstep.copy_(torch.tensor(lanes["tstep"].astype(np.int16)).view(torch.uint16))
    b.log_std.copy_(torch.tensor(lanes["old_log_std"]))
    b.adv.copy_(torch.tensor(lanes["adv"]))
    if masked:
        b.flags.copy_(torch.tensor(np.where(lanes["valid"], 0, L.FLAG_MASKED).astype(np.uint8)))
        b.count.fill_(float(lanes["valid"].sum()))
        b.masked = True
    lanes["old_mean"] = lanes["old_mean"].astype(np.float64)
    return b, theta, lanes


# (T, lanes): 20000 lanes are 157 tiles of 128, more than one tile per CTA of the gradient pass on 132 SMs, and more
# lanes than one grid-stride round of the float64 kernel
@pytest.mark.parametrize("T,N", [(1, 37 * 128), (16, 300), (100, 77), (500, 19), (16, 20000)])
@pytest.mark.parametrize("masked", [False, True])
def test_passes_match_oracle(dev, T, N, masked):
    ops, L = _ops(), _L()
    b, theta, lanes = _lane_case(dev, N, T, masked, 10 + T + int(masked))
    dims = ops.GRUDims(4, 32, 1, True)
    th32 = torch.tensor(theta, dtype=torch.float32, device=dev)
    th64 = torch.tensor(theta, dtype=torch.float64, device=dev)
    out = torch.empty(3, dtype=torch.float64, device=dev)
    g = torch.empty(DIMS.P, dtype=torch.float64, device=dev)
    tol = F32_TOL[T]
    errs = {}
    for kind, lk in (("trpo", L.LOSS_TRPO), ("vpg", L.LOSS_VPG)):
        ref = G.loss_kl(theta, lanes, DIMS, kind)
        ops.loss_kl(lk, th32, dims, None, b, out)
        np.testing.assert_allclose(out.cpu().numpy(), ref, rtol=1e-5, atol=1e-7)
        ops.update_f64(0, lk, th64, dims, None, b, None, 0.0, 0.0, None, out)
        np.testing.assert_allclose(out.cpu().numpy(), ref, rtol=1e-10, atol=1e-13)
        for pen in (0.0, 0.5):
            gref = G.grad(theta, lanes, DIMS, kind, penalty=pen)
            if pen:
                ops.grad_penalized(lk, pen, th32, dims, None, b, g, out)
            else:
                ops.grad(lk, th32, dims, None, b, g, out)
            errs["grad_%s_%g" % (kind, pen)] = _rel(g.cpu().numpy(), gref)
        ops.update_f64(1, lk, th64, dims, None, b, None, 0.0, 0.0, g, out)
        np.testing.assert_allclose(g.cpu().numpy(), G.grad(theta, lanes, DIMS, kind), rtol=0,
                                   atol=1e-10 * np.abs(G.grad(theta, lanes, DIMS, kind)).max())
    # the KL gradient away from theta_old (FiniteDifferenceHvp evaluates it at theta +- eps x)
    th_kl = theta + 1e-3 * np.random.RandomState(T + 1).randn(DIMS.P)
    gk = G.grad(th_kl, lanes, DIMS, "kl")
    ops.update_f64(1, L.LOSS_KL, torch.tensor(th_kl, device=dev), dims, None, b, None, 0.0, 0.0, g, None)
    np.testing.assert_allclose(g.cpu().numpy(), gk, rtol=0, atol=1e-10 * np.abs(gk).max())
    # Fisher product at theta_old: old_mean = the policy's own mean
    b.mean.copy_(torch.tensor(G.forward(theta, lanes, DIMS)[0].astype(np.float32)))
    lanes["old_mean"] = G.forward(theta, lanes, DIMS)[0]
    x = torch.tensor(np.random.RandomState(T).randn(DIMS.P), dtype=torch.float64, device=dev)
    ref = G.fvp(theta, lanes, DIMS, x.cpu().numpy(), 1e-5)
    hx = torch.empty_like(x)
    ops.fvp(th32, dims, None, b, x, 1e-5, 1.0, hx)
    errs["fvp"] = _rel(hx.cpu().numpy(), ref)
    hc = b.hcache(32, 0)
    ops.grad(L.LOSS_TRPO, th32, dims, None, b, g, out, hc)           # writes the cache at theta
    hx2 = torch.empty_like(x)
    ops.fvp(th32, dims, None, b, x, 1e-5, 1.0, hx2, hc)
    np.testing.assert_array_equal(hx2.cpu().numpy(), hx.cpu().numpy())
    ops.update_f64(2, L.LOSS_TRPO, th64, dims, None, b, x, 1e-5, 1.0, hx, None)
    np.testing.assert_allclose(hx.cpu().numpy(), ref, rtol=0, atol=1e-10 * np.abs(ref).max())
    print("GRU float32 error T=%d masked=%s: %s" % (T, masked, " ".join("%s=%.2e" % kv for kv in sorted(errs.items()))))
    assert max(errs.values()) < tol, errs


def _algo(algo_name, n_envs=40, T=100, n_itr=3, **kw):
    from rllab_b200.algos.erwr import ERWR
    from rllab_b200.algos.ppo import PPO
    from rllab_b200.algos.trpo import TRPO
    from rllab_b200.algos.vpg import VPG
    from rllab_b200.baselines.linear_feature_baseline import LinearFeatureBaseline
    from rllab_b200.envs.box2d.cartpole_env import CartpoleEnv
    from rllab_b200.envs.normalized_env import normalize
    from rllab_b200.policies.gaussian_gru_policy import GaussianGRUPolicy
    env = normalize(CartpoleEnv())
    policy = GaussianGRUPolicy(env_spec=env.spec, seed=3)
    args = dict(env=env, policy=policy, baseline=LinearFeatureBaseline(env_spec=env.spec), batch_size=n_envs * T,
                max_path_length=T, n_itr=n_itr, discount=0.99, sampler_args=dict(n_envs=n_envs, seed=7))
    args.update(kw)
    return dict(trpo=TRPO, vpg=VPG, ppo=PPO, erwr=ERWR)[algo_name](**args)


def _oracle_lanes(sd):
    b = sd.lane_batch
    t = b.to_numpy()
    return dict(obs=t["obs"], act=t["act"], tstep=t["tstep"], adv=b.adv.cpu().numpy(),
                old_mean=t["mean"].astype(np.float64), old_log_std=t["log_std"], valid=b.valid_mask())


@pytest.mark.parametrize("precision,tol", [("f32", 5e-3), ("f64", 1e-5)])
def test_trpo_step_matches_oracle(dev, precision, tol):
    algo = _algo("trpo", optimizer_args=dict(cg_iters=4, precision=precision))
    algo.start_worker()
    algo.init_opt()
    sd = algo.sampler.process_samples(0, algo.sampler.obtain_samples(0))
    lanes = _oracle_lanes(sd)
    theta0 = algo.policy.get_param_values()
    theta0 = algo.policy.theta32.double().cpu().numpy() if precision == "f32" else theta0
    algo.optimize_policy(0, sd)
    theta_dev = algo.policy.get_param_values()
    theta_ref, info = G.trpo_step(theta0, lanes, DIMS, 0.01, 4)
    li = algo.optimizer.last_info
    assert not li["rejected"] and not info["rejected"] and li["n_iter"] == info["n_iter"]
    assert _rel(theta_dev - theta0, theta_ref - theta0) < tol, _rel(theta_dev - theta0, theta_ref - theta0)
    assert 0 < li["constraint_val"] <= 0.01


def test_trpo_finite_difference_hvp(dev):
    from rllab_b200.optimizers.conjugate_gradient_optimizer import ConjugateGradientOptimizer, FiniteDifferenceHvp
    algo = _algo("trpo", optimizer=ConjugateGradientOptimizer(cg_iters=4, hvp_approach=FiniteDifferenceHvp(base_eps=1e-5)))
    algo.start_worker()
    algo.init_opt()
    sd = algo.sampler.process_samples(0, algo.sampler.obtain_samples(0))
    lanes = _oracle_lanes(sd)
    theta0 = algo.policy.get_param_values()
    algo.optimize_policy(0, sd)
    theta_ref, info = G.trpo_step(theta0, lanes, DIMS, 0.01, 4)
    li = algo.optimizer.last_info
    assert not li["rejected"] and 0 < li["constraint_val"] <= 0.01
    d = algo.policy.get_param_values() - theta0
    assert _rel(d, theta_ref - theta0) < 2e-2, _rel(d, theta_ref - theta0)


@pytest.mark.parametrize("name", ["vpg", "ppo", "erwr"])
def test_first_order_and_penalty_algos_run(dev, name):
    algo = _algo(name, n_itr=2)
    theta0 = algo.policy.get_param_values()
    algo.train()
    theta1 = algo.policy.get_param_values()
    assert np.all(np.isfinite(theta1)) and np.abs(theta1 - theta0).max() > 0


def test_subsample_and_cem_are_rejected(dev):
    from rllab_b200.algos.cem import CEM
    algo = _algo("trpo", optimizer_args=dict(subsample_factor=0.5))
    algo.start_worker()
    algo.init_opt()
    sd = algo.sampler.process_samples(0, algo.sampler.obtain_samples(0))
    with pytest.raises(NotImplementedError):
        algo.optimize_policy(0, sd)
    with pytest.raises(NotImplementedError):
        CEM(env=algo.env, policy=algo.policy, n_itr=1, max_path_length=10, batch_size=10)


def test_recurrent_wire_format(dev):
    algo = _algo("trpo", n_envs=12, T=100)
    algo.start_worker()
    algo.init_opt()
    sd = algo.sampler.process_samples(0, algo.sampler.obtain_samples(0))
    paths = sd["paths"]
    for p in paths:
        np.testing.assert_array_equal(p["agent_infos"]["prev_action"][0], 0.0)
        np.testing.assert_array_equal(p["agent_infos"]["prev_action"][1:], p["actions"][:-1])
    n, Lmax = len(paths), max(len(p["rewards"]) for p in paths)
    assert "valids" in sd and sd["valids"].shape == (n, Lmax)
    np.testing.assert_array_equal(sd["valids"].sum(1), [len(p["rewards"]) for p in paths])
    assert sd["observations"].shape == (n, Lmax, 4) and sd["actions"].shape == (n, Lmax, 1)
    assert sd["agent_infos"]["prev_action"].shape == (n, Lmax, 1) and sd["advantages"].shape == (n, Lmax)
    np.testing.assert_array_equal(sd["observations"][sd["valids"] == 0], 0.0)
    # the policy's own step API reproduces the recorded means of a path (prev_action fed back, h carried)
    pol = algo.policy
    p = paths[0]
    pol.reset()
    for t in range(len(p["rewards"])):
        _, info = pol.get_action(p["observations"][t])
        np.testing.assert_allclose(info["mean"], p["agent_infos"]["mean"][t], rtol=0, atol=1e-5)
        pol._prev_actions[0] = p["actions"][t]                  # continue with the recorded action


def test_gradient_pass_ignores_stale_cache(dev):
    """A partial last tile (77 lanes): the threads past the last lane must not read the activation cache, whose first
    use finds whatever the allocator left there.  With the cache filled with NaN first, the passes are still finite and
    equal to the ones on a zeroed cache."""
    ops, L = _ops(), _L()
    b, theta, lanes = _lane_case(dev, 77, 100, False, 5)
    dims = ops.GRUDims(4, 32, 1, True)
    th32 = torch.tensor(theta, dtype=torch.float32, device=dev)
    x = torch.tensor(np.random.RandomState(2).randn(DIMS.P), dtype=torch.float64, device=dev)
    res = []
    for fill in (float("nan"), 0.0):
        hc = b.hcache(32, 0)
        g = torch.empty(DIMS.P, dtype=torch.float64, device=dev)
        hx = torch.empty_like(x)
        hc.fill_(fill)
        ops.grad(L.LOSS_TRPO, th32, dims, None, b, g, None, hc)
        hc.fill_(fill)
        ops.fvp(th32, dims, None, b, x, 1e-5, 1.0, hx)            # no valid cache: the pass rewrites it
        res.append((g.cpu().numpy(), hx.cpu().numpy()))
    for a in res[0]:
        assert np.all(np.isfinite(a))
    np.testing.assert_array_equal(res[0][0], res[1][0])
    np.testing.assert_array_equal(res[0][1], res[1][1])


CURVE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "oracle_cartpole_gru_trpo_curve.json")


def test_reference_example_learns(dev):
    """examples/trpo_cartpole_recurrent.py: TRPO, GaussianGRUPolicy, LinearFeatureBaseline, batch 4000, path length
    100, FiniteDifferenceHvp(base_eps=1e-5) on normalize(CartpoleEnv()), against the band of the float64 oracle's curves
    over five seeds (tests/golden/make_cartpole_gru_curve.py; the RNG streams differ, so bands, not values), with the
    rule of test_gpu_categorical.py: at iteration 0 at most the band's top plus its width; over the last 5 iterations a
    mean of at least the lowest seed's mean less its spread."""
    import json
    from rllab_b200.algos.trpo import TRPO
    from rllab_b200.baselines.linear_feature_baseline import LinearFeatureBaseline
    from rllab_b200.envs.box2d.cartpole_env import CartpoleEnv
    from rllab_b200.envs.normalized_env import normalize
    from rllab_b200.misc import logger
    from rllab_b200.optimizers.conjugate_gradient_optimizer import ConjugateGradientOptimizer, FiniteDifferenceHvp
    from rllab_b200.policies.gaussian_gru_policy import GaussianGRUPolicy
    curves = np.array(list(json.load(open(CURVE))["AverageReturn"].values()))
    n_itr = curves.shape[1]
    first_hi = curves[:, 0].max() + (curves[:, 0].max() - curves[:, 0].min())
    late = curves[:, -5:].mean(axis=1)
    late_lo = late.min() - (late.max() - late.min())
    np.random.seed(1)
    env = normalize(CartpoleEnv())
    policy = GaussianGRUPolicy(env_spec=env.spec)
    algo = TRPO(env=env, policy=policy, baseline=LinearFeatureBaseline(env_spec=env.spec), batch_size=4000,
                max_path_length=100, n_itr=n_itr, discount=0.99, step_size=0.01,
                optimizer=ConjugateGradientOptimizer(hvp_approach=FiniteDifferenceHvp(base_eps=1e-5)))
    algo.start_worker()
    algo.init_opt()
    rets = []
    for itr in range(n_itr):
        algo.train_itr(itr)
        rets.append(logger.get_last_table()["AverageReturn"])
    print("GRU CartPole TRPO AverageReturn per iteration:", [round(r, 1) for r in rets], "bounds", first_hi, late_lo)
    assert rets[0] <= first_hi, (rets[0], first_hi)
    assert np.mean(rets[-5:]) >= late_lo, (rets, late_lo)
