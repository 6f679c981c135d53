"""GPU: CategoricalGRUPolicy -- the fused recurrent discrete-action rollout and get_actions, the loss/KL, BPTT gradient
(+ KL penalty) and Fisher-vector passes in float32, and the float64 parity passes, against the float64 oracle
(tests/categorical_gru_oracle.py) on lanes whose paths restart mid-lane, masked and unmasked, for both values of
state_include_action; saturated softmax probabilities; whole TRPO steps (float32, precision="f64",
FiniteDifferenceHvp), VPG / PPO / ERWR through the host API, the rejections of CEM / REPS / sub-sampling, and the
recurrent wire format on gym CartPole-v0."""
import os

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import categorical_gru_oracle as C   # noqa: E402
import categorical_oracle as CO      # noqa: E402

# float32 BPTT error bound per T, relative to the largest entry of the float64 result: the largest error an H100 80GB
# HBM3 measured over the passes, lane counts, mask settings and both input layouts of test_passes_match_oracle at that
# T (DESIGN.md section 5: at most 9e-7 at every T outside the 20000-lane case), with a margin of about 4x; T = 16 keeps
# the Gaussian GRU's bound for the 20000-lane case, whose penalised gradients sum the most samples.
F32_TOL = {1: 4e-6, 16: 2e-5, 100: 4e-6, 200: 4e-6}


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
    return _f32(C.init_params(dims, rng) + scale * rng.randn(dims.P))


def _dims(inc):
    return C.CatGruDims(4, 32, 2, inc), _ops().CategoricalGRUDims(4, 32, 2, inc)


def _rollout(dev, inc, th32, N, T, mpl, u=None, rr=None, seed=3, it=0):
    ops = _ops()
    b = ops.LaneBatch(4, 2, N, T, dev)
    b.recurrent = b.categorical = True
    ops.gru_rollout(ops.CategoricalGRUDims(4, 32, 2, inc), th32, b, mpl, _L().ENV_GYM_CARTPOLE, u, rr, seed, it)
    return b


@pytest.mark.parametrize("N,T", [(1, 1), (77, 2), (77, 100), (37 * 128, 100), (150000, 3)])
@pytest.mark.parametrize("inc", [True, False])
def test_rollout_against_oracle(dev, N, T, inc):
    """Each recorded prob is the oracle's net on the recorded lanes (h and the one-hot prev_action reset at every path
    start), each action weighted_sample(prob, u) of the recorded prob, the lane bookkeeping that of the categorical
    rollout; the Philox run is the injected-u run bit for bit, and a replay reproduces it."""
    L, ops = _L(), _ops()
    dims, _ = _dims(inc)
    mpl = 13
    theta = _theta(dims, 2)
    th32 = torch.tensor(theta, dtype=torch.float32, device=dev)
    u = torch.empty((T, 1, N), dtype=torch.float32, device=dev)
    rr = torch.empty((T + 1, 4, N), dtype=torch.float32, device=dev)
    ops.fill_noise(u, T, 0, 1, N, 0, L.NOISE_UNIFORM, 3, 0, 0)
    ops.fill_noise(rr, T + 1, 0, 4, N, 0, L.NOISE_UNIFORM, 3, 0, 1)
    b = _rollout(dev, inc, th32, N, T, mpl, u.view(T, N), rr)
    t = b.to_numpy()
    lanes = dict(obs=t["obs"], act=t["act"], tstep=t["tstep"])
    p_ref, _, _ = C.forward(theta, lanes, dims)
    np.testing.assert_allclose(t["mean"], np.moveaxis(p_ref, -1, 0), rtol=0, atol=2e-5)
    assert np.all(t["act"].sum(0) == 1.0)
    cum = np.cumsum(np.moveaxis(t["mean"], 0, -1), axis=-1, dtype=np.float32)
    k = np.minimum((cum < u.cpu().numpy()[:, 0][..., None]).sum(-1), 1)
    np.testing.assert_array_equal(np.argmax(t["act"], axis=0), k)
    ends = (t["flags"] & L.FLAG_END) != 0
    assert np.all(t["tstep"][0] == 0)
    if T > 1:
        np.testing.assert_array_equal(t["tstep"][1:], np.where(ends[:-1], 0, t["tstep"][:-1] + 1))
        assert np.all(t["tstep"] < mpl)
    if N * T <= 7700:    # the float64 oracle rollout from the same uniforms: same path until a near-tie in the draw
        ref = C.rollout_cartpole_v0(theta, dims, N, T, mpl, u.cpu().numpy()[:, 0].astype(np.float64),
                                    rr.cpu().numpy().astype(np.float64))
        same = np.all(ref["act"] == t["act"], axis=0).all(axis=0)
        assert same.mean() > 0.9
        np.testing.assert_allclose(t["mean"][:, :, same], ref["mean"][:, :, same], rtol=0, atol=2e-5)
    bp = _rollout(dev, inc, th32, N, T, mpl)
    bq = _rollout(dev, inc, th32, N, T, mpl)
    tp, tq = bp.to_numpy(), bq.to_numpy()
    for key in ("obs", "act", "mean", "rew", "flags", "tstep"):
        np.testing.assert_array_equal(tq[key], tp[key], err_msg=key)
    # the Philox run draws u from stream 0 row t, as fill_noise(kind uniform, stream 0) does
    np.testing.assert_array_equal(tp["act"], t["act"])


def test_get_actions_against_oracle_and_philox(dev):
    L, ops = _L(), _ops()
    dims, gd = _dims(True)
    n = 333
    rng = np.random.RandomState(4)
    theta = _theta(dims, 5, 0.3)
    th32 = torch.tensor(theta, dtype=torch.float32, device=dev)
    obs = rng.randn(4, n).astype(np.float32)
    pa = np.eye(2, dtype=np.float32)[rng.randint(0, 2, n)].T.copy()
    pa[:, :40] = 0.0                                   # rows at a path start
    h = np.tanh(rng.randn(32, n)).astype(np.float32)
    obs_d, pa_d, h_d = (torch.tensor(a, device=dev) for a in (obs, pa, h))
    u = torch.empty((1, 1, n), dtype=torch.float32, device=dev)
    ops.fill_noise(u, 1, 5, 1, n, 9, L.NOISE_UNIFORM, 11, 2, 0)
    outs = []
    for uu in (u.view(n), None):
        act = torch.empty(n, dtype=torch.int32, device=dev)
        prob = torch.empty((2, n), dtype=torch.float32, device=dev)
        h_out = torch.empty((32, n), dtype=torch.float32, device=dev)
        if uu is None:
            L.call("b200rl_categorical_gru_get_actions", L.ptr(th32), 4, 32, 2, 1, L.ptr(obs_d), L.ptr(pa_d), L.ptr(h_d),
                   n, None, 11, 2, 5, 9, L.ptr(act), L.ptr(prob), L.ptr(h_out), ops._stream())
        else:
            ops.categorical_gru_get_actions(th32, gd, obs_d, pa_d, h_d, n, uu, 0, 0, 0, 0, act, prob, h_out)
        outs.append([v.cpu().numpy() for v in (act, prob, h_out)])
    for a, b in zip(*outs):
        np.testing.assert_array_equal(a, b)
    import gru_oracle as G
    p = G.unpack(theta, dims)
    x = np.concatenate([obs.T, pa.T], axis=1).astype(np.float64)
    hn = G.cell(p, x, h.T.astype(np.float64))[0]
    np.testing.assert_allclose(outs[0][2], hn.T, rtol=0, atol=2e-6)
    pr = CO.softmax(hn @ p["W_out"] + p["b_out"])
    np.testing.assert_allclose(outs[0][1], pr.T, rtol=0, atol=1e-5)
    k = np.minimum((np.cumsum(outs[0][1].T, axis=1, dtype=np.float32) < u.cpu().numpy().reshape(n, 1)).sum(1), 1)
    np.testing.assert_array_equal(outs[0][0], k)


@pytest.mark.parametrize("inc", [True, False])
def test_loss_at_theta_old_is_exact(dev, inc):
    """The loss pass recomputes the rollout's probabilities bit for bit: mean and max KL exactly 0, ratio exactly 1."""
    ops, L = _ops(), _L()
    dims, gd = _dims(inc)
    N, T = 1000, 100
    theta = _theta(dims, 6)
    th32 = torch.tensor(theta, dtype=torch.float32, device=dev)
    b = _rollout(dev, inc, th32, N, T, 37)
    adv = np.random.RandomState(1).randn(T, N).astype(np.float32)
    b.adv.copy_(torch.tensor(adv))
    out = torch.empty(3, dtype=torch.float64, device=dev)
    ops.loss_kl(L.LOSS_TRPO, th32, gd, None, b, out)
    loss, mkl, xkl = out.cpu().numpy()
    assert mkl == 0.0 and xkl == 0.0
    np.testing.assert_allclose(loss, -adv.astype(np.float64).mean(), rtol=1e-12, atol=1e-14)
    g = torch.empty(dims.P, dtype=torch.float64, device=dev)
    tri = torch.empty(3, dtype=torch.float64, device=dev)
    ops.grad(L.LOSS_TRPO, th32, gd, None, b, g, tri)
    assert tri[1].item() == 0.0 and tri[2].item() == 0.0


def _lane_case(dev, dims, N, T, masked, seed, theta=None):
    ops, L = _ops(), _L()
    rng = np.random.RandomState(seed)
    theta = _theta(dims, seed) if theta is None else theta
    lanes = C.synthetic_lanes(dims, N, T, rng, theta, path_len=(1, min(T, 60)), masked_frac=0.3 if masked else 0.0)
    b = ops.LaneBatch(4, 2, N, T, dev)
    b.recurrent = b.categorical = True
    for k, src in (("obs", "obs"), ("act", "act"), ("mean", "old_prob")):
        getattr(b, k).copy_(torch.tensor(lanes[src]))
    b.tstep.copy_(torch.tensor(lanes["tstep"].astype(np.int16)).view(torch.uint16))
    b.adv.copy_(torch.tensor(lanes["adv"]))
    if masked:
        b.flags.copy_(torch.tensor(np.where(lanes["valid"], 0, L.FLAG_MASKED).astype(np.uint8)))
        b.count.fill_(float(lanes["valid"].sum()))
        b.masked = True
    return b, theta, lanes


def _check_passes(dev, inc, b, theta, lanes, tol, tag, f64_only_rel=1e-10):
    ops, L = _ops(), _L()
    dims, gd = _dims(inc)
    th32 = torch.tensor(theta, dtype=torch.float32, device=dev)
    th64 = torch.tensor(theta, dtype=torch.float64, device=dev)
    out = torch.empty(3, dtype=torch.float64, device=dev)
    g = torch.empty(dims.P, dtype=torch.float64, device=dev)
    errs = {}
    for kind, lk in (("trpo", L.LOSS_TRPO), ("vpg", L.LOSS_VPG)):
        ref = np.array(C.loss_kl(theta, lanes, dims, kind))
        ops.loss_kl(lk, th32, gd, None, b, out)
        # atol: the float32 KL near 0 is a difference of two logs of nearly equal probabilities, ~1e-7 absolute
        np.testing.assert_allclose(out.cpu().numpy(), ref, rtol=1e-5, atol=5e-7)
        ops.update_f64(0, lk, th64, gd, None, b, None, 0.0, 0.0, None, out)
        np.testing.assert_allclose(out.cpu().numpy(), ref, rtol=1e-10, atol=1e-13)
        for pen in (0.0, 0.5):
            gref = C.grad(theta, lanes, dims, kind, penalty=pen)
            if pen:
                ops.grad_penalized(lk, pen, th32, gd, None, b, g, out)
            else:
                ops.grad(lk, th32, gd, None, b, g, out)
            assert np.all(np.isfinite(g.cpu().numpy()))
            errs["grad_%s_%g" % (kind, pen)] = _rel(g.cpu().numpy(), gref)
        gref = C.grad(theta, lanes, dims, kind)
        ops.update_f64(1, lk, th64, gd, None, b, None, 0.0, 0.0, g, out)
        np.testing.assert_allclose(g.cpu().numpy(), gref, rtol=0, atol=f64_only_rel * np.abs(gref).max())
    th_kl = theta + 1e-3 * np.random.RandomState(7).randn(dims.P)
    gk = C.grad(th_kl, lanes, dims, "kl")
    ops.update_f64(1, L.LOSS_KL, torch.tensor(th_kl, device=dev), gd, None, b, None, 0.0, 0.0, g, None)
    np.testing.assert_allclose(g.cpu().numpy(), gk, rtol=0, atol=f64_only_rel * np.abs(gk).max())
    # Fisher product at theta_old: old_prob = the policy's own float32 probabilities
    p32 = np.moveaxis(C.forward(theta, lanes, dims)[0], -1, 0).astype(np.float32)
    b.mean.copy_(torch.tensor(p32))
    lanes = dict(lanes, old_prob=p32)
    x = torch.tensor(np.random.RandomState(3).randn(dims.P), dtype=torch.float64, device=dev)
    ref = C.fvp(theta, lanes, dims, x.cpu().numpy(), 1e-5)
    hx = torch.empty_like(x)
    ops.fvp(th32, gd, None, b, x, 1e-5, 1.0, hx)
    errs["fvp"] = _rel(hx.cpu().numpy(), ref)
    hc = b.hcache(32, 0)
    ops.grad(L.LOSS_TRPO, th32, gd, None, b, g, out, hc)
    hx2 = torch.empty_like(x)
    ops.fvp(th32, gd, None, b, x, 1e-5, 1.0, hx2, hc)
    np.testing.assert_array_equal(hx2.cpu().numpy(), hx.cpu().numpy())
    ops.update_f64(2, L.LOSS_TRPO, th64, gd, None, b, x, 1e-5, 1.0, hx, None)
    np.testing.assert_allclose(hx.cpu().numpy(), ref, rtol=0, atol=f64_only_rel * np.abs(ref).max())
    print("categorical GRU float32 error %s: %s" % (tag, " ".join("%s=%.2e" % kv for kv in sorted(errs.items()))))
    assert max(errs.values()) < tol, errs


# 20000 lanes are 157 tiles of 128: more than one tile per CTA of the gradient pass on 132 SMs
@pytest.mark.parametrize("T,N", [(1, 37 * 128), (16, 300), (100, 77), (200, 19), (16, 20000)])
@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("inc", [True, False])
def test_passes_match_oracle(dev, T, N, masked, inc):
    dims, _ = _dims(inc)
    b, theta, lanes = _lane_case(dev, dims, N, T, masked, 10 + T + int(masked))
    _check_passes(dev, inc, b, theta, lanes, F32_TOL[T], "T=%d N=%d masked=%s inc=%s" % (T, N, masked, inc))


@pytest.mark.parametrize("gap", [8.0, 17.0, 40.0])
@pytest.mark.parametrize("sign", [1.0, -1.0])
def test_saturated_softmax(dev, gap, sign):
    """Probabilities within ~1e-7 of 0 or 1 (logit gaps 17 and 40) give finite passes that agree with the oracle: the
    output bias sets the gap, and W_out is scaled so that h moves it by at most 0.25."""
    inc = True
    dims, _ = _dims(inc)
    rng = np.random.RandomState(int(gap))
    theta = C.init_params(dims, rng) + 0.05 * rng.randn(dims.P)
    nW = 32 * 2
    Wo = theta[-nW - 2:-2].reshape(32, 2)
    Wo *= 0.25 / np.abs(Wo[:, 0] - Wo[:, 1]).sum()
    theta[-nW - 2:-2] = Wo.reshape(-1)
    theta[-2:] = sign * 0.5 * gap * np.array([1.0, -1.0])
    theta = _f32(theta)
    b, theta, lanes = _lane_case(dev, dims, 300, 16, True, 3, theta)
    _check_passes(dev, inc, b, theta, lanes, 1e-4, "gap=%g sign=%g" % (gap, sign), f64_only_rel=1e-9)


def test_gradient_pass_ignores_stale_cache(dev):
    ops, L = _ops(), _L()
    dims, gd = _dims(True)
    b, theta, lanes = _lane_case(dev, dims, 77, 100, False, 5)
    th32 = torch.tensor(theta, dtype=torch.float32, device=dev)
    x = torch.tensor(np.random.RandomState(2).randn(dims.P), dtype=torch.float64, device=dev)
    res = []
    for fill in (float("nan"), 0.0):
        hc = b.hcache(32, 0)
        g = torch.empty(dims.P, dtype=torch.float64, device=dev)
        hx = torch.empty_like(x)
        hc.fill_(fill)
        ops.grad(L.LOSS_TRPO, th32, gd, None, b, g, None, hc)
        hc.fill_(fill)
        ops.fvp(th32, gd, None, b, x, 1e-5, 1.0, hx)
        res.append((g.cpu().numpy(), hx.cpu().numpy()))
    for a in res[0]:
        assert np.all(np.isfinite(a))
    np.testing.assert_array_equal(res[0][0], res[1][0])
    np.testing.assert_array_equal(res[0][1], res[1][1])


def _algo(algo_name, n_envs=40, T=100, n_itr=3, inc=True, **kw):
    from rllab_b200.algos.erwr import ERWR
    from rllab_b200.algos.ppo import PPO
    from rllab_b200.algos.trpo import TRPO
    from rllab_b200.algos.vpg import VPG
    from rllab_b200.baselines.linear_feature_baseline import LinearFeatureBaseline
    from rllab_b200.envs.gym_env import GymEnv
    from rllab_b200.envs.normalized_env import normalize
    from rllab_b200.policies.categorical_gru_policy import CategoricalGRUPolicy
    env = normalize(GymEnv("CartPole-v0"))
    policy = CategoricalGRUPolicy(env_spec=env.spec, state_include_action=inc, seed=3)
    args = dict(env=env, policy=policy, baseline=LinearFeatureBaseline(env_spec=env.spec), batch_size=n_envs * T,
                max_path_length=T, n_itr=n_itr, discount=0.99, sampler_args=dict(n_envs=n_envs, seed=7))
    args.update(kw)
    return dict(trpo=TRPO, vpg=VPG, ppo=PPO, erwr=ERWR)[algo_name](**args)


def _oracle_lanes(sd):
    b = sd.lane_batch
    t = b.to_numpy()
    return dict(obs=t["obs"], act=t["act"], tstep=t["tstep"], adv=b.adv.cpu().numpy(), old_prob=t["mean"],
                mean=t["mean"], valid=b.valid_mask())


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
    theta_ref, info = C.trpo_step(theta0, lanes, C.CatGruDims(4, 32, 2, True), 0.01, 4)
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
    theta_ref, info = C.trpo_step(theta0, lanes, C.CatGruDims(4, 32, 2, True), 0.01, 4)
    li = algo.optimizer.last_info
    assert not li["rejected"] and 0 < li["constraint_val"] <= 0.01
    d = algo.policy.get_param_values() - theta0
    assert _rel(d, theta_ref - theta0) < 2e-2, _rel(d, theta_ref - theta0)


@pytest.mark.parametrize("name", ["vpg", "ppo", "erwr"])
@pytest.mark.parametrize("inc", [True, False])
def test_first_order_and_penalty_algos_run(dev, name, inc):
    algo = _algo(name, n_itr=2, inc=inc)
    theta0 = algo.policy.get_param_values()
    algo.train()
    theta1 = algo.policy.get_param_values()
    assert np.all(np.isfinite(theta1)) and np.abs(theta1 - theta0).max() > 0


def test_cem_reps_and_subsample_are_rejected(dev):
    from rllab_b200.algos.cem import CEM
    from rllab_b200.algos.reps import REPS
    algo = _algo("trpo", optimizer_args=dict(subsample_factor=0.5))
    algo.start_worker()
    algo.init_opt()
    sd = algo.sampler.process_samples(0, algo.sampler.obtain_samples(0))
    with pytest.raises(NotImplementedError):
        algo.optimize_policy(0, sd)
    with pytest.raises(NotImplementedError):
        CEM(env=algo.env, policy=algo.policy, n_itr=1, max_path_length=10, batch_size=10)
    reps = REPS(env=algo.env, policy=algo.policy, baseline=algo.baseline, batch_size=1000, max_path_length=100, n_itr=1,
                sampler_args=dict(n_envs=10, seed=7))
    with pytest.raises(NotImplementedError):
        reps.init_opt()


def test_recurrent_wire_format(dev):
    algo = _algo("trpo", n_envs=12, T=100)
    algo.start_worker()
    algo.init_opt()
    sd = algo.sampler.process_samples(0, algo.sampler.obtain_samples(0))
    paths = sd["paths"]
    for p in paths:
        np.testing.assert_array_equal(p["agent_infos"]["prev_action"][0], 0.0)
        np.testing.assert_array_equal(p["agent_infos"]["prev_action"][1:], p["actions"][:-1])
        assert np.all(p["actions"].sum(1) == 1.0) and "prob" in p["agent_infos"] and "mean" not in p["agent_infos"]
    n, Lmax = len(paths), max(len(p["rewards"]) for p in paths)
    assert sd["valids"].shape == (n, Lmax)
    np.testing.assert_array_equal(sd["valids"].sum(1), [len(p["rewards"]) for p in paths])
    assert sd["observations"].shape == (n, Lmax, 4) and sd["actions"].shape == (n, Lmax, 2)
    assert sd["agent_infos"]["prev_action"].shape == (n, Lmax, 2) and sd["agent_infos"]["prob"].shape == (n, Lmax, 2)
    np.testing.assert_array_equal(sd["agent_infos"]["prob"][sd["valids"] == 0], 0.0)
    # Entropy: the mean over valid samples of entropy(prob), the reference's recurrent branch
    ent = algo.sampler.stats["Entropy"]
    v = sd["valids"] == 1
    ref = CO.entropy(sd["agent_infos"]["prob"][v]).mean()
    np.testing.assert_allclose(ent, ref, rtol=1e-6)
    np.testing.assert_allclose(ent, C.entropy_mean(_oracle_lanes(sd)), rtol=1e-6)
    # the policy's own step API reproduces the recorded probabilities of a path (prev_action fed back, h carried)
    pol = algo.policy
    p = paths[0]
    pol.reset()
    for t in range(len(p["rewards"])):
        _, info = pol.get_action(p["observations"][t])
        np.testing.assert_allclose(info["prob"], p["agent_infos"]["prob"][t], rtol=0, atol=1e-5)
        np.testing.assert_array_equal(info["prev_action"], p["agent_infos"]["prev_action"][t])
        pol._prev_actions[0] = p["actions"][t]                  # continue with the recorded action


def test_pickle_round_trip(dev):
    import pickle
    algo = _algo("trpo", n_envs=4, T=10)
    pol = algo.policy
    pol.set_param_values(pol.get_param_values() + 0.01)
    pol2 = pickle.loads(pickle.dumps(pol))
    np.testing.assert_array_equal(pol2.get_param_values(), pol.get_param_values())
    assert pol2.state_include_action == pol.state_include_action and pol2.n_params == pol.n_params


def test_fvp_past_the_workspace_plane(dev):
    """A batch whose M J x plane (2 floats per sample) is larger than the shared workspace could hold (over 4.85M
    samples): the plane comes from the batch, and the product is finite and positive along x."""
    ops, L = _ops(), _L()
    dims, gd = _dims(True)
    N, T = 24832, 200                                   # 4 966 400 samples
    theta = _theta(dims, 4)
    th32 = torch.tensor(theta, dtype=torch.float32, device=dev)
    b = _rollout(dev, True, th32, N, T, 200)
    x = torch.tensor(np.random.RandomState(5).randn(dims.P), dtype=torch.float64, device=dev)
    hx = torch.empty_like(x)
    ops.fvp(th32, gd, None, b, x, 0.0, 1.0, hx)
    h = hx.cpu().numpy()
    assert np.all(np.isfinite(h)) and float(h @ x.cpu().numpy()) > 0


CURVE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "oracle_cartpole_v0_gru_trpo_curve.json")


def test_example_learns(dev):
    """TRPO, CategoricalGRUPolicy, LinearFeatureBaseline, batch 4000, path length 200, step size 0.01 on
    normalize(GymEnv("CartPole-v0")), against the band of the float64 oracle's curves over five seeds
    (tests/golden/make_cartpole_v0_gru_curve.py; the RNG streams differ, so bands, not values), with the rule of
    test_gpu_gru.py: at iteration 0 at most the band's top plus its width; over the last 5 iterations a mean of at least
    the lowest seed's mean less its spread."""
    import json
    from rllab_b200.algos.trpo import TRPO
    from rllab_b200.baselines.linear_feature_baseline import LinearFeatureBaseline
    from rllab_b200.envs.gym_env import GymEnv
    from rllab_b200.envs.normalized_env import normalize
    from rllab_b200.misc import logger
    from rllab_b200.policies.categorical_gru_policy import CategoricalGRUPolicy
    curves = np.array(list(json.load(open(CURVE))["AverageReturn"].values()))
    n_itr = curves.shape[1]
    first_hi = curves[:, 0].max() + (curves[:, 0].max() - curves[:, 0].min())
    late = curves[:, -5:].mean(axis=1)
    late_lo = late.min() - (late.max() - late.min())
    np.random.seed(1)
    env = normalize(GymEnv("CartPole-v0"))
    policy = CategoricalGRUPolicy(env_spec=env.spec)
    algo = TRPO(env=env, policy=policy, baseline=LinearFeatureBaseline(env_spec=env.spec), batch_size=4000,
                max_path_length=200, n_itr=n_itr, discount=0.99, step_size=0.01)
    algo.start_worker()
    algo.init_opt()
    rets = []
    for itr in range(n_itr):
        algo.train_itr(itr)
        rets.append(logger.get_last_table()["AverageReturn"])
    print("categorical GRU CartPole-v0 TRPO AverageReturn per iteration:", [round(r, 1) for r in rets], "bounds",
          first_hi, late_lo)
    assert rets[0] <= first_hi, (rets[0], first_hi)
    assert np.mean(rets[-5:]) >= late_lo, (rets, late_lo)
