"""GPU: the discrete-action path -- gym CartPole-v0 lanes, the categorical rollout and get_actions, the categorical
loss/KL, gradient and Fisher-vector passes against the float64 oracle (tests/categorical_oracle.py) at the batch sizes
of test_gpu_update_shapes.py, and TRPO / VPG / PPO / ERWR / REPS with CategoricalMLPPolicy through the host API."""
import os

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import categorical_oracle as C          # noqa: E402

DIMS = C.CatDims(4, (32, 32), 2)
TILE = 128
SIZES = ["1", "77", "exact", "large"]


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from rllab_b200 import _lib
    _lib.load()
    from rllab_b200.misc import logger
    logger.set_quiet(True)
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def n_sm(dev):
    return torch.cuda.get_device_properties(dev).multi_processor_count


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


def test_env_reset_and_step_match_oracle(dev):
    L, ops = _L(), _ops()
    N = 300
    rng = np.random.RandomState(1)
    raw = rng.rand(4, N).astype(np.float32)
    state = torch.empty((4, N), dtype=torch.float32, device=dev)
    obs = torch.empty_like(state)
    ops.env_reset(L.ENV_GYM_CARTPOLE, N, state, obs, torch.tensor(raw, device=dev))
    env = C.CartPoleV0(np.float32)
    s = env.reset(raw)
    np.testing.assert_allclose(state.cpu().numpy(), s, rtol=0, atol=1e-7)
    acts = rng.randint(0, 2, N)
    rew = torch.empty(N, dtype=torch.float32, device=dev)
    done = torch.empty(N, dtype=torch.uint8, device=dev)
    for _ in range(30):
        s0 = state.cpu().numpy().astype(np.float64)
        ops.env_step(L.ENV_GYM_CARTPOLE, N, state, torch.tensor(acts[None].astype(np.float32), device=dev), obs, rew,
                     done, normalized=True)       # an index passes NormalizedEnv unscaled
        ns, r, d = C.CartPoleV0().step(s0, acts)
        np.testing.assert_allclose(state.cpu().numpy(), ns, rtol=1e-5, atol=1e-6)
        np.testing.assert_array_equal(rew.cpu().numpy(), r)
        clear = np.all(np.abs(np.abs(ns[[0, 2]]) - [[2.4], [C.CartPoleV0.THR]]) > 1e-5, axis=0)
        np.testing.assert_array_equal(done.cpu().numpy().astype(bool)[clear], d[clear])
        acts = rng.randint(0, 2, N)


def _rollout(dev, theta32, N, T, mpl, u=None, rr=None, seed=3, it=0):
    ops = _ops()
    b = ops.LaneBatch(4, 2, N, T, dev)
    b.categorical = True
    ops.rollout(_L().ENV_GYM_CARTPOLE, theta32, 32, 32, None, b, mpl, u, rr, seed, it)
    return b


def test_rollout_per_step_against_oracle(dev):
    L, ops = _L(), _ops()
    N, T, mpl = 500, 120, 60
    theta = C.init_params(DIMS, np.random.RandomState(2))
    th32 = torch.tensor(theta, dtype=torch.float32, device=dev)
    theta = _f32(theta)
    u = torch.empty((T, 1, N), dtype=torch.float32, device=dev)
    rr = torch.empty((T + 1, 4, N), dtype=torch.float32, device=dev)
    ops.fill_noise(u, T, 0, 1, N, 0, L.NOISE_UNIFORM, 3, 0, 0)
    ops.fill_noise(rr, T + 1, 0, 4, N, 0, L.NOISE_UNIFORM, 3, 0, 1)
    b = _rollout(dev, th32, N, T, mpl, u.view(T, N), rr)
    t = b.to_numpy()
    un, rrn = u.cpu().numpy()[:, 0], rr.cpu().numpy()
    obs, act, prob = t["obs"], t["act"], t["mean"]
    # prob = softmax of the recorded obs
    p_ref = C.prob(theta, obs.reshape(4, -1).T, DIMS)
    np.testing.assert_allclose(prob.reshape(2, -1).T, p_ref, rtol=2e-5, atol=2e-6)
    # action = weighted_sample(recorded prob, u), except at a tie within 1e-6
    pr = prob.reshape(2, -1).T.astype(np.float64)
    k_ref = C.weighted_sample_n(pr, un.reshape(-1))
    k_dev = act.reshape(2, -1).T.argmax(axis=1)
    assert np.all(act.sum(axis=0) == 1) and set(np.unique(act)) <= {0.0, 1.0}
    tie = np.abs(np.cumsum(pr, axis=1)[:, 0] - un.reshape(-1)) < 1e-6
    assert np.all((k_dev == k_ref) | tie)
    # dynamics and bookkeeping, step by step from the recorded obs
    env = C.CartPoleV0()
    flags, tstep = t["flags"], t["tstep"]
    plen = np.zeros(N, dtype=int)
    for s in range(T):
        ns, r, d = env.step(obs[:, s].astype(np.float64), k_dev.reshape(T, N)[s])
        np.testing.assert_array_equal(t["rew"][s], 1.0)
        np.testing.assert_array_equal(tstep[s], plen)
        done = (flags[s] & L.FLAG_DONE) != 0
        end = (flags[s] & L.FLAG_END) != 0
        clear = np.all(np.abs(np.abs(ns[[0, 2]]) - [[2.4], [C.CartPoleV0.THR]]) > 1e-4, axis=0)
        np.testing.assert_array_equal(done[clear], d[clear])
        assert np.all(end == (done | (plen + 1 >= mpl) | (s == T - 1)))
        assert np.all(((flags[s] & L.FLAG_CUT) != 0) == (end & ~done & (plen + 1 < mpl)))
        if s + 1 < T:
            cont = ~end
            np.testing.assert_allclose(obs[:, s + 1][:, cont], ns[:, cont], rtol=1e-4, atol=1e-5)
            np.testing.assert_allclose(obs[:, s + 1][:, end], env.reset(rrn[s + 1])[:, end].astype(np.float32),
                                       rtol=0, atol=1e-7)
        plen = np.where(end, 0, plen + 1)
    # the in-kernel Philox draw is the injected stream
    bp = _rollout(dev, th32, N, T, mpl)
    tp = bp.to_numpy()
    for k in ("obs", "act", "mean", "rew", "flags", "tstep"):
        np.testing.assert_array_equal(tp[k], t[k], err_msg=k)


def test_get_actions_matches_oracle_and_philox(dev):
    L, ops = _L(), _ops()
    n = 333
    rng = np.random.RandomState(4)
    theta = C.init_params(DIMS, rng) + 0.3 * rng.randn(DIMS.P)
    th32 = torch.tensor(theta, dtype=torch.float32, device=dev)
    obs = rng.randn(4, n).astype(np.float32)
    ot = torch.tensor(obs, device=dev)
    u = torch.empty((1, 1, n), dtype=torch.float32, device=dev)
    ops.fill_noise(u, 1, 5, 1, n, 9, L.NOISE_UNIFORM, 11, 2, 0)
    outs = []
    for uu in (u.view(n), None):
        act = torch.empty(n, dtype=torch.int32, device=dev)
        prob = torch.empty((2, n), dtype=torch.float32, device=dev)
        if uu is None:
            L.call("b200rl_categorical_get_actions", L.ptr(th32), 4, 32, 32, 2, L.ptr(ot), n, None, 11, 2, 5, 9,
                   L.ptr(act), L.ptr(prob), ops._stream())
        else:
            ops.categorical_get_actions(th32, (4, 32, 32, 2), ot, n, uu, 0, 0, 0, 0, act, prob)
        outs.append((act.cpu().numpy(), prob.cpu().numpy()))
    np.testing.assert_array_equal(outs[0][0], outs[1][0])
    np.testing.assert_array_equal(outs[0][1], outs[1][1])
    p_ref = C.prob(_f32(theta), obs.T.astype(np.float64), DIMS)
    np.testing.assert_allclose(outs[0][1].T, p_ref, rtol=2e-5, atol=2e-6)
    un = u.cpu().numpy().reshape(-1)
    pr = outs[0][1].T.astype(np.float64)
    tie = np.abs(pr[:, 0] - un) < 1e-6
    assert np.all((outs[0][0] == C.weighted_sample_n(pr, un)) | tie)


def _batch_size(size, n_sm):
    return {"1": 1, "77": 77, "exact": TILE * 37, "large": (17 * n_sm + 5) * TILE - 51}[size]


def _pass_case(dev, n_sm, size, masked):
    """A synthetic batch of B samples (lanes N = B, T = 1) recorded at theta_old, with the oracle's view of it."""
    ops = _ops()
    B = _batch_size(size, n_sm)
    rng = np.random.RandomState(B + (7 if masked else 0))
    theta_old = _f32(C.init_params(DIMS, rng) + 0.2 * rng.randn(DIMS.P))
    obs = (rng.randn(4, B) * [[1.0], [1.5], [0.2], [1.5]]).astype(np.float32)
    b = ops.LaneBatch(4, 2, B, 1, dev)
    b.categorical = True
    b.obs.copy_(torch.tensor(obs.reshape(4, 1, B)))
    th32 = torch.tensor(theta_old, dtype=torch.float32, device=dev)
    u = torch.tensor(rng.rand(B).astype(np.float32), device=dev)
    act = torch.empty(B, dtype=torch.int32, device=dev)
    prob = torch.empty((2, B), dtype=torch.float32, device=dev)
    ops.categorical_get_actions(th32, (4, 32, 32, 2), b.obs.view(4, B), B, u, 0, 0, 0, 0, act, prob)
    b.mean.copy_(prob.view(2, 1, B))
    b.act.copy_(torch.nn.functional.one_hot(act.long(), 2).t().float().view(2, 1, B))
    b.adv.copy_(torch.tensor(rng.randn(1, B).astype(np.float32)))
    keep = np.ones(B, dtype=bool)
    if masked:
        keep = rng.rand(B) > 0.3
        keep[0] = True
        b.flags.copy_(torch.tensor(np.where(keep, 0, _L().FLAG_MASKED).astype(np.uint8).reshape(1, B)))
        b.count.fill_(float(keep.sum()))
        b.masked = True
    batch = dict(obs=obs.T.astype(np.float64)[keep], actions=b.act.view(2, B).t().double().cpu().numpy()[keep],
                 adv=b.adv.view(B).double().cpu().numpy()[keep], old_prob=prob.t().double().cpu().numpy()[keep])
    return b, theta_old, batch


@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("size", SIZES)
def test_passes_match_oracle(dev, n_sm, size, masked):
    L, ops = _L(), _ops()
    b, theta_old, batch = _pass_case(dev, n_sm, size, masked)
    dims = ops.CategoricalDims(4, 32, 32, 2)
    P = DIMS.P
    out = torch.zeros(3, dtype=torch.float64, device=dev)
    th_old32 = torch.tensor(theta_old, dtype=torch.float32, device=dev)
    # at theta_old: every ratio is exactly 1 and every KL exactly 0
    ops.loss_kl(L.LOSS_TRPO, th_old32, dims, None, b, out)
    adv_mean = float(np.sum(batch["adv"]) / len(batch["adv"]))
    o = out.cpu().numpy()
    assert o[1] == 0.0 and o[2] == 0.0
    np.testing.assert_allclose(o[0], -adv_mean, rtol=1e-12, atol=1e-15)
    # off theta_old
    rng = np.random.RandomState(11)
    theta = _f32(theta_old + 0.05 * rng.randn(P))
    th32 = torch.tensor(theta, dtype=torch.float32, device=dev)
    hc = b.hcache(32, 32)
    for kind, lk in (("trpo", L.LOSS_TRPO), ("vpg", L.LOSS_VPG)):
        ops.loss_kl(lk, th32, dims, None, b, out)
        o = out.cpu().numpy()
        np.testing.assert_allclose(o[0], C.surr_loss(theta, batch, DIMS, kind), rtol=2e-5, atol=1e-7)
        mkl, xkl = C.kl_stats(theta, batch, DIMS)
        np.testing.assert_allclose(o[1:], [mkl, xkl], rtol=2e-3, atol=1e-8)
        for pen in (0.0, 2.5):
            g = torch.zeros(P, dtype=torch.float64, device=dev)
            tri = torch.zeros(3, dtype=torch.float64, device=dev)
            if pen:
                ops.grad_penalized(lk, pen, th32, dims, None, b, g, tri)
            else:
                ops.grad(lk, th32, dims, None, b, g, tri, hc)
            g_ref = C.grad_surr(theta, batch, DIMS, kind, pen)
            gd = g.cpu().numpy()
            np.testing.assert_allclose(gd, g_ref, rtol=1e-3, atol=2e-5 * np.abs(g_ref).max() + 1e-12)
            # the loss pass's triple: per-sample terms are bit-identical, the float64 block sums run in another order
            np.testing.assert_allclose(tri.cpu().numpy(), out.cpu().numpy(), rtol=1e-12, atol=1e-18)
            g2 = torch.zeros_like(g)
            (ops.grad_penalized(lk, pen, th32, dims, None, b, g2) if pen else ops.grad(lk, th32, dims, None, b, g2))
            assert torch.equal(g, g2)                                                  # bit-identical rerun
    # Fisher-vector product at theta_old: recomputed, from the activation cache of a gradient pass, and on a tile list
    x = rng.randn(P)
    xt = torch.tensor(x, device=dev)
    g = torch.zeros(P, dtype=torch.float64, device=dev)
    ops.grad(L.LOSS_TRPO, th_old32, dims, None, b, g, None, hc)
    ref = C.fvp(theta_old, batch, _f32(x), DIMS, 1e-5)
    res = []
    for cache in (None, hc):
        Hx = torch.zeros(P, dtype=torch.float64, device=dev)
        ops.fvp(th_old32, dims, None, b, xt, 1e-5, 1.0, Hx, cache)
        res.append(Hx.cpu().numpy())
        np.testing.assert_allclose(res[-1], ref, rtol=1e-3, atol=2e-5 * np.abs(ref).max())
    np.testing.assert_allclose(res[0], res[1], rtol=1e-5, atol=1e-7 * np.abs(ref).max())
    n_tiles = -(-b.B // TILE)
    tiles_np = np.arange(0, n_tiles, 2).astype(np.int32)
    tiles = torch.tensor(tiles_np, device=dev)
    cnt = torch.zeros(1, dtype=torch.float64, device=dev)
    ops.count_valid(b, tiles, cnt)
    Hx = torch.zeros(P, dtype=torch.float64, device=dev)
    ops.fvp(th_old32, dims, None, b, xt, 1e-5, 1.0, Hx, hc, tiles, cnt)
    in_tiles = np.zeros(b.B, dtype=bool)
    for ti in tiles_np:
        in_tiles[ti * TILE:(ti + 1) * TILE] = True
    keep = b.valid_mask().reshape(-1)
    sub = {k: v[in_tiles[keep]] for k, v in batch.items()}
    ref_sub = C.fvp(theta_old, sub, _f32(x), DIMS, 1e-5)
    assert cnt.item() == len(sub["adv"])
    np.testing.assert_allclose(Hx.cpu().numpy(), ref_sub, rtol=1e-3, atol=2e-5 * np.abs(ref_sub).max())
    # float64 parity mode (<= 1e-10 relative): loss/KL and gradients off theta_old, the KL gradient of
    # FiniteDifferenceHvp, and the exact Fisher product at theta_old
    th64 = torch.tensor(theta, dtype=torch.float64, device=dev)
    th_old64 = torch.tensor(theta_old, dtype=torch.float64, device=dev)
    v = torch.zeros(P, dtype=torch.float64, device=dev)
    for kind, lk in (("trpo", L.LOSS_TRPO), ("vpg", L.LOSS_VPG)):
        ops.update_f64(0, lk, th64, dims, None, b, None, 0.0, 0.0, None, out)
        o = out.cpu().numpy()
        np.testing.assert_allclose(o[0], C.surr_loss(theta, batch, DIMS, kind), rtol=1e-10, atol=1e-15)
        np.testing.assert_allclose(o[1:], C.kl_stats(theta, batch, DIMS), rtol=1e-10, atol=1e-18)
        ops.update_f64(1, lk, th64, dims, None, b, None, 0.0, 0.0, v, out)
        ref = C.grad_surr(theta, batch, DIMS, kind)
        np.testing.assert_allclose(v.cpu().numpy(), ref, rtol=0, atol=1e-10 * np.abs(ref).max())
    ops.update_f64(1, L.LOSS_KL, th64, dims, None, b, None, 0.0, 0.0, v, None)
    ref = C.grad_surr(theta, batch, DIMS, "vpg", 1.0) - C.grad_surr(theta, batch, DIMS, "vpg", 0.0)
    np.testing.assert_allclose(v.cpu().numpy(), ref, rtol=0, atol=1e-10 * np.abs(ref).max())
    ops.update_f64(2, L.LOSS_TRPO, th_old64, dims, None, b, xt, 1e-5, 1.0, v, None)
    ref = C.fvp(theta_old, batch, x, DIMS, 1e-5)
    np.testing.assert_allclose(v.cpu().numpy(), ref, rtol=0, atol=1e-10 * np.abs(ref).max())


def _algo(algo_name, n_envs=1000, T=200, n_itr=3, **kw):
    from rllab_b200.algos.erwr import ERWR
    from rllab_b200.algos.ppo import PPO
    from rllab_b200.algos.reps import REPS
    from rllab_b200.algos.trpo import TRPO
    from rllab_b200.algos.vpg import VPG
    from rllab_b200.baselines.linear_feature_baseline import LinearFeatureBaseline
    from rllab_b200.envs.gym_env import GymEnv
    from rllab_b200.envs.normalized_env import normalize
    from rllab_b200.policies.categorical_mlp_policy import CategoricalMLPPolicy
    env = normalize(GymEnv("CartPole-v0"))
    policy = CategoricalMLPPolicy(env_spec=env.spec, hidden_sizes=(32, 32), seed=3)
    args = dict(env=env, policy=policy, baseline=LinearFeatureBaseline(env_spec=env.spec), batch_size=(n_envs or 1) * T,
                max_path_length=T, n_itr=n_itr, discount=0.99, sampler_args=dict(n_envs=n_envs, seed=7))
    args.update(kw)
    return dict(trpo=TRPO, vpg=VPG, ppo=PPO, erwr=ERWR, reps=REPS)[algo_name](**args)


@pytest.mark.parametrize("cg_iters", [1, 4])
def test_trpo_step_matches_oracle(dev, cg_iters):
    algo = _algo("trpo", 512, 50, optimizer_args=dict(cg_iters=cg_iters))
    algo.start_worker()
    algo.init_opt()
    paths = algo.sampler.obtain_samples(0)
    sd = algo.sampler.process_samples(0, paths)
    b = sd.lane_batch
    keep = b.valid_mask().reshape(-1)
    t = b.to_numpy()
    batch = dict(obs=t["obs"].reshape(4, -1).T.astype(np.float64)[keep],
                 actions=t["act"].reshape(2, -1).T.astype(np.float64)[keep],
                 adv=b.adv.cpu().numpy().reshape(-1).astype(np.float64)[keep],
                 old_prob=t["mean"].reshape(2, -1).T.astype(np.float64)[keep])
    theta0 = algo.policy.theta32.double().cpu().numpy()
    algo.optimize_policy(0, sd)
    theta_dev = algo.policy.get_param_values()
    theta_ref, info = C.trpo_step(theta0, batch, DIMS, 0.01, cg_iters)
    li = algo.optimizer.last_info
    assert li["n_iter"] == info["n_iter"] and li["rejected"] == info["rejected"] and not info["rejected"]
    assert _rel(theta_dev - theta0, theta_ref - theta0) < 1e-3, _rel(theta_dev - theta0, theta_ref - theta0)
    assert _rel(theta_dev, theta_ref) < 1e-5
    np.testing.assert_allclose(li["constraint_val"], info["constraint_val"], rtol=2e-3)
    assert 0 < li["constraint_val"] <= 0.01


def _oracle_batch(sd):
    b = sd.lane_batch
    keep = b.valid_mask().reshape(-1)
    t = b.to_numpy()
    return dict(obs=t["obs"].reshape(4, -1).T.astype(np.float64)[keep],
                actions=t["act"].reshape(2, -1).T.astype(np.float64)[keep],
                adv=b.adv.cpu().numpy().reshape(-1).astype(np.float64)[keep],
                old_prob=t["mean"].reshape(2, -1).T.astype(np.float64)[keep])


@pytest.mark.parametrize("cg_iters,tol", [(6, 1e-5), (10, 5e-3)])
def test_trpo_f64_mode_matches_oracle(dev, cg_iters, tol):
    """precision="f64": the whole TRPO step against the float64 oracle on the same batch, with the tolerances of
    test_gpu_algos.py's Gaussian case (at 10 CG iterations the oracle's own self-sensitivity sets the bound)."""
    algo = _algo("trpo", 512, 50, optimizer_args=dict(cg_iters=cg_iters, precision="f64"))
    algo.start_worker()
    algo.init_opt()
    sd = algo.sampler.process_samples(0, algo.sampler.obtain_samples(0))
    batch = _oracle_batch(sd)
    theta0 = algo.policy.get_param_values()
    algo.optimize_policy(0, sd)
    theta_dev = algo.policy.get_param_values()
    theta_ref, info = C.trpo_step(theta0, batch, DIMS, 0.01, cg_iters)
    li = algo.optimizer.last_info
    assert li["n_iter"] == info["n_iter"] and li["rejected"] == info["rejected"] and not info["rejected"]
    assert _rel(theta_dev, theta_ref) < tol, _rel(theta_dev, theta_ref)
    np.testing.assert_allclose(li["constraint_val"], info["constraint_val"], rtol=100 * tol)


def test_trpo_finite_difference_hvp(dev):
    """FiniteDifferenceHvp: the Hessian-vector product from two float64 KL-gradient passes; the step it takes agrees
    with the oracle's exact-product step to the accuracy of the finite difference."""
    from rllab_b200.optimizers.conjugate_gradient_optimizer import ConjugateGradientOptimizer, FiniteDifferenceHvp
    opt = ConjugateGradientOptimizer(cg_iters=4, hvp_approach=FiniteDifferenceHvp())
    algo = _algo("trpo", 512, 50, optimizer=opt)
    algo.start_worker()
    algo.init_opt()
    sd = algo.sampler.process_samples(0, algo.sampler.obtain_samples(0))
    batch = _oracle_batch(sd)
    theta0 = algo.policy.get_param_values()
    algo.optimize_policy(0, sd)
    theta_dev = algo.policy.get_param_values()
    theta_ref, info = C.trpo_step(theta0, batch, DIMS, 0.01, 4)
    li = algo.optimizer.last_info
    assert not li["rejected"] and not info["rejected"] and 0 < li["constraint_val"] <= 0.01
    assert _rel(theta_dev - theta0, theta_ref - theta0) < 1e-2, _rel(theta_dev - theta0, theta_ref - theta0)


def test_reps_l2_reg_loss_regularizes_the_weight_matrices(dev):
    """REPS's L2_reg_loss term over CategoricalMLPPolicy: W0, W1 and Wout (lasagne's regularizable parameters; the
    DenseLayer biases are not), divided by 3."""
    from rllab_b200.algos.reps import regularizable_slices
    algo = _algo("reps", 64, 50, n_itr=1, L2_reg_loss=1e-2)
    sl = regularizable_slices(algo.policy)
    P = DIMS.P
    assert [(x.start, x.stop) for x in sl] == [(0, 128), (160, 160 + 1024), (1216, 1280)] and P == 1282
    algo.train()
    assert np.all(np.isfinite(algo.policy.get_param_values()))


def test_entropy_and_samples_data_wire_format(dev):
    algo = _algo("trpo", 256, 100, n_itr=1)
    algo.start_worker()
    algo.init_opt()
    paths = algo.sampler.obtain_samples(0)
    sd = algo.sampler.process_samples(0, paths)
    b = sd.lane_batch
    keep = b.valid_mask().reshape(-1)
    prob = b.mean.cpu().numpy().reshape(2, -1).T.astype(np.float64)[keep]
    ent = algo.sampler.stats["Entropy"]
    np.testing.assert_allclose(ent, np.mean(C.entropy(prob)), rtol=1e-6)
    np.testing.assert_allclose(algo.sampler.stats["Perplexity"], np.exp(ent), rtol=1e-12)
    acts = sd["actions"]
    assert acts.shape == (keep.sum(), 2) and np.all(acts.sum(axis=1) == 1) and set(np.unique(acts)) <= {0.0, 1.0}
    assert set(sd["agent_infos"]) == {"prob"}
    np.testing.assert_allclose(sd["agent_infos"]["prob"], prob, rtol=0, atol=0)
    p0 = paths.to_paths()[0]
    assert set(p0["agent_infos"]) == {"prob"} and p0["actions"].shape[1] == 2
    np.testing.assert_array_equal(p0["rewards"], 1.0)


@pytest.mark.parametrize("algo_name", ["vpg", "ppo", "erwr", "reps"])
def test_other_algos_update_through_host_api(dev, algo_name):
    from rllab_b200.misc import logger
    algo = _algo(algo_name, 256, 100, n_itr=2)
    th0 = algo.policy.get_param_values()
    algo.train()
    th1 = algo.policy.get_param_values()
    assert np.all(np.isfinite(th1)) and np.any(th1 != th0)
    tab = logger.get_last_table()
    assert np.isfinite(tab["AverageReturn"]) and tab["Iteration"] == 1


CURVE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "oracle_cartpole_v0_trpo_curve.json")


def test_reference_example_learns(dev):
    """examples/trpo_gym_cartpole.py: TRPO, CategoricalMLPPolicy (32, 32), LinearFeatureBaseline, batch 4000,
    max_path_length 200, discount 0.99, step_size 0.01, against the band of the float64 oracle's curves over several
    seeds (tests/golden/make_cartpole_v0_curve.py; the RNG streams differ, so bands, not values): at iteration 0 at most
    the band's top plus its width; over the last 5 iterations a mean of at least the lowest seed's mean less its spread."""
    import json
    from rllab_b200.misc import logger
    curves = np.array(list(json.load(open(CURVE))["AverageReturn"].values()))
    n_itr = curves.shape[1]
    first_hi = curves[:, 0].max() + (curves[:, 0].max() - curves[:, 0].min())
    late = curves[:, -5:].mean(axis=1)
    late_lo = late.min() - (late.max() - late.min())
    algo = _algo("trpo", None, 200, n_itr=n_itr, batch_size=4000, step_size=0.01, sampler_args=dict(seed=7))
    algo.start_worker()
    algo.init_opt()
    rets = []
    for itr in range(n_itr):
        algo.train_itr(itr)
        rets.append(logger.get_last_table()["AverageReturn"])
    print("CartPole-v0 TRPO AverageReturn per iteration:", [round(r, 1) for r in rets], "bounds", first_hi, late_lo)
    assert rets[0] <= first_hi, (rets[0], first_hi)
    assert np.mean(rets[-5:]) >= late_lo, (rets, late_lo)
