"""GPU: GaussianGRUPolicy -- the fused recurrent rollout and get_actions, the loss/KL, BPTT gradient (+ KL penalty) and
Fisher-vector passes in float32, and the float64 parity passes, against the float64 oracle (tests/gru_oracle.py) on
lanes whose paths restart mid-lane, masked and unmasked, both input layouts, at theta_old and away from it; whole TRPO
steps (float32, precision="f64", FiniteDifferenceHvp) and their accepted points, VPG, PPO and ERWR steps against the
oracle-driven optimizers, the recurrent wire format, and the reference's examples/trpo_cartpole_recurrent.py."""
import os

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import gru_oracle as G          # noqa: E402

DIMS = G.GruDims(4, 32, 1, True)
# The points the update passes are evaluated at: theta_old (ratio 1, KL 0); near, theta_old + 0.02 randn with log_std
# + 0.05, what TRPO's backtracking line search and the first L-BFGS iterates evaluate; far, the theta3 rule of
# test_gpu_update_shapes.py (log likelihood ratios spanning e^-2 .. e^2), where PPO's penalty L-BFGS probes.
POINTS = ("old", "near", "far")
PENALTIES = (0.0, 1.0, 1e3)
# float32 BPTT error bound per T, relative to the largest entry of the float64 result, at every point: the largest error
# an H100 80GB HBM3 measured over the passes, lane counts, layouts and mask settings of test_passes_match_oracle at that
# T with a margin of about 4x (DESIGN.md section 5).  theta_old: 1.2e-6, 4.7e-6, 7.9e-7, 2.6e-6 at T = 1, 16, 100,
# 500 (penalty 1 and the Fisher product included; the T = 16 maximum is the 20000-lane case, whose penalised gradients
# sum the most samples); near and far without a penalty at most 1.2e-6.
F32_TOL = {1: 5e-6, 16: 2e-5, 100: 4e-6, 500: 1e-5}
# penalty 1e3: the per-sample output delta 2 pen (old_mean - mu) / var2 carries the float32 mean's rounding, about one
# ulp of |mu|, so on top of F32_TOL the gradient may err by PEN_FLOOR_K * 2 pen ulp(max |mu|) / var2 (_grad_err); the
# largest error measured was 0.36 of that term
PEN_FLOOR_K = 1.5
# relative bound of the float32 (loss, mean KL, max KL) triple over an absolute floor of 1e-7 (largest measured excess
# 2.1e-6 at theta_old, 1.2e-6 near, 3.4e-7 far)
TRIPLE_RTOL = 1e-5
# relative bound of the loss and mean KL TRPO records at its accepted parameters, float32 and float64 passes (measured
# 4.4e-7 and 6.7e-16)
ACCEPTED_RTOL = {"f32": 2e-6, "f64": 1e-12}
# theta after one or two L-BFGS iterations of PPO / ERWR against the oracle-driven run (measured at most 5.5e-8)
LBFGS_THETA_RTOL = 2.5e-7


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


def _grad_err(g, ref, floor):
    """The error of a float32 gradient relative to the largest oracle entry, less what an absolute floor (the rounding
    a KL penalty amplifies) accounts for, and the error as a multiple of that floor."""
    e = np.max(np.abs(g - ref))
    return max(e - PEN_FLOOR_K * floor, 0.0) / np.max(np.abs(ref)), (e / floor if floor else 0.0)


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


def _lane_case(dev, N, T, masked, seed, inc=True):
    """Synthetic lanes recorded at theta (paths of random lengths) as a LaneBatch, and the oracle's dict."""
    ops, L = _ops(), _L()
    rng = np.random.RandomState(seed)
    dims = G.GruDims(4, 32, 1, inc)
    theta = _theta(dims, seed)
    lanes = G.synthetic_lanes(dims, N, T, rng, theta, path_len=(1, min(T, 60)), masked_frac=0.3 if masked else 0.0)
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


def _eval_point(point, theta, lanes, dims, seed):
    """The evaluation point of POINTS for lanes recorded at theta, rounded to float32 as the kernels read it."""
    if point == "old":
        return theta
    if point == "near":
        th = theta + 0.02 * np.random.RandomState(seed).randn(dims.P)
        th[-dims.A:] = theta[-dims.A:] + 0.05
        return _f32(th)
    v = G.valid_of(lanes)
    for s in range(10, 20):
        d = np.random.RandomState(s).randn(dims.P)
        d[-dims.A:] = 0.2                                  # the std moves too
        for step in (0.1, 0.15, 0.2, 0.3):
            th = _f32(theta + d * step)
            lr = G.log_ratio(th, lanes, dims)[v]
            if lr.min() <= -2.0 and lr.max() >= 2.0:
                return th
    raise AssertionError("no far point spans the likelihood ratios e^-2 .. e^2")


def _assert_triple(o, ref, point, what):
    np.testing.assert_allclose(o, ref, rtol=TRIPLE_RTOL, atol=1e-7, err_msg="%s at %s" % (what, point))
    return np.max(np.maximum(np.abs(o - ref) - 1e-7, 0.0) / np.abs(ref))


# (T, lanes, layout): 20000 lanes are 157 tiles of 128, more than one tile per CTA of the gradient pass on 132 SMs, and
# more lanes than one grid-stride round of the float64 kernel; "noact" is state_include_action=False (GruNet<4,1,0>:
# I = 4, the Gram's other row map)
@pytest.mark.parametrize("T,N,inc", [pytest.param(1, 37 * 128, True, id="1-4736"), pytest.param(16, 300, True, id="16-300"),
                                     pytest.param(100, 77, True, id="100-77"), pytest.param(500, 19, True, id="500-19"),
                                     pytest.param(16, 20000, True, id="16-20000"),
                                     pytest.param(1, 37 * 128, False, id="1-4736-noact"),
                                     pytest.param(100, 77, False, id="100-77-noact"),
                                     pytest.param(16, 20000, False, id="16-20000-noact")])
@pytest.mark.parametrize("masked", [False, True])
def test_passes_match_oracle(dev, T, N, inc, masked):
    """At each of POINTS: the float32 loss/KL triple, gradient and penalised gradient passes (the penalised pass's
    triple is the gradient pass's, bit for bit) and the float64 parity passes against the oracle; the float64 KL gradient
    near theta_old; the Fisher product, float32 with and without the activation cache and float64, at theta_old only,
    the one point CG evaluates it."""
    ops, L = _ops(), _L()
    b, theta, lanes = _lane_case(dev, N, T, masked, 10 + T + int(masked), inc)
    D = G.GruDims(4, 32, 1, inc)
    dims = ops.GRUDims(4, 32, 1, inc)
    out = torch.empty(3, dtype=torch.float64, device=dev)
    tri0, tri = (torch.empty(3, dtype=torch.float64, device=dev) for _ in range(2))
    g0, g = (torch.empty(D.P, dtype=torch.float64, device=dev) for _ in range(2))
    tag = "T=%d N=%d masked=%s inc=%s" % (T, N, masked, inc)
    for point in POINTS:
        th = _eval_point(point, theta, lanes, D, T)
        tri_ref, g_ref = G.pass_refs(th, lanes, D)
        if point != "old":
            assert tri_ref["trpo"][1] > 1e-3
        th32 = torch.tensor(th, dtype=torch.float32, device=dev)
        th64 = torch.tensor(th, dtype=torch.float64, device=dev)
        errs, terr, fl = {}, {}, {}
        floor = 2.0 * np.spacing(np.float32(np.abs(lanes["old_mean"]).max())) / (2.0 * np.exp(2.0 * th[-1]) + 1e-8)
        for kind, lk in (("trpo", L.LOSS_TRPO), ("vpg", L.LOSS_VPG)):
            ref = np.array(tri_ref[kind])
            ops.loss_kl(lk, th32, dims, None, b, out)
            terr["loss_pass_" + kind] = _assert_triple(out.cpu().numpy(), ref, point, "loss pass " + kind)
            ops.update_f64(0, lk, th64, dims, None, b, None, 0.0, 0.0, None, out)
            np.testing.assert_allclose(out.cpu().numpy(), ref, rtol=1e-10, atol=1e-13)
            ops.grad(lk, th32, dims, None, b, g0, tri0)
            terr["grad_pass_" + kind] = _assert_triple(tri0.cpu().numpy(), ref, point, "gradient pass " + kind)
            for pen in PENALTIES:
                gref = g_ref[kind] + pen * g_ref["kl"]
                if pen:
                    ops.grad_penalized(lk, pen, th32, dims, None, b, g, tri)
                    assert torch.equal(tri, tri0)
                else:
                    g.copy_(g0)
                key = "grad_%s_%g" % (kind, pen)
                errs[key], efl = _grad_err(g.cpu().numpy(), gref, pen * floor if pen >= 1e3 else 0.0)
                if pen >= 1e3:
                    fl[key] = efl
                assert errs[key] < F32_TOL[T], (point, key, errs[key], efl)
            gref = g_ref[kind]
            ops.update_f64(1, lk, th64, dims, None, b, None, 0.0, 0.0, g, out)
            np.testing.assert_allclose(g.cpu().numpy(), gref, rtol=0, atol=1e-10 * np.abs(gref).max())
        print("GRU float32 error %s point=%s: %s | of the penalty floor %s | triple %s" % (
            tag, point, " ".join("%s=%.2e" % kv for kv in sorted(errs.items())),
            " ".join("%s=%.2e" % kv for kv in sorted(fl.items())), " ".join("%s=%.2e" % kv for kv in sorted(terr.items()))))
    # the KL gradient away from theta_old (FiniteDifferenceHvp evaluates it at theta +- eps x)
    th_kl = theta + 1e-3 * np.random.RandomState(T + 1).randn(D.P)
    gk = G.grad(th_kl, lanes, D, "kl")
    ops.update_f64(1, L.LOSS_KL, torch.tensor(th_kl, device=dev), dims, None, b, None, 0.0, 0.0, g, None)
    np.testing.assert_allclose(g.cpu().numpy(), gk, rtol=0, atol=1e-10 * np.abs(gk).max())
    # Fisher product at theta_old: old_mean = the policy's own mean
    th32 = torch.tensor(theta, dtype=torch.float32, device=dev)
    th64 = torch.tensor(theta, dtype=torch.float64, device=dev)
    lanes["old_mean"] = G.forward(theta, lanes, D)[0]
    b.mean.copy_(torch.tensor(lanes["old_mean"].astype(np.float32)))
    x = torch.tensor(np.random.RandomState(T).randn(D.P), dtype=torch.float64, device=dev)
    ref = G.fvp(theta, lanes, D, x.cpu().numpy(), 1e-5)
    hx = torch.empty_like(x)
    ops.fvp(th32, dims, None, b, x, 1e-5, 1.0, hx)
    err = _rel(hx.cpu().numpy(), ref)
    hc = b.hcache(32, 0)
    ops.grad(L.LOSS_TRPO, th32, dims, None, b, g, out, hc)           # writes the cache at theta
    hx2 = torch.empty_like(x)
    ops.fvp(th32, dims, None, b, x, 1e-5, 1.0, hx2, hc)
    np.testing.assert_array_equal(hx2.cpu().numpy(), hx.cpu().numpy())
    ops.update_f64(2, L.LOSS_TRPO, th64, dims, None, b, x, 1e-5, 1.0, hx, None)
    np.testing.assert_allclose(hx.cpu().numpy(), ref, rtol=0, atol=1e-10 * np.abs(ref).max())
    print("GRU float32 error %s: fvp=%.2e" % (tag, err))
    assert err < F32_TOL[T], err


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
    # the line search's loss pass off theta_old: the loss and mean KL recorded at the accepted parameters (as the
    # kernels read them) are the oracle's there
    th_acc = algo.policy.theta32.double().cpu().numpy() if precision == "f32" else theta_dev
    loss, mkl, _ = G.loss_kl(th_acc, lanes, DIMS, "trpo")
    print("GRU TRPO %s accepted point: loss %.3e rel err %.2e, mean KL %.3e rel err %.2e" % (
        precision, loss, abs(li["loss"] / loss - 1), mkl, abs(li["constraint_val"] / mkl - 1)))
    rtol = ACCEPTED_RTOL[precision]
    np.testing.assert_allclose(li["loss"], loss, rtol=rtol, atol=1e-7 if precision == "f32" else 1e-13)
    np.testing.assert_allclose(li["constraint_val"], mkl, rtol=rtol)


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


def test_vpg_updates_match_oracle(dev):
    """Three VPG iterations (Adam moments and step counter carried): theta after each device Adam step is the oracle's
    Adam step on the oracle gradient at float32(theta), and the after-step (loss, mean KL, max KL), off theta_old, is the
    oracle's at the device's new parameters; each iteration restarts from the oracle's theta."""
    from oracle import policy as P
    algo = _algo("vpg")
    algo.start_worker()
    algo.init_opt()
    adam = (np.zeros(DIMS.P), np.zeros(DIMS.P), 0)
    for itr in range(3):
        sd = algo.sampler.process_samples(itr, algo.sampler.obtain_samples(itr))
        lanes = _oracle_lanes(sd)
        theta0 = algo.policy.get_param_values()
        g_ref = G.grad(algo.policy.theta32.double().cpu().numpy(), lanes, DIMS, "vpg")
        theta_ref, m, v, t = P.adam_step(theta0, g_ref, *adam)
        adam = (m, v, t)
        algo.optimize_policy(itr, sd)
        after = np.array([algo.optimizer.eval_lazy(sd)[i] for i in range(3)])    # LossAfter, MeanKL, MaxKL
        ref = np.array(G.loss_kl(algo.policy.theta32.double().cpu().numpy(), lanes, DIMS, "vpg"))
        rel = _rel(algo.policy.get_param_values(), theta_ref)
        print("GRU VPG itr %d: theta rel err %.2e, after-step triple %s vs oracle %s" % (itr, rel, after, ref))
        assert rel < 1e-5, (itr, rel)
        assert ref[1] > 0
        np.testing.assert_allclose(after, ref, rtol=TRIPLE_RTOL, atol=1e-7)
        algo.policy.set_param_values(theta_ref)     # keep both sides on the same trajectory of parameters


def _lbfgs_steps(name, optimizer_args):
    """One PPO (kind trpo, KL <= 0.01) or ERWR (kind vpg, shifted advantages) policy update on the device, and the same
    host optimizer driven by the oracle over the read-back lanes from the same theta."""
    from rllab_b200.optimizers.lbfgs_optimizer import LbfgsOptimizer
    from rllab_b200.optimizers.penalty_lbfgs_optimizer import PenaltyLbfgsOptimizer
    algo = _algo(name, optimizer_args=optimizer_args)
    algo.start_worker()
    algo.init_opt()
    sd = algo.sampler.process_samples(0, algo.sampler.obtain_samples(0))
    lanes = _oracle_lanes(sd)
    theta0 = algo.policy.get_param_values()
    before = algo._objective.eval_lazy(sd)[0]
    algo.optimize_policy(0, sd)
    after = (algo._objective.eval_lazy(sd)[0], algo._objective.eval_lazy(sd)[1])
    if name == "ppo":
        opt = PenaltyLbfgsOptimizer(**optimizer_args)
        th_ref, before_ref, after_ref = G.lbfgs_step(opt, theta0, lanes, DIMS, "trpo", step_size=0.01)
    else:
        opt = LbfgsOptimizer(**optimizer_args)
        th_ref, before_ref, after_ref = G.lbfgs_step(opt, theta0, lanes, DIMS, "vpg")
    th = algo.policy.get_param_values()
    rel = np.max(np.abs(th - th_ref)) / np.max(np.abs(th_ref))
    print("GRU %s %s: penalties %s vs oracle %s; theta rel err %.2e; loss %.6g -> %.6g (oracle %.6g -> %.6g), kl %.4g "
          "(oracle %.4g)" % (name, optimizer_args, getattr(algo.optimizer, "tried_penalties", None),
                             getattr(opt, "tried_penalties", None), rel, before, after[0], before_ref[0], after_ref[0],
                             after[1], after_ref[1]))
    return algo, opt, theta0, th, th_ref, rel, (before, after), (before_ref, after_ref)


@pytest.mark.parametrize("max_opt_itr", [1, 2])
def test_ppo_step_short_matches_oracle(dev, max_opt_itr):
    """max_opt_itr 1 / 2: the same penalties tried as the oracle-driven PenaltyLbfgsOptimizer, theta close to its."""
    algo, opt, _, _, _, rel, _, _ = _lbfgs_steps("ppo", dict(max_opt_itr=max_opt_itr))
    assert algo.optimizer.tried_penalties == opt.tried_penalties
    assert rel < LBFGS_THETA_RTOL, rel


def test_ppo_step_defaults(dev):
    """Default settings: the loss decreases, the accept decision (theta moved or restored) is the oracle's, and the mean
    KL is within the step size whenever the oracle's is."""
    _, _, theta0, th, th_ref, _, (before, after), (_, after_ref) = _lbfgs_steps("ppo", dict())
    assert after[0] < before
    assert np.array_equal(th, theta0) == np.array_equal(th_ref, theta0)
    if after_ref[1] <= 0.01:
        assert after[1] <= 0.01


@pytest.mark.parametrize("max_opt_itr", [1, 2])
def test_erwr_step_matches_oracle(dev, max_opt_itr):
    """ERWR's LbfgsOptimizer on the VPG surrogate of the shifted (non-negative) advantages, max_opt_itr 1 / 2: theta
    close to the oracle-driven run's."""
    _, _, _, _, _, rel, _, _ = _lbfgs_steps("erwr", dict(max_opt_itr=max_opt_itr))
    assert rel < LBFGS_THETA_RTOL, rel


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
