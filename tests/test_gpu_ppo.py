"""GPU: PPO and ERWR.

Kernel (b200rl_grad_penalized) against the float64 oracle grad_surr + penalty * grad_mean_kl (tests/ppo_oracle.py), on
the synthetic batches of test_gpu_update_shapes.py: every compiled net, B in {1, 77, 128*37, (17 n_sm + 5)*128 - 51},
penalty in {0, 1, 1e3} at the off-policy theta_3 (KL > 0), unmasked and masked, TRPO kind, plus VPG kind at one size;
the bounds of that file (2e-4 relative + 5e-6 of the largest entry).  Then: bit-identity with b200rl_grad, the
PenaltyLbfgsOptimizer step against the same host optimizer driven by the oracle, and end-to-end runs.
"""
import pickle

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import ppo_oracle as K                                                   # noqa: E402
from oracle import policy as P                                           # noqa: E402
from test_gpu_update_shapes import SHAPES, SIZES, _assert_grad, _case, _f32, _id, dev, n_sm  # noqa: E402,F401

PENALTIES = (0.0, 1.0, 1e3)


def _ops():
    from rllab_b200 import ops
    return ops


def _L():
    from rllab_b200 import _lib
    return _lib


def _run_pen(c, th_d, kind, pen, dev, min_std=1e-6):
    g = torch.zeros(c.dims.P, dtype=torch.float64, device=dev)
    tri = torch.zeros(3, dtype=torch.float64, device=dev)
    _ops().grad_penalized(kind, pen, th_d, c.dd, min_std, c.b, g, tri)
    return g, tri


def _check_penalized(c, dev, kinds):
    L = _L()
    th, _ = c.theta3()
    th_d = torch.tensor(th, dtype=torch.float32, device=dev)
    assert P.kl_stats(th, c.batch(), c.dims)[0] > 1e-3
    for kind, name in kinds:
        for pen in PENALTIES:
            g, _ = _run_pen(c, th_d, kind, pen, dev)
            ref = c.ref(("pen", name, pen), lambda: K.grad_penalized(th, c.batch(), c.dims, name, pen))
            _assert_grad(g.cpu().numpy(), ref)


@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("shape", SHAPES, ids=_id)
def test_penalized_gradient_matches_oracle(dev, n_sm, shape, size):
    kinds = [(_L().LOSS_TRPO, "trpo")] + ([(_L().LOSS_VPG, "vpg")] if size == "exact" else [])
    _check_penalized(_case(dev, n_sm, shape, size), dev, kinds)


@pytest.mark.parametrize("size", ["77", "large"])
@pytest.mark.parametrize("shape", SHAPES, ids=_id)
def test_penalized_gradient_masked(dev, n_sm, shape, size):
    _check_penalized(_case(dev, n_sm, shape, size, masked=True), dev, [(_L().LOSS_TRPO, "trpo")])


def _assert_grad_clamped(g, ref):
    # a component clamped at sigma = 1e-3 gives its mean the KL weight 2 / (2 sigma^2 + 1e-8) ~ 1e6: the float32-grade
    # mean's own error (~1e-7) becomes ~0.1 per sample in that component's output delta.  Measured on an H100 up to
    # 6.4e-6 of the largest entry and 1.2e-3 relative on the log_std slot of the unclamped component (B = 77)
    np.testing.assert_allclose(g, ref, rtol=2e-3, atol=5e-5 * np.abs(ref).max() + 1e-9)


@pytest.mark.parametrize("shape", [s for s in SHAPES if s[1] > 1], ids=_id)
def test_penalized_gradient_min_std_clamp(dev, n_sm, shape):
    """log_std[0] below log(min_std = 1e-3): its slot is exactly 0; the other components keep their gradient."""
    L = _L()
    c = _case(dev, n_sm, shape, "77")
    A, ols = c.A, c.dims.P - c.A
    th = c.theta2()
    th[ols] = np.log(1e-3) - 1.0
    th = _f32(th)
    th_d = torch.tensor(th, dtype=torch.float32, device=dev)
    g, _ = _run_pen(c, th_d, L.LOSS_TRPO, 1.0, dev, min_std=1e-3)
    g = g.cpu().numpy()
    ref = K.grad_penalized(th, c.batch(), c.dims, "trpo", 1.0, min_std=1e-3)
    assert g[ols] == 0.0 and ref[ols] == 0.0
    _assert_grad_clamped(g, ref)
    _assert_grad_clamped(g[ols:], ref[ols:])


@pytest.mark.parametrize("shape", SHAPES, ids=_id)
def test_penalty_zero_and_triple_equal_grad_pass(dev, n_sm, shape):
    """penalty 0: g and the triple equal b200rl_grad's exactly (the same pass); penalty > 0: the triple equals
    b200rl_grad's exactly and g differs; two runs are bit-identical."""
    ops, L = _ops(), _L()
    c = _case(dev, n_sm, shape, "large", masked=True)
    th_d = torch.tensor(c.theta3()[0], dtype=torch.float32, device=dev)
    for kind in (L.LOSS_TRPO, L.LOSS_VPG):
        g0 = torch.zeros(c.dims.P, dtype=torch.float64, device=dev)
        t0 = torch.zeros(3, dtype=torch.float64, device=dev)
        ops.grad(kind, th_d, c.dd, 1e-6, c.b, g0, t0)
        g, t = _run_pen(c, th_d, kind, 0.0, dev)
        assert torch.equal(g, g0) and torch.equal(t, t0)
        for pen in (1.0, 1e3):
            g1, t1 = _run_pen(c, th_d, kind, pen, dev)
            g2, t2 = _run_pen(c, th_d, kind, pen, dev)
            assert torch.equal(t1, t0)
            assert torch.equal(g1.view(torch.int64), g2.view(torch.int64)) and torch.equal(t1, t2)
            assert not torch.equal(g1, g0)


# ------------------------------------------------------------------------------------------- host optimizer
def _make(env_name):
    import bench
    return bench.make_env(env_name)


def _algo(algo_name, n_envs, T, n_itr=3, hidden=32, env_name="cartpole", baseline=None, **kw):
    from rllab_b200.algos.erwr import ERWR
    from rllab_b200.algos.ppo import PPO
    from rllab_b200.baselines.linear_feature_baseline import LinearFeatureBaseline
    from rllab_b200.policies.gaussian_mlp_policy import GaussianMLPPolicy
    env = _make(env_name)
    policy = GaussianMLPPolicy(env.spec, hidden_sizes=(hidden, hidden), seed=3)
    if baseline is None:
        baseline = LinearFeatureBaseline(env.spec)
    args = dict(env=env, policy=policy, baseline=baseline, batch_size=n_envs * T, max_path_length=T, n_itr=n_itr,
                discount=0.99, sampler_args=dict(n_envs=n_envs, seed=7))
    args.update(kw)
    return PPO(**args) if algo_name == "ppo" else ERWR(**args)


class _HostTarget(object):
    def __init__(self, theta):
        self.theta = np.array(theta, dtype=np.float64)

    def get_param_values(self, trainable=False):
        return self.theta.copy()

    def set_param_values(self, v, trainable=False):
        self.theta = np.array(v, dtype=np.float64)


def _oracle_step(b, pol, theta0, optimizer_args, step_size=0.01):
    """The host PenaltyLbfgsOptimizer on the oracle's float64 callables over the read-back batch."""
    from rllab_b200.optimizers.penalty_lbfgs_optimizer import PenaltyLbfgsOptimizer
    valid = b.valid_mask().reshape(-1)
    O, A = b.O, b.A
    batch = dict(obs=b.obs.cpu().numpy().reshape(O, -1).T[valid].astype(np.float64),
                 actions=b.act.cpu().numpy().reshape(A, -1).T[valid].astype(np.float64),
                 adv=b.adv.cpu().numpy().reshape(-1)[valid].astype(np.float64),
                 old_mean=b.mean.cpu().numpy().reshape(A, -1).T[valid].astype(np.float64),
                 old_log_std=b.log_std.cpu().numpy().astype(np.float64))
    dims = P.Dims(O, (pol.h1, pol.h2), A)
    tgt = _HostTarget(theta0)
    opt = PenaltyLbfgsOptimizer(**optimizer_args)
    ms = pol.min_std
    opt.update_opt(loss=lambda d: K.penalized_loss(tgt.theta, d, dims, "trpo", 0.0, ms)[1], target=tgt,
                   leq_constraint=(lambda d: P.kl_stats(tgt.theta, d, dims, ms)[0], step_size),
                   f_opt=lambda d, pen: (K.penalized_loss(tgt.theta, d, dims, "trpo", pen, ms)[0],
                                         K.grad_penalized(tgt.theta, d, dims, "trpo", pen, ms)),
                   f_penalized_loss=lambda d, pen: K.penalized_loss(tgt.theta, d, dims, "trpo", pen, ms))
    before = (opt.loss([batch]), opt.constraint_val([batch]))
    opt.optimize([batch])
    after = (opt.loss([batch]), opt.constraint_val([batch]))
    return tgt.theta, opt, before, after


def _device_step(optimizer_args, n_envs=2048, T=100):
    algo = _algo("ppo", n_envs, T, optimizer_args=optimizer_args)
    algo.start_worker()
    algo.init_opt()
    paths = algo.sampler.obtain_samples(0)
    sd = algo.sampler.process_samples(0, paths)
    theta0 = algo.policy.get_param_values()
    before = algo._objective.eval_lazy(sd)          # the same (cached) pass optimize_policy records as LossBefore
    algo.optimize_policy(0, sd)
    return algo, sd.lane_batch, theta0, before, algo._objective.eval_lazy(sd)


@pytest.mark.parametrize("max_opt_itr", [1, 2])
def test_penalty_lbfgs_step_short_matches_oracle(dev, max_opt_itr):
    """max_opt_itr 1 / 2 on a 2048 x 100 CartPole batch: the same penalties tried, theta within 1e-5 of max |theta| of
    the oracle-driven step.  The device's loss and gradient are float32-grade (~1e-7 relative at this batch size); one or
    two L-BFGS iterations from the same start scale that by the step length.  Measured on an H100: 4.5e-8 (1 iteration)
    and 7.8e-8 (2 iterations), penalties 1, 2 in both runs."""
    algo, b, theta0, _, _ = _device_step(dict(max_opt_itr=max_opt_itr))
    th_ref, opt, _, _ = _oracle_step(b, algo.policy, theta0, dict(max_opt_itr=max_opt_itr))
    th = algo.policy.get_param_values()
    rel = np.max(np.abs(th - th_ref)) / np.max(np.abs(th_ref))
    print("max_opt_itr %d: penalties %s vs %s, theta rel err %.3g" %
          (max_opt_itr, algo.optimizer.tried_penalties, opt.tried_penalties, rel))
    assert algo.optimizer.tried_penalties == opt.tried_penalties
    assert rel < 1e-5, rel


def test_penalty_lbfgs_step_defaults(dev):
    """Default optimizer settings: the loss decreases, the accept decision (theta moved or restored) is the oracle's, and
    the mean KL is within step_size whenever the oracle's is."""
    algo, b, theta0, before, after = _device_step(dict())
    th_ref, opt, before_ref, after_ref = _oracle_step(b, algo.policy, theta0, dict())
    th = algo.policy.get_param_values()
    print("defaults: penalties %s (%s) vs oracle %s; loss after %.6g (oracle %.6g), kl %.4g (oracle %.4g)" %
          (algo.optimizer.tried_penalties, [t[1:] for t in algo.optimizer.terminations], opt.tried_penalties,
           after[0], after_ref[0], after[1], after_ref[1]))
    assert after[0] < before[0]
    assert np.array_equal(th, theta0) == np.array_equal(th_ref, theta0)
    if after_ref[1] <= 0.01:
        assert after[1] <= 0.01


# ------------------------------------------------------------------------------------------- end to end
def _train_logged(algo, n):
    from rllab_b200.misc import logger
    algo.start_worker()
    algo.init_opt()
    tables = []
    for itr in range(n):
        algo.train_itr(itr)
        tables.append(logger.get_last_table())
    return tables


@pytest.fixture(scope="module", autouse=True)
def _quiet(dev):
    from rllab_b200.misc import logger
    logger.set_quiet(True)


def test_ppo_cartpole_learns(dev):
    tables = _train_logged(_algo("ppo", 256, 100, n_itr=10), 10)
    for t in tables:
        for k in ("LossBefore", "LossAfter", "MeanKLBefore", "MeanKL", "dLoss"):
            assert k in t and np.isfinite(t[k]), k
    r = [t["AverageReturn"] for t in tables]
    print("PPO CartPole AverageReturn", np.round(r, 2))
    assert np.mean(r[-3:]) > np.mean(r[:3])


def test_ppo_hopper_and_mlp_baseline_run(dev):
    from rllab_b200.baselines.gaussian_mlp_baseline import GaussianMLPBaseline
    for algo in (_algo("ppo", 256, 100, n_itr=2, hidden=64, env_name="hopper"),
                 _algo("ppo", 256, 100, n_itr=2, baseline=GaussianMLPBaseline(_make("cartpole").spec))):
        for t in _train_logged(algo, 2):
            for k in ("LossBefore", "LossAfter", "MeanKL", "AverageReturn"):
                assert np.isfinite(t[k]), k
        assert np.isfinite(algo.policy.get_param_values()).all()


def test_erwr_cartpole(dev):
    algo = _algo("erwr", 256, 100, n_itr=3)
    assert algo.positive_adv
    algo.start_worker()
    algo.init_opt()
    from rllab_b200.misc import logger
    for itr in range(3):
        sd = algo.train_itr(itr)
        adv = sd.lane_batch.adv.cpu().numpy()[sd.lane_batch.valid_mask()]
        assert adv.min() >= -1e-6 * adv.max(), adv.min()        # shifted to >= 0 up to float32 rounding of the centring
        t = logger.get_last_table()
        assert t["LossAfter"] <= t["LossBefore"], (t["LossBefore"], t["LossAfter"])
        assert np.isfinite(t["MeanKL"]) and np.isfinite(t["MaxKL"])


def test_ppo_snapshot_and_resume(dev, tmp_path):
    from rllab_b200.misc import logger
    logger.set_snapshot_dir(str(tmp_path))
    logger.set_snapshot_mode("last")
    try:
        algo = _algo("ppo", 256, 50, n_itr=2)
        algo.train()
        data = pickle.load(open(str(tmp_path / "params.pkl"), "rb"))
    finally:
        logger.set_snapshot_mode("none")
        logger.set_snapshot_dir(None)
    assert data["algo"].optimizer._penalty == algo.optimizer._penalty
    resumed = data["algo"]
    resumed.n_itr = 3
    resumed.train()
    algo3 = _algo("ppo", 256, 50, n_itr=3)
    algo3.start_worker()
    algo3.init_opt()
    algo3.train_itr(0)
    algo3.train_itr(1)
    algo3.init_opt()
    algo3.train_itr(2)
    np.testing.assert_array_equal(resumed.policy.get_param_values(), algo3.policy.get_param_values())
    assert resumed.optimizer._penalty == algo3.optimizer._penalty
