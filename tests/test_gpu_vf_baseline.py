"""GPU: the GaussianMLPBaseline kernels (csrc/vf.cu) against the float64 oracle (tests/vf_oracle.py), the sampler hook,
the whole fit against the oracle's fit, and end-to-end runs.

Kernel matrix: every compiled obs dim x batch sizes B in {1, 77, 128*37, (17 n_sm + 5)*128 - 51} (the last runs the
persistent tile loop at least 8 times per CTA), with and without masked samples and whole masked tiles.
Bounds (the ones of the policy passes in test_gpu_update_shapes.py):
  statistics       float64 sums of float32 data: mean 1e-12, std 1e-10 relative
  forward / loss   float32 per sample and inside a tile: 2e-5 relative
  gradient         2e-4 relative + 5e-6 of the largest entry
"""
import pickle

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import vf_oracle as V                    # noqa: E402

OBS_DIMS = (2, 3, 4, 6, 13, 20)


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
    return torch.cuda.get_device_properties(0).multi_processor_count


def _sizes(n_sm):
    return [1, 77, 128 * 37, (17 * n_sm + 5) * 128 - 51]


def _data(O, B, masked, seed=0):
    rng = np.random.RandomState(seed + 97 * O + B)
    obs = (rng.randn(O, B) * (1.0 + 0.3 * np.arange(O))[:, None] + (0.5 + np.arange(O))[:, None]).astype(np.float32)
    y = (rng.randn(B) * 7.0 + 3.0).astype(np.float32)
    flags = np.zeros(B, dtype=np.uint8)
    if masked:
        flags[rng.rand(B) < 0.1] = 8
        if B > 3 * 128:
            flags[128:256] = 8                     # a whole masked tile
        flags[0] = 0
    return obs, y, flags


def _dev_arrays(dev, obs, y, flags):
    return (torch.tensor(obs, device=dev).contiguous(), torch.tensor(y, device=dev),
            torch.tensor(flags, device=dev))


def _theta(O, seed):
    rng = np.random.RandomState(seed)
    th = V.init_params(O, rng, init_std=1.0)
    P = th.size
    th[O * 32:O * 32 + 32] += 0.1 * rng.randn(32)          # non-zero biases
    th[P - 2] = 0.3
    th[P - 1] = -0.2
    return th.astype(np.float32).astype(np.float64)


def _stats_dev(dev, O, obs, y, flags, valid):
    from rllab_b200 import ops
    o, yy, fl = _dev_arrays(dev, obs, y, flags)
    acc = torch.zeros(2 * O + 3, dtype=torch.float64, device=dev)
    st = torch.zeros(2 * O + 2, dtype=torch.float64, device=dev)
    ops.vf_norm_stats(O, len(y), o, yy, fl if valid is not None else None, ops.VF_STATS_ALL, acc, st)
    return o, yy, fl, acc, st


def _id(O, B, m):
    return "O%d-B%d-%s" % (O, B, "masked" if m else "full")


CASES = [(O, i, m) for O in OBS_DIMS for i in range(4) for m in (False, True)]


@pytest.mark.parametrize("O,bi,masked", CASES, ids=[_id(O, i, m) for O, i, m in CASES])
def test_norm_stats(dev, n_sm, O, bi, masked):
    B = _sizes(n_sm)[bi]
    obs, y, flags = _data(O, B, masked)
    valid = flags == 0
    _, _, _, acc, st = _stats_dev(dev, O, obs, y, flags, valid if masked else None)
    ref = V.norm_stats(obs.T[valid].astype(np.float64), y[valid].astype(np.float64))
    got = st.cpu().numpy()
    assert acc.cpu().numpy()[O + 1] == valid.sum()
    np.testing.assert_allclose(got[:O], ref[:O], rtol=1e-12)
    np.testing.assert_allclose(got[2 * O], ref[2 * O], rtol=1e-12)
    np.testing.assert_allclose(got[O:2 * O], ref[O:2 * O], rtol=1e-10)
    np.testing.assert_allclose(got[2 * O + 1], ref[2 * O + 1], rtol=1e-10)


def _grad_close(g, ref):
    bound = 2e-4 * np.abs(ref) + 5e-6 * np.abs(ref).max()
    err = np.abs(g - ref)
    assert (err <= bound).all(), (np.argmax(err - bound), err.max(), np.abs(ref).max())


@pytest.mark.parametrize("O,bi,masked", CASES, ids=[_id(O, i, m) for O, i, m in CASES])
def test_forward_loss_and_gradient(dev, n_sm, O, bi, masked):
    from rllab_b200 import ops
    B = _sizes(n_sm)[bi]
    obs, y, flags = _data(O, B, masked, seed=1)
    valid = flags == 0
    o, yy, fl, acc, st = _stats_dev(dev, O, obs, y, flags, valid if masked else None)
    stats = st.cpu().numpy()
    th_old, th = _theta(O, 5), _theta(O, 6)
    t_old = torch.tensor(th_old, dtype=torch.float32, device=dev)
    t_new = torch.tensor(th, dtype=torch.float32, device=dev)
    nx, ny = V.normalize(obs.T.astype(np.float64), y.astype(np.float64), stats, O)
    # forward: normalised (trust region input) and denormalised (predict)
    mu_old = torch.empty(B, dtype=torch.float32, device=dev)
    ops.vf_forward(t_old, O, B, o, st, mu_old, False)
    den = torch.empty(B, dtype=torch.float32, device=dev)
    ops.vf_forward(t_old, O, B, o, st, den, True)
    ref_mu = V.forward(th_old, nx, O)[0]
    np.testing.assert_allclose(mu_old.cpu().numpy(), ref_mu, rtol=2e-5, atol=2e-5 * np.abs(ref_mu).max())
    ref_den = ref_mu * stats[2 * O + 1] + stats[2 * O]
    np.testing.assert_allclose(den.cpu().numpy(), ref_den, rtol=2e-5, atol=2e-5 * np.abs(ref_den).max())
    mo = mu_old.cpu().numpy().astype(np.float64)
    ls_old = float(np.float32(th_old[-1]))
    cnt = acc[O + 1:O + 2]
    P = th.size
    w = valid.astype(np.float64) if masked else None
    flp = fl if masked else None
    for trust, learn_std, penalties in ((True, True, (0.0, 1.0, 1e3)), (True, False, (1.0,)), (False, True, (0.0,))):
        for pen in penalties:
            g = torch.zeros(P, dtype=torch.float64, device=dev)
            lo = torch.zeros(3, dtype=torch.float64, device=dev)
            ops.vf_loss_grad(t_new, O, B, o, yy, flp, st, mu_old if trust else None, ls_old, pen, learn_std, 1.0, cnt,
                             g, lo)
            nll, kl, mkl, rg = V.loss_grad(th, nx, ny, O, pen, mo if trust else None, ls_old if trust else None,
                                           learn_std, w)
            lv = lo.cpu().numpy()
            np.testing.assert_allclose(lv[0], nll, rtol=2e-5)
            if trust:
                np.testing.assert_allclose(lv[1], kl, rtol=2e-5, atol=2e-5 * abs(kl) + 1e-7)
                np.testing.assert_allclose(lv[2], mkl, rtol=2e-5, atol=1e-7)
            _grad_close(g.cpu().numpy(), rg)
            # forward-only pass: the same loss triple; two runs bit for bit
            lo2 = torch.zeros(3, dtype=torch.float64, device=dev)
            ops.vf_loss_grad(t_new, O, B, o, yy, flp, st, mu_old if trust else None, ls_old, pen, learn_std, 1.0, cnt,
                             None, lo2)
            np.testing.assert_allclose(lo2.cpu().numpy()[:2], lv[:2], rtol=1e-6, atol=1e-9)
            g2 = torch.zeros(P, dtype=torch.float64, device=dev)
            lo3 = torch.zeros(3, dtype=torch.float64, device=dev)
            ops.vf_loss_grad(t_new, O, B, o, yy, flp, st, mu_old if trust else None, ls_old, pen, learn_std, 1.0, cnt,
                             g2, lo3)
            assert torch.equal(g, g2) and torch.equal(lo, lo3)


def test_unsupported_shape_fails(dev):
    from rllab_b200 import _lib
    with pytest.raises(_lib.B200RLError):
        _lib.vf_num_params(7)
    assert _lib.vf_num_params(4) == 4 * 32 + 32 + 32 * 32 + 32 + 32 + 1 + 1


# ---------------------------------------------------------------- sampler level
def _make(env_name):
    import bench
    return bench.make_env(env_name)


def _algo(algo_name, n_envs, T, baseline=None, n_itr=3, regressor_args=None, hidden=32, **kw):
    from rllab_b200.algos.trpo import TRPO
    from rllab_b200.algos.vpg import VPG
    from rllab_b200.baselines.gaussian_mlp_baseline import GaussianMLPBaseline
    from rllab_b200.policies.gaussian_mlp_policy import GaussianMLPPolicy
    env = _make("cartpole")
    policy = GaussianMLPPolicy(env.spec, hidden_sizes=(hidden, hidden), seed=3)
    if baseline is None:
        np.random.seed(11)
        baseline = GaussianMLPBaseline(env.spec, regressor_args=regressor_args)
    args = dict(env=env, policy=policy, baseline=baseline, batch_size=n_envs * T, max_path_length=T, n_itr=n_itr,
                discount=0.99, sampler_args=dict(n_envs=n_envs, seed=7))
    args.update(kw)
    return TRPO(**args) if algo_name == "trpo" else VPG(**args)


def test_process_samples_base_matches_lfb(dev):
    """b200rl_process_samples_base on the base that b200rl_process_samples wrote for LFB weights: bit-identical."""
    from rllab_b200 import ops
    from rllab_b200.baselines.linear_feature_baseline import LinearFeatureBaseline
    algo = _algo("trpo", 512, 100, baseline=LinearFeatureBaseline(None))
    algo.start_worker()
    paths = algo.sampler.obtain_samples(0)
    b = paths.lane_batch
    w = torch.tensor(np.random.RandomState(3).randn(2 * b.O + 4) * 0.1, dtype=torch.float64, device=dev)
    flags0 = b.flags.clone()
    ops.process_samples(b, w, 0.99, 0.97, drop_cut_paths=True)
    ref = [t.clone() for t in (b.adv, b.ret, b.sums, b.maxs, b.flags)]
    base = b.base.clone()
    b.adv.zero_(), b.ret.zero_(), b.sums.zero_(), b.maxs.zero_()
    b.flags.copy_(flags0)
    b.base.copy_(base)
    ops.process_samples_base(b, 0.99, 0.97, drop_cut_paths=True)
    for r, t in zip(ref, (b.adv, b.ret, b.sums, b.maxs, b.flags)):
        assert torch.equal(r, t)
    assert torch.equal(base, b.base)


def test_process_samples_base_with_regressor_matches_oracle(dev, monkeypatch):
    """predict_lanes + b200rl_process_samples_base against the oracle's process_samples with the regressor's baseline.
    oracle.sampler.process_samples_lanes takes LinearFeatureBaseline weights; its feature map is replaced by the one
    feature `base` (weight 1), so the oracle's own GAE scan and statistics run on the regressor's prediction."""
    from oracle import sampler as S
    from rllab_b200 import ops
    from rllab_b200.baselines.gaussian_mlp_baseline import GaussianMLPBaseline
    algo = _algo("trpo", 512, 100)
    algo.start_worker()
    paths = algo.sampler.obtain_samples(0)
    b = paths.lane_batch
    bl = GaussianMLPBaseline(algo.env.spec)
    bl.set_param_values(_theta(b.O, 9))
    stats = np.concatenate([[0.1, -0.2, 0.05, 0.3], [0.5, 1.5, 0.2, 2.0], [20.0, 15.0]])
    bl.regressor._ensure_device()["stats"].copy_(torch.as_tensor(stats))
    bl.predict_lanes(b)
    ops.process_samples_base(b, 0.99, 0.97, drop_cut_paths=True)
    traj = b.to_numpy()
    xs = traj["obs"].reshape(b.O, -1).T.astype(np.float64)
    ref_base = V.predict(bl.get_param_values(), xs, stats, b.O).reshape(b.T, b.N)
    np.testing.assert_allclose(b.base.cpu().numpy(), ref_base, rtol=2e-5, atol=2e-5 * np.abs(ref_base).max())
    base = b.base.cpu().numpy().astype(np.float64)       # the scan is compared on the device's own prediction
    monkeypatch.setattr(S, "lfb_features_lanes", lambda obs, tstep: base[None])
    ref = S.process_samples_lanes(traj, np.ones(1), 0.99, 0.97, center_adv=True, drop_cut=True)
    np.testing.assert_allclose(b.ret.cpu().numpy(), ref["ret"], rtol=1e-5, atol=1e-4)
    np.testing.assert_allclose(b.adv.cpu().numpy(), ref["adv_raw"], rtol=1e-5, atol=2e-4)
    s = b.sums.cpu().numpy()
    m = b.maxs.cpu().numpy()
    assert int(round(s[3])) == ref["stats"]["NumTrajs"]
    np.testing.assert_allclose(s[0] / s[2], ref["stats"]["adv_mean"], rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(np.sqrt(s[1] / s[2] - (s[0] / s[2]) ** 2), ref["stats"]["adv_std"], rtol=1e-6)
    vary = s[8] / s[2] - (s[7] / s[2]) ** 2
    varres = s[12] / s[2] - (s[11] / s[2]) ** 2
    np.testing.assert_allclose(1 - varres / (vary + 1e-8), ref["stats"]["ExplainedVariance"], rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose([m[0], -m[1]], [ref["stats"]["MaxReturn"], ref["stats"]["MinReturn"]], rtol=1e-6)


def _fit_setup(dev, max_opt_itr, n_envs=2048, T=100):
    """One TRPO CartPole batch; returns the baseline's theta before the fit, the batch, the regressor."""
    from rllab_b200.optimizers.penalty_lbfgs_optimizer import PenaltyLbfgsOptimizer
    ra = dict(optimizer=PenaltyLbfgsOptimizer(max_opt_itr=max_opt_itr))
    algo = _algo("trpo", n_envs, T, regressor_args=ra)
    algo.start_worker()
    algo.init_opt()
    reg = algo.baseline.regressor
    theta0 = reg.get_param_values().astype(np.float32).astype(np.float64)
    paths = algo.sampler.obtain_samples(0)
    sd = algo.sampler.process_samples(0, paths)
    return algo, sd.lane_batch, reg, theta0


def _oracle_fit(b, theta0, max_opt_itr):
    from rllab_b200.optimizers.penalty_lbfgs_optimizer import PenaltyLbfgsOptimizer
    valid = b.valid_mask().reshape(-1)
    xs = b.obs.cpu().numpy().reshape(b.O, -1).T[valid].astype(np.float64)
    ys = b.ret.cpu().numpy().reshape(-1)[valid].astype(np.float64)
    opt = PenaltyLbfgsOptimizer(max_opt_itr=max_opt_itr)
    th, stats, info = V.fit(theta0, xs, ys, b.O, opt)
    return th, stats, info, opt


@pytest.mark.parametrize("max_opt_itr", [1, 2])
def test_whole_fit_short_matches_oracle(dev, max_opt_itr):
    """max_opt_itr 1 / 2: same penalty sequence, parameters within 1e-5 of the largest parameter.  The device's loss and
    gradient are float32-grade (1e-7 relative on a batch of this size, far inside the 2e-4 bound above); one or two
    L-BFGS iterations from the same start scale that error by the step length, at most the parameters' own scale.
    Measured on an H100: 1.2e-7 (1 iteration) and 2.3e-7 (2 iterations)."""
    from rllab_b200.misc import logger
    algo, b, reg, theta0 = _fit_setup(dev, max_opt_itr)
    tab = dict(logger._tabular)
    th_ref, stats_ref, info, opt = _oracle_fit(b, theta0, max_opt_itr)
    np.testing.assert_allclose(reg.get_stats(), stats_ref, rtol=1e-10)
    np.testing.assert_allclose(tab["vf_LossBefore"], info["LossBefore"], rtol=2e-5)
    assert reg._optimizer.tried_penalties == opt.tried_penalties
    th = reg.get_param_values()
    rel = np.max(np.abs(th - th_ref)) / np.max(np.abs(th_ref))
    print("max_opt_itr %d: penalties %s, theta rel err %.3g, loss after %.8g vs %.8g" %
          (max_opt_itr, opt.tried_penalties, rel, tab["vf_LossAfter"], info["LossAfter"]))
    assert rel < 1e-5, rel


def test_whole_fit_defaults(dev):
    """Default settings: the loss decreases, the accepted KL is inside the trust region, and the loss after the fit is
    within 1e-3 (absolute, on a per-sample NLL of order 1) of the oracle's fit on the same float32 data."""
    from rllab_b200.misc import logger
    algo, b, reg, theta0 = _fit_setup(dev, 20)
    tab = dict(logger._tabular)
    th_ref, _, info, opt = _oracle_fit(b, theta0, 20)
    print("defaults: device penalties %s (%s) evals %d; oracle penalties %s; loss %.6g -> %.6g (oracle %.6g), kl %.4g" %
          (reg._optimizer.tried_penalties, [t[1] for t in reg._optimizer.terminations], reg.last_fit["n_evals"],
           opt.tried_penalties, tab["vf_LossBefore"], tab["vf_LossAfter"], info["LossAfter"], tab["vf_MeanKL"]))
    assert tab["vf_LossAfter"] <= tab["vf_LossBefore"]
    assert tab["vf_MeanKL"] <= 0.01
    assert abs(tab["vf_LossAfter"] - info["LossAfter"]) < 1e-3


def test_vpg_reference_case(dev):
    """rllab's tests/test_baselines.py with GaussianMLPBaseline: VPG, normalize(CartpoleEnv()), 1 iteration, batch 1000,
    max_path_length 100 ((32,32) policy: (6,) is not compiled)."""
    algo = _algo("vpg", 10, 100, n_itr=1)
    algo.train()
    assert np.isfinite(algo.policy.get_param_values()).all()
    assert np.isfinite(algo.baseline.get_param_values()).all()


def _train_logged(algo, n):
    from rllab_b200.misc import logger
    algo.start_worker()
    algo.init_opt()
    tables = []
    for itr in range(n):
        algo.train_itr(itr)
        tables.append(logger.get_last_table())
    return tables


def test_trpo_run_logs_and_improves(dev):
    tables = _train_logged(_algo("trpo", 1024, 100, n_itr=5), 5)
    for t in tables:
        for k in ("vf_LossBefore", "vf_LossAfter", "vf_dLoss", "vf_MeanKL"):
            assert k in t and np.isfinite(t[k]), k
        assert t["vf_LossAfter"] <= t["vf_LossBefore"]
    assert tables[-1]["ExplainedVariance"] > tables[0]["ExplainedVariance"]


def test_snapshot_and_resume(dev, tmp_path):
    from rllab_b200.misc import logger
    logger.set_snapshot_dir(str(tmp_path))
    logger.set_snapshot_mode("last")
    try:
        algo = _algo("trpo", 256, 50, n_itr=2)
        algo.train()
        data = pickle.load(open(str(tmp_path / "params.pkl"), "rb"))
    finally:
        logger.set_snapshot_mode("none")
        logger.set_snapshot_dir(None)
    reg = data["baseline"].regressor
    assert reg._optimizer._penalty == algo.baseline.regressor._optimizer._penalty
    np.testing.assert_array_equal(reg.get_stats(), algo.baseline.regressor.get_stats())
    resumed = data["algo"]
    resumed.n_itr = 3
    resumed.train()
    algo3 = _algo("trpo", 256, 50, n_itr=3)
    algo3.start_worker()
    algo3.init_opt()
    algo3.train_itr(0)
    algo3.train_itr(1)
    algo3.init_opt()
    algo3.train_itr(2)
    np.testing.assert_array_equal(resumed.policy.get_param_values(), algo3.policy.get_param_values())
    np.testing.assert_array_equal(resumed.baseline.get_param_values(), algo3.baseline.get_param_values())


def test_host_api_matches_lane_hooks(dev):
    """fit(paths) / predict(path) on the host path dicts against fit_lanes / predict_lanes on the same samples.
    The host path uploads the samples in path order (lane-major), the lane hooks read them in time-major lane order, so
    every 128-sample tile holds different samples and the float32 per-tile sums of loss and gradient differ at ~1e-7
    relative.  Four penalty tries of 20 L-BFGS iterations, each step built from gradient differences over a 10-pair
    history, amplify that: measured 3.7e-4 of max |theta| on an H100 (same penalty sequence).  Bound: 1e-3."""
    from rllab_b200.baselines.gaussian_mlp_baseline import GaussianMLPBaseline
    algo = _algo("trpo", 256, 100)
    algo.start_worker()
    algo.init_opt()
    paths = algo.sampler.obtain_samples(0)
    algo.sampler.process_samples(0, paths)
    b = paths.lane_batch
    host = GaussianMLPBaseline(algo.env.spec)
    lanes = GaussianMLPBaseline(algo.env.spec)
    th0 = _theta(b.O, 9)
    host.set_param_values(th0)
    lanes.set_param_values(th0)
    host.fit(paths.to_paths())
    lanes.fit_lanes(b, None)
    s_h, s_l = host.regressor.get_stats(), lanes.regressor.get_stats()
    np.testing.assert_allclose(s_h, s_l, rtol=1e-10)
    assert host.regressor._optimizer.tried_penalties == lanes.regressor._optimizer.tried_penalties
    th_h, th_l = host.get_param_values(), lanes.get_param_values()
    rel = np.max(np.abs(th_h - th_l)) / np.max(np.abs(th_l))
    print("host fit vs lane hooks: theta rel diff %.3g" % rel)
    assert rel < 1e-3
    p = paths.to_paths()[0]
    lanes.predict_lanes(b)
    n = len(p["rewards"])
    np.testing.assert_allclose(lanes.predict(p), b.base.cpu().numpy()[:n, 0], rtol=1e-6, atol=1e-6)
