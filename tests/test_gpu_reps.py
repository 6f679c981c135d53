"""GPU: REPS.

Kernels (b200rl_reps_delta_max + b200rl_reps_dual_sums, formed into g and its gradient by the host half,
rllab_b200.algos.reps.dual_from_sums) against the float64 oracle (tests/reps_oracle.py) on synthetic lane batches: every
compiled obs_dim, B in {1, 77, a multi-wave size}, unmasked / masked (dropped cut paths) / cut paths kept
(whole_paths=False), eta in {1e-2, 1, 15, 1e3} with random v; the extreme cases (delta / eta ~ 1e4, eta = 0); the weights;
the VPG gradient pass on adv = w.  Then the host class: short L-BFGS steps against the same steps driven by the oracle,
the default settings, end-to-end runs and the snapshot.
"""
import copy
import pickle

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import reps_oracle as K                                                  # noqa: E402
from oracle import policy as P                                           # noqa: E402
from test_gpu_update_shapes import SHAPES, _assert_grad, _case, _id, dev, n_sm  # noqa: E402,F401

OBS_DIMS = (2, 3, 4, 6, 13, 20)
ETAS = (1e-2, 1.0, 15.0, 1e3)
MODES = ("unmasked", "masked", "cut")


def _ops():
    from rllab_b200 import ops
    return ops


def _L():
    from rllab_b200 import _lib
    return _lib


def _geometry(size, n_sm):
    # "wave": more samples than one sweep of the persistent grid (n_sm x 4 CTAs x 256 threads), ~3 sweeps
    return {"1": (1, 1), "77": (7, 11), "wave": (1031, (3 * n_sm * 4 * 256) // 1031 + 1)}[size]


class LaneCase(object):
    """A synthetic lane batch: random paths (ends with probability 0.06 per step), each lane's last path cut by the end
    of the buffer (FLAG_END | FLAG_CUT); "masked" drops the cut paths as process_samples(drop_cut_paths) does."""

    def __init__(self, dev, O, N, T, mode, seed=0):
        ops, L = _ops(), _L()
        rng = np.random.RandomState(seed + 100 * O + N)
        self.O, self.N, self.T, self.mode = O, N, T, mode
        obs = (rng.randn(O, T, N) * 3.0).astype(np.float32)
        big = rng.rand(O, T, N) < 0.05
        obs[big] = (np.sign(rng.randn(int(big.sum()))) * rng.uniform(10.0, 30.0, int(big.sum()))).astype(np.float32)
        rew = (rng.rand(T, N) * 2.0 - 0.5).astype(np.float32)
        ends = rng.rand(T, N) < 0.06
        flags = np.where(ends, L.FLAG_END, 0).astype(np.uint8)
        flags[T - 1] |= L.FLAG_END
        if mode != "unmasked":              # "unmasked": every lane's last path happens to end with the buffer
            flags[T - 1] |= np.where(ends[T - 1], 0, L.FLAG_CUT).astype(np.uint8)
        tstep = np.zeros((T, N), np.uint16)
        for t in range(1, T):
            tstep[t] = np.where(flags[t - 1] & L.FLAG_END, 0, tstep[t - 1] + 1)
        keep = np.ones((T, N), bool)
        if mode == "masked":
            for n in range(N):
                if flags[T - 1, n] & L.FLAG_CUT:
                    e = np.nonzero(flags[:T - 1, n] & L.FLAG_END)[0]
                    start = e[-1] + 1 if len(e) else 0
                    keep[start:, n] = False
                    flags[start:, n] |= L.FLAG_MASKED
        if not keep.any():                  # B = 1 with its only path dropped: keep the sample (a count of 0 is no case)
            keep[:] = True
            flags &= ~np.uint8(L.FLAG_MASKED)
        b = ops.LaneBatch(O, 1, N, T, dev)
        b.obs.copy_(torch.tensor(obs))
        b.rew.copy_(torch.tensor(rew))
        b.flags.copy_(torch.tensor(flags))
        b.tstep.copy_(torch.tensor(tstep.view(np.int16)).view(torch.uint16))
        b.masked = bool((flags & L.FLAG_MASKED).any())
        b.sums[2] = float(keep.sum())
        self.b, self.keep, self.flags = b, keep, flags
        fd = K.feat_diff_lanes(obs, flags, tstep)
        self.fd = fd[keep]
        self.rew = rew[keep].astype(np.float64)
        self.count = float(keep.sum())
        torch.cuda.synchronize()


_LCASES = {}


def _lcase(dev, n_sm, O, size, mode):
    key = (O, size, mode)
    if key not in _LCASES:
        _LCASES.clear()                     # one case alive at a time (the oracle's feat_diff is the large part)
        _LCASES[key] = LaneCase(dev, O, *_geometry(size, n_sm), mode)
    return _LCASES[key]


def _device_dual(c, eta, v, w_out=None, epsilon=0.5, l2=0.0):
    from rllab_b200.algos.reps import dual_from_sums
    ops, dev = _ops(), c.b.device
    D = 2 * c.O + 4
    vd = torch.tensor(v, dtype=torch.float64, device=dev)
    M = torch.zeros(1, dtype=torch.float64, device=dev)
    sums = torch.zeros(D + 2, dtype=torch.float64, device=dev)
    ops.reps_delta_max(c.b, vd, M)
    ops.reps_dual_sums(c.b, vd, eta, M, sums, w_out)
    g, grad = dual_from_sums(eta, float(M.cpu()[0]), sums.cpu().numpy(), c.count, epsilon, l2)
    return np.concatenate([[g], grad]), float(M.cpu()[0])


def _oracle_dual(c, eta, v, epsilon=0.5, l2=0.0):
    return np.concatenate([[K.dual(eta, v, c.rew, c.fd, epsilon, l2)], K.dual_grad(eta, v, c.rew, c.fd, epsilon, l2)])


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("size", ["1", "77", "wave"])
@pytest.mark.parametrize("O", OBS_DIMS)
def test_dual_matches_oracle(dev, n_sm, O, size, mode):
    c = _lcase(dev, n_sm, O, size, mode)
    rng = np.random.RandomState(O)
    worst = 0.0
    for eta in ETAS:
        v = rng.randn(2 * O + 4) * 0.5
        for l2 in (0.0, 1e-3):
            got, M = _device_dual(c, eta, v, l2=l2)
            ref = _oracle_dual(c, eta, v, l2=l2)
            assert M == pytest.approx(np.max(K.delta(c.rew, c.fd, v)), rel=1e-12, abs=1e-12)
            err = np.max(np.abs(got - ref)) / np.max(np.abs(ref))
            worst = max(worst, err)
            assert err < 1e-9, (eta, l2, err)
    print("O=%d %s %s B=%d: max error %.3g of the largest entry" % (O, size, mode, c.N * c.T, worst))


@pytest.mark.parametrize("O", (4, 20))
def test_dual_extreme_eta(dev, n_sm, O):
    """delta / eta ~ 1e4 stays finite and matches; eta = 0 gives the oracle's non-finite values."""
    c = _lcase(dev, n_sm, O, "wave", "masked")
    v = np.random.RandomState(1).randn(2 * O + 4) * 0.5
    d = K.delta(c.rew, c.fd, v)
    eta = float(np.max(np.abs(d))) / 1e4
    got, _ = _device_dual(c, eta, v)
    ref = _oracle_dual(c, eta, v)
    assert np.isfinite(got).all() and np.isfinite(ref).all()
    err = np.max(np.abs(got - ref)) / np.max(np.abs(ref))
    print("O=%d delta/eta up to 1e4 (eta %.3g): error %.3g" % (O, eta, err))
    assert err < 1e-9, err
    got0, _ = _device_dual(c, 0.0, v)
    ref0 = _oracle_dual(c, 0.0, v)
    print("eta = 0: device %s, oracle %s" % (got0[:2], ref0[:2]))
    assert not np.isfinite(got0).all()
    for pred in (np.isnan, np.isposinf, np.isneginf):
        assert np.array_equal(pred(got0), pred(ref0)), pred.__name__


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("O", (2, 13))
def test_weights_match_oracle(dev, n_sm, O, mode):
    c = _lcase(dev, n_sm, O, "wave", mode)
    v = np.random.RandomState(2).randn(2 * O + 4) * 0.5
    for eta in ETAS:
        w = torch.full((c.T, c.N), 7.0, dtype=torch.float32, device=dev)
        _device_dual(c, eta, v, w_out=w)
        w = w.cpu().numpy()
        assert (w[~c.keep] == 0).all()
        ref = K.weights(eta, v, c.rew, c.fd)
        np.testing.assert_allclose(w[c.keep], ref.astype(np.float32), rtol=1.2e-7, atol=1e-38)   # (subnormals: 1e-38)
    w2 = torch.zeros((c.T, c.N), dtype=torch.float32, device=dev)
    w3 = torch.zeros((c.T, c.N), dtype=torch.float32, device=dev)
    a, _ = _device_dual(c, 1.0, v, w_out=w2)
    b, _ = _device_dual(c, 1.0, v, w_out=w3)
    assert np.array_equal(a, b) and torch.equal(w2, w3)          # reruns are bit-identical


@pytest.mark.parametrize("size", ["77", "large"])
@pytest.mark.parametrize("shape", SHAPES, ids=_id)
def test_vpg_gradient_on_weights(dev, n_sm, shape, size):
    """b200rl_grad(LOSS_VPG) with adv := w (the REPS policy loss) against oracle grad_surr(..., "vpg") on the weights."""
    ops, L = _ops(), _L()
    c = _case(dev, n_sm, shape, size, masked=True)
    view = copy.copy(c.b)                   # the shared case keeps its own rew / tstep / adv
    rng = np.random.RandomState(11)
    view.rew = torch.tensor(rng.rand(1, c.B).astype(np.float32) * 3.0 - 1.0, device=dev)
    view.tstep = torch.zeros((1, c.B), dtype=torch.uint16, device=dev)
    view.adv = torch.zeros((1, c.B), dtype=torch.float32, device=dev)
    D = 2 * c.O + 4
    vd = torch.tensor(rng.randn(D) * 0.3, dtype=torch.float64, device=dev)
    M = torch.zeros(1, dtype=torch.float64, device=dev)
    sums = torch.zeros(D + 2, dtype=torch.float64, device=dev)
    ops.reps_delta_max(view, vd, M)
    ops.reps_dual_sums(view, vd, 2.0, M, sums, view.adv)
    w = view.adv.cpu().numpy().reshape(-1)
    assert (w[~c.keep] == 0).all()
    th = c.theta2()
    g = torch.zeros(c.dims.P, dtype=torch.float64, device=dev)
    ops.grad(L.LOSS_VPG, torch.tensor(th, dtype=torch.float32, device=dev), c.dd, 1e-6, view, g)
    batch = c.batch()
    batch["adv"] = w[c.keep].astype(np.float64)
    _assert_grad(g.cpu().numpy(), P.grad_surr(th, batch, c.dims, "vpg"))


# ------------------------------------------------------------------------------------------- host class
def _make(env_name):
    import bench
    return bench.make_env(env_name)


def _algo(n_envs, T, n_itr=3, hidden=32, env_name="cartpole", **kw):
    from rllab_b200.algos.reps import REPS
    from rllab_b200.baselines.linear_feature_baseline import LinearFeatureBaseline
    from rllab_b200.policies.gaussian_mlp_policy import GaussianMLPPolicy
    env = _make(env_name)
    policy = GaussianMLPPolicy(env.spec, hidden_sizes=(hidden, hidden), seed=3)
    args = dict(env=env, policy=policy, baseline=LinearFeatureBaseline(env.spec), batch_size=n_envs * T,
                max_path_length=T, n_itr=n_itr, discount=0.99, sampler_args=dict(n_envs=n_envs, seed=7))
    args.update(kw)
    return REPS(**args)


@pytest.fixture(scope="module", autouse=True)
def _quiet(dev):
    from rllab_b200.misc import logger
    logger.set_quiet(True)


def _device_step(n_envs=2048, T=100, **kw):
    from rllab_b200.misc import logger
    np.random.seed(5)
    algo = _algo(n_envs, T, **kw)
    algo.start_worker()
    algo.init_opt()
    paths = algo.sampler.obtain_samples(0)
    sd = algo.sampler.process_samples(0, paths)
    start = (float(algo.param_eta), np.array(algo.param_v), algo.policy.get_param_values())
    b = sd.lane_batch
    adv_before = b.adv.clone()
    algo.optimize_policy(0, sd)
    assert torch.equal(b.adv, adv_before)                       # samples_data's advantages are untouched
    logger.dump_tabular(with_prefix=False)
    return algo, b, start, logger.get_last_table()


def _oracle_step(algo, b, start, **kw):
    t = b.to_numpy()
    keep = b.valid_mask()
    O, A = b.O, b.A
    fd = K.feat_diff_lanes(t["obs"], t["flags"], t["tstep"])[keep]
    batch = dict(obs=np.moveaxis(t["obs"], 0, -1)[keep].astype(np.float64),
                 actions=np.moveaxis(t["act"], 0, -1)[keep].astype(np.float64),
                 old_mean=np.moveaxis(t["mean"], 0, -1)[keep].astype(np.float64),
                 old_log_std=t["log_std"].astype(np.float64))
    dims = P.Dims(O, (algo.policy.h1, algo.policy.h2), A)
    return K.optimize_policy(start[0], start[1], start[2], batch, t["rew"][keep].astype(np.float64), fd, dims,
                             epsilon=algo.epsilon, l2_reg_dual=algo.L2_reg_dual, l2_reg_loss=algo.L2_reg_loss,
                             max_opt_itr=algo.max_opt_itr, min_std=algo.policy.min_std)


@pytest.mark.parametrize("max_opt_itr", [1, 2])
def test_short_step_matches_oracle(dev, max_opt_itr):
    """max_opt_itr 1 / 2 on a 2048 x 100 CartPole batch against the same step driven by the oracle's callables: eta and
    v within 1e-6 relative, theta within 1e-5 of max |theta|."""
    algo, b, start, tab = _device_step(max_opt_itr=max_opt_itr, L2_reg_loss=1e-2)
    ref = _oracle_step(algo, b, start)
    th = algo.policy.get_param_values()
    e_eta = abs(algo.param_eta - ref["eta"]) / abs(ref["eta"])
    e_v = np.max(np.abs(algo.param_v - ref["v"])) / np.max(np.abs(ref["v"]))
    e_th = np.max(np.abs(th - ref["theta"])) / np.max(np.abs(ref["theta"]))
    print("max_opt_itr %d: eta %.6g (oracle %.6g), rel errors eta %.3g v %.3g theta %.3g; dual evals %d, policy evals %d"
          % (max_opt_itr, algo.param_eta, ref["eta"], e_eta, e_v, e_th, algo.n_dual_evals, algo.n_policy_evals))
    assert e_eta < 1e-6 and e_v < 1e-6, (e_eta, e_v)
    assert e_th < 1e-5, e_th
    for key in ("DualBefore", "DualAfter"):
        assert tab[key] == pytest.approx(ref[key], rel=1e-9), key
    for key in ("LossBefore", "LossAfter", "MeanKL"):
        assert tab[key] == pytest.approx(ref[key], rel=1e-4, abs=1e-7), key


def test_default_settings_decrease_dual_and_loss(dev):
    algo, _, start, tab = _device_step()
    print("defaults: eta %.4g -> %.4g, dual %.6g -> %.6g, loss %.6g -> %.6g, MeanKL %.4g; %d dual / %d policy evals" %
          (start[0], algo.param_eta, tab["DualBefore"], tab["DualAfter"], tab["LossBefore"], tab["LossAfter"],
           tab["MeanKL"], algo.n_dual_evals, algo.n_policy_evals))
    for key in ("LossBefore", "LossAfter", "DualBefore", "DualAfter", "MeanKL"):
        assert np.isfinite(tab[key]), key
    assert tab["LossAfter"] <= tab["LossBefore"]
    assert tab["DualAfter"] <= tab["DualBefore"]


def _train_logged(algo, n):
    from rllab_b200.misc import logger
    algo.start_worker()
    algo.init_opt()
    tables = []
    for itr in range(n):
        algo.train_itr(itr)
        tables.append(logger.get_last_table())
    return tables


def test_reps_cartpole_learns(dev):
    np.random.seed(1)
    tables = _train_logged(_algo(256, 100, n_itr=10), 10)
    for t in tables:
        for k in ("LossBefore", "LossAfter", "DualBefore", "DualAfter", "MeanKL"):
            assert k in t and np.isfinite(t[k]), k
    r = [t["AverageReturn"] for t in tables]
    print("REPS CartPole AverageReturn", np.round(r, 2))
    assert np.mean(r[-3:]) > np.mean(r[:3])


def test_reps_hopper_runs(dev):
    np.random.seed(2)
    algo = _algo(256, 100, n_itr=2, hidden=64, env_name="hopper")
    for t in _train_logged(algo, 2):
        for k in ("LossBefore", "LossAfter", "DualBefore", "DualAfter", "MeanKL", "AverageReturn"):
            assert np.isfinite(t[k]), k
    assert np.isfinite(algo.policy.get_param_values()).all()
    assert np.isfinite(algo.param_eta) and np.isfinite(algo.param_v).all()


def test_reps_snapshot_and_resume(dev, tmp_path):
    from rllab_b200.misc import logger
    logger.set_snapshot_dir(str(tmp_path))
    logger.set_snapshot_mode("last")
    try:
        np.random.seed(3)
        algo = _algo(256, 50, n_itr=2)
        algo.train()
        data = pickle.load(open(str(tmp_path / "params.pkl"), "rb"))
    finally:
        logger.set_snapshot_mode("none")
        logger.set_snapshot_dir(None)
    resumed = data["algo"]
    assert resumed.param_eta == algo.param_eta and np.array_equal(resumed.param_v, algo.param_v)
    resumed.n_itr = 3
    resumed.train()
    np.random.seed(3)
    algo3 = _algo(256, 50, n_itr=3)
    algo3.train()
    np.testing.assert_array_equal(resumed.policy.get_param_values(), algo3.policy.get_param_values())
    assert resumed.param_eta == algo3.param_eta and np.array_equal(resumed.param_v, algo3.param_v)
