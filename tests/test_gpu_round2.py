"""GPU parity tests added in round 2: whole-path masking, the time-parallel process_samples scan at awkward sizes,
FiniteDifferenceHvp / subsample_factor / TNPG, full-episode planar dynamics with per-step re-synchronisation, the
end-to-end TRPO train loop on the Swimmer (32,32) and Hopper (64,64) configurations, and the learning-curve comparison
with the committed float64 oracle curves."""
import json
import os

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from oracle import envs as E            # noqa: E402
from oracle import optim as OPT         # noqa: E402
from oracle import policy as P          # noqa: E402
from oracle import sampler as S         # noqa: E402
import planar_tree_oracle as TREE       # noqa: E402

from test_gpu_kernels import _L, _close_frac, _gpu_rollout, _ops, _stats_from_device   # noqa: E402
from test_gpu_algos import _algo, _rel, _trpo_setup                                    # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from rllab_b200 import _lib
    _lib.load()
    from rllab_b200.misc import logger
    logger.set_quiet(True)
    return torch.device("cuda:0")


# ------------------------------------------------------------------------------------------- process_samples
@pytest.mark.parametrize("N,T,mpl", [(1, 5, 3), (33, 7, 3), (200, 64, 64), (70, 65, 20), (257, 130, 41), (40, 500, 500),
                                     (96, 129, 500)])
@pytest.mark.parametrize("drop", [False, True])
def test_process_samples_scan_shapes(dev, N, T, mpl, drop):
    """The chunked two-pass scan (8 warps x 8 steps per window) against the oracle's plain reverse loop: window /
    chunk boundaries that do not divide T, lanes that do not fill a warp, paths that span several windows, and (drop) the
    whole-paths mask carried across chunks."""
    ops = _ops()
    env, dims, theta, b, eps, rr = _gpu_rollout("cartpole", 32, N, T, mpl, dev)
    traj = b.to_numpy()
    w = np.random.RandomState(5).randn(2 * env.O + 4) * 0.3
    ops.process_samples(b, torch.tensor(w, dtype=torch.float64, device=dev), 0.99, 0.95, drop_cut_paths=drop)
    ref = S.process_samples_lanes(traj, w, 0.99, 0.95, center_adv=True, drop_cut=drop)
    valid = ref["valid"]
    np.testing.assert_allclose(b.ret.cpu().numpy(), ref["ret"], rtol=1e-5, atol=1e-4)
    np.testing.assert_allclose(b.base.cpu().numpy(), ref["base"], rtol=1e-5, atol=1e-4)
    np.testing.assert_allclose(b.adv.cpu().numpy(), ref["adv_raw"], rtol=1e-5, atol=2e-4)
    fl = b.flags.cpu().numpy()
    assert np.array_equal((fl & 8) != 0, ~valid)                          # FLAG_MASKED exactly on the dropped samples
    assert np.array_equal(fl & 7, traj["flags"] & 7)                      # the other bits are untouched
    st = _stats_from_device(b)
    assert st["NumTrajs"] == ref["stats"]["NumTrajs"]
    assert int(round(float(b.count.cpu()[0]))) == int(valid.sum())
    for key in ("AverageDiscountedReturn", "AverageReturn", "StdReturn", "MaxReturn", "MinReturn", "adv_mean", "adv_std"):
        np.testing.assert_allclose(st[key], ref["stats"][key], rtol=1e-6, atol=1e-6, err_msg=key)
    ops.center_advantages(b, True, False)
    np.testing.assert_allclose(b.adv.cpu().numpy(), ref["adv"], rtol=1e-4, atol=2e-5)


def test_whole_paths_masking_through_update_passes(dev):
    """Dropped (cut) paths contribute nothing to the baseline normal equations, loss / KL, gradient and Fisher-vector
    product, and every mean is over the valid samples (device-resident count): kernels on the masked lane batch ==
    oracle on the batch with the dropped samples removed."""
    ops, L = _ops(), _L()
    N, T, mpl = 300, 50, 50
    for hidden in (32, 64):
        env, dims, theta, b, eps, rr = _gpu_rollout("cartpole", hidden, N, T, mpl, dev)
        traj = b.to_numpy()
        ops.process_samples(b, None, 0.99, 1.0, drop_cut_paths=True)
        ops.center_advantages(b, True, False)
        ref = S.process_samples_lanes(traj, None, 0.99, 1.0, center_adv=True, drop_cut=True)
        valid = ref["valid"]
        assert 0.02 < (~valid).mean() < 0.9                                  # the case has a real share of cut paths
        np.testing.assert_allclose(b.adv.cpu().numpy(), ref["adv"], rtol=1e-4, atol=2e-5)
        batch = S.batch_from_traj(traj, b.adv.cpu().numpy(), valid)      # the device's own (float32) advantages
        d1 = 2 * b.O + 5
        ops.lfb_gram(b, b.gram)
        F = S.lfb_features_lanes(traj["obs"], traj["tstep"]).reshape(d1 - 1, -1)
        F = np.concatenate([F, ref["ret"].reshape(1, -1)], axis=0)[:, valid.reshape(-1)]
        np.testing.assert_allclose(b.gram.cpu().numpy(), (F @ F.T)[np.triu_indices(d1)], rtol=2e-5, atol=1e-3)
        dd = (env.O, hidden, hidden, env.A)
        th32 = torch.tensor(theta, dtype=torch.float32, device=dev)
        th2 = theta + 0.02 * np.random.RandomState(9).randn(dims.P)
        th2_32 = torch.tensor(th2, dtype=torch.float32, device=dev)
        th2 = th2_32.double().cpu().numpy()
        out = torch.zeros(3, dtype=torch.float64, device=dev)
        ops.loss_kl(L.LOSS_TRPO, th2_32, dd, 1e-6, b, out)
        o = out.cpu().numpy()
        np.testing.assert_allclose(o[0], P.surr_loss_trpo(th2, batch, dims), rtol=2e-5, atol=1e-7)
        np.testing.assert_allclose(o[1:], P.kl_stats(th2, batch, dims), rtol=2e-4)
        g = torch.zeros(dims.P, dtype=torch.float64, device=dev)
        hc = b.hcache(hidden, hidden)
        ops.grad(L.LOSS_TRPO, th2_32, dd, 1e-6, b, g, out, None)
        ref_g = P.grad_surr(th2, batch, dims, "trpo")
        np.testing.assert_allclose(g.cpu().numpy(), ref_g, rtol=0, atol=2e-4 * np.abs(ref_g).max())
        np.testing.assert_allclose(out.cpu().numpy()[0], P.surr_loss_trpo(th2, batch, dims), rtol=2e-5, atol=1e-7)
        x = np.random.RandomState(4).randn(dims.P)
        xd = torch.tensor(x, dtype=torch.float64, device=dev)
        ref_H = P.fvp(theta, batch, xd.float().double().cpu().numpy(), dims, 0.0) + 1e-5 * x
        for cache in (None, hc):
            if cache is not None:
                ops.grad(L.LOSS_TRPO, th32, dd, 1e-6, b, g, None, cache)
            Hx = torch.zeros_like(g)
            ops.fvp(th32, dd, 1e-6, b, xd, 1e-5, 1.0, Hx, cache)
            np.testing.assert_allclose(Hx.cpu().numpy(), ref_H, rtol=0, atol=2e-4 * np.abs(ref_H).max())
        # float64 parity kernels honour the mask as well
        out64 = torch.zeros(3, dtype=torch.float64, device=dev)
        g64 = torch.zeros_like(g)
        ops.update_f64(1, L.LOSS_TRPO, torch.tensor(th2, dtype=torch.float64, device=dev), dd, 1e-6, b, None, 0.0, 0.0,
                       g64, out64)
        np.testing.assert_allclose(g64.cpu().numpy(), ref_g, rtol=1e-7, atol=1e-9 * np.abs(ref_g).max())


def test_whole_paths_false_keeps_truncated_paths(dev):
    """whole_paths=False (batch_polopt.py:30-34 -> truncate_paths): the path cut by the end of the lane buffer stays in
    the batch as a truncated path; every (t, lane) cell is a sample."""
    from rllab_b200.misc import logger
    a_true = _algo("cartpole", "vpg", 256, 50)
    a_false = _algo("cartpole", "vpg", 256, 50, whole_paths=False)
    tabs = []
    for algo in (a_true, a_false):
        algo.start_worker()
        algo.init_opt()
        paths = algo.sampler.obtain_samples(0)
        sd = algo.sampler.process_samples(0, paths)
        logger.dump_tabular()
        tabs.append((sd, logger.get_last_table(), paths))
    (sd_t, tab_t, p_t), (sd_f, tab_f, p_f) = tabs
    bt, bf = sd_t.lane_batch, sd_f.lane_batch
    assert torch.equal(bt.obs, bf.obs)                                     # same seeds -> same rollout
    cut = (bt.flags.cpu().numpy()[-1] & 4) != 0
    assert cut.any()
    assert tab_f["NumTrajs"] == tab_t["NumTrajs"] + int(cut.sum())
    assert bf.valid_mask().all() and not bt.valid_mask().all()
    assert len(sd_f["rewards"]) == bf.B and len(sd_t["rewards"]) == int(bt.valid_mask().sum())
    assert len(p_f.to_paths()) == len(p_t.to_paths()) + int(cut.sum())
    assert sum(len(p["rewards"]) for p in p_f.to_paths()) == bf.B


# ------------------------------------------------------------------------------------------- optimizer variants
def test_finite_difference_hvp_matches_oracle(dev):
    """FiniteDifferenceHvp (conjugate_gradient_optimizer.py:58-115): (grad_kl(theta + eps x) - grad_kl(theta - eps x)) /
    (2 eps) + reg x with eps = base_eps / |theta|, float64 kernels, against the oracle's closed-form product and
    against the same finite difference taken on the oracle."""
    from rllab_b200 import ops
    from rllab_b200.optimizers.conjugate_gradient_optimizer import FiniteDifferenceHvp
    algo, sd, theta0, batch, dims = _trpo_setup("cartpole", 32, 2, hvp_approach=FiniteDifferenceHvp())
    b, pol, opt = sd.lane_batch, algo.policy, algo.optimizer
    theta = pol.get_param_values()
    bufs = opt._buffers(pol.n_params, b.device)
    Hx = opt._make_Hx(b, bufs, None, None)
    x = np.random.RandomState(1).randn(dims.P)
    xd = torch.tensor(x, dtype=torch.float64, device=b.device)
    out = torch.zeros_like(xd)
    Hx(xd, out)
    ref = P.fvp(theta, batch, x, dims, 1e-5)
    # base_eps = 1e-8 in float64: truncation ~ eps^2, rounding ~ 1e-16 / eps ~ 1e-7 relative
    np.testing.assert_allclose(out.cpu().numpy(), ref, rtol=0, atol=5e-6 * np.abs(ref).max())
    # ... and the whole TRPO step with this product accepts like the oracle's
    algo.optimize_policy(0, sd)
    theta_ref, info = OPT.trpo_step(theta, batch, dims, step_size=0.01, cg_iters=2)
    li = opt.last_info
    assert li["n_iter"] == info["n_iter"] and not li["rejected"]
    assert _rel(pol.get_param_values(), theta_ref) < 1e-4


def test_subsample_factor_fvp_matches_oracle_on_the_subset(dev):
    """subsample_factor < 1 (conjugate_gradient_optimizer.py:235-245): the Fisher-vector products run on a random subset
    (np.random.choice, drawn per 128-sample tile), the mean is over the valid samples of the subset."""
    from rllab_b200 import ops
    np.random.seed(11)
    algo, sd, theta0, batch_full, dims = _trpo_setup("cartpole", 32, 3, subsample_factor=0.3)
    b, pol, opt = sd.lane_batch, algo.policy, algo.optimizer
    bufs = opt._buffers(pol.n_params, b.device)
    tiles = opt._draw_subsample(b, bufs)
    inds = opt.last_subsample
    n_tiles = -(-b.B // 128)
    assert len(inds) == int(n_tiles * 0.3) and len(set(inds.tolist())) == len(inds)
    sel = np.zeros(n_tiles * 128, dtype=bool)
    for t in inds:
        sel[t * 128:(t + 1) * 128] = True
    sel = sel[:b.B].reshape(b.T, b.N) & b.valid_mask()
    assert int(round(float(bufs["cnt"].cpu()[0]))) == int(sel.sum())
    sub = S.batch_from_traj(b.to_numpy(), b.adv.cpu().numpy(), sel)
    x = np.random.RandomState(2).randn(dims.P)
    xd = torch.tensor(x, dtype=torch.float64, device=b.device)
    Hx = opt._make_Hx(b, bufs, None, tiles)
    out = torch.zeros_like(xd)
    Hx(xd, out)
    ref = P.fvp(theta0, sub, xd.float().double().cpu().numpy(), dims, 0.0) + 1e-5 * x
    np.testing.assert_allclose(out.cpu().numpy(), ref, rtol=0, atol=2e-4 * np.abs(ref).max())
    algo.optimize_policy(0, sd)                     # and the full step runs with a fresh subset
    assert not opt.last_info["rejected"] and 0 < opt.last_info["constraint_val"] <= 0.01


def test_tnpg_is_trpo_with_one_backtrack(dev):
    """rllab/algos/tnpg.py:17: ConjugateGradientOptimizer(max_backtracks=1) -- only the full natural-gradient step is
    tried; the update equals the oracle's with the same setting."""
    from rllab_b200.algos.trpo import TNPG
    from rllab_b200.baselines.linear_feature_baseline import LinearFeatureBaseline
    from rllab_b200.policies.gaussian_mlp_policy import GaussianMLPPolicy
    import bench
    env = bench.make_env("cartpole")
    policy = GaussianMLPPolicy(env.spec, hidden_sizes=(32, 32), seed=3)
    algo = TNPG(env=env, policy=policy, baseline=LinearFeatureBaseline(env.spec), batch_size=1024 * 50, max_path_length=50,
                n_itr=1, discount=0.99, step_size=0.01, optimizer_args=dict(cg_iters=4),
                sampler_args=dict(n_envs=1024, seed=7))
    assert algo.optimizer._max_backtracks == 1
    algo.start_worker()
    algo.init_opt()
    paths = algo.sampler.obtain_samples(0)
    sd = algo.sampler.process_samples(0, paths)
    b = sd.lane_batch
    theta0 = policy.theta32.double().cpu().numpy()
    batch = S.batch_from_traj(b.to_numpy(), b.adv.cpu().numpy(), b.valid_mask())
    dims = P.Dims(b.O, (32, 32), b.A)
    algo.optimize_policy(0, sd)
    theta_ref, info = OPT.trpo_step(theta0, batch, dims, step_size=0.01, cg_iters=4, max_backtracks=1)
    li = algo.optimizer.last_info
    assert li["n_iter"] == 0 and li["rejected"] == info["rejected"]
    assert _rel(policy.get_param_values(), theta_ref) < 1e-5


# ------------------------------------------------------------------------------------------- planar envs, full episodes
PLANAR_EPISODES = [("hopper", 500), ("swimmer", 200), ("half_cheetah", 1000)]


@pytest.mark.parametrize("env_name,steps", PLANAR_EPISODES)
def test_planar_full_episode_with_resync(dev, env_name, steps):
    """Device env.step against the float32 oracle over whole episodes (Hopper: 500 steps including ground contact, falls
    and the auto-reset that follows `done`; HalfCheetah: the float32 tree oracle over its 1000-step benchmark horizon),
    with the oracle re-synchronised to the device state every step so that the comparison is of ONE step of dynamics at
    a time (the chains are chaotic in float32).  Some lane-steps must have active contact rows in the oracle (limit
    rows on Swimmer, which has no contacts)."""
    ops, L = _ops(), _L()
    env32 = TREE.make(env_name, np.float32) if env_name == "half_cheetah" else E.make(env_name, np.float32)
    nq = env32.m.n + 2
    n_lim = 2 * sum(lim is not None for lim in env32.m.limits)        # constraint_residuals: limit rows, then contacts
    kind = L.ENV_KINDS[env_name]
    N = 256
    rng = np.random.RandomState(0)
    raw = rng.randn(env32.K, N).astype(np.float32)
    state = torch.empty((env32.S, N), dtype=torch.float32, device=dev)
    obs = torch.empty((env32.O, N), dtype=torch.float32, device=dev)
    rew = torch.empty((N,), dtype=torch.float32, device=dev)
    done = torch.empty((N,), dtype=torch.uint8, device=dev)
    ops.env_reset(kind, N, state, obs, torch.tensor(raw, device=dev))
    s = env32.reset(raw)
    n_done = 0
    worst_obs = worst_rew = 0.0
    n_constrained = 0
    for t in range(steps):
        # the oracle's active rows at the step's input state: a negative residual
        res = TREE.constraint_residuals(env32.m, list(s[:nq]), np.float32)
        n_constrained += int(((res[n_lim:] if env32.m.contacts else res) < 0).any(axis=0).sum())
        a = (rng.randn(env32.A, N) * 0.5).astype(np.float32)
        ops.env_step(kind, N, state, torch.tensor(a, device=dev), obs, rew, done)
        s, r, d = env32.step(s, env32.scale_action(a))
        o_dev, o_ref = obs.cpu().numpy(), env32.obs(s)
        _close_frac(o_dev, o_ref, 4e-3, 1e-3, 0.995)
        _close_frac(rew.cpu().numpy(), r, 4e-3, 1e-2, 0.995)
        dd = done.cpu().numpy().astype(bool)
        assert (dd != d).mean() < 0.02, (t, (dd != d).mean())
        # re-sync; lanes that finished start a new episode on both sides (vec_env_executor.py:14-26)
        s = state.cpu().numpy()
        if dd.any():
            n_done += int(dd.sum())
            fresh_raw = rng.randn(env32.K, N).astype(np.float32)
            fresh = env32.reset(fresh_raw)
            s = np.where(dd[None], fresh, s).astype(np.float32)
            state.copy_(torch.tensor(s, device=dev))
    assert n_constrained > 0                             # the body touches the ground (Swimmer: reaches a limit)
    if env_name == "hopper":
        assert n_done > N // 4                           # episodes end (falls)


# ------------------------------------------------------------------------------------------- cfg3 / cfg4 end to end
@pytest.mark.parametrize("env_name,hidden,lanes", [("swimmer", 32, 512), ("hopper", 64, 512)])
def test_trpo_train_loop_planar(dev, env_name, hidden, lanes):
    """BASELINE.json configs[2] / configs[3] through the plugin API (examples/trpo_swimmer.py:17-26 shape): TRPO with
    cg_iters=10, LinearFeatureBaseline, horizon 500; finite parameters, accepted steps, KL within the trust region, the
    reference's tabular keys, and a return that moves the right way within a few iterations."""
    from rllab_b200.misc import logger
    algo = _algo(env_name, "trpo", lanes, 500, hidden, n_itr=4, step_size=0.01)
    algo.start_worker()
    algo.init_opt()
    rets, kls = [], []
    for itr in range(4):
        algo.train_itr(itr)
        tab = logger.get_last_table()
        rets.append(tab["AverageReturn"]), kls.append(tab["MeanKL"])
        assert not algo.optimizer.last_info["rejected"]
        assert tab["LossAfter"] < tab["LossBefore"]
    assert np.all(np.isfinite(algo.policy.get_param_values()))
    assert all(0 < k <= 0.01 for k in kls), kls
    assert rets[-1] > rets[0], rets
    if env_name == "swimmer":
        assert tab["NumTrajs"] == lanes                   # never done: one whole path per lane, nothing dropped
    else:
        assert tab["NumTrajs"] > lanes                    # early terminations -> several whole paths per lane


def _curve(env_name, n_itr, precision="f32"):
    from rllab_b200.algos.trpo import TRPO
    from rllab_b200.baselines.linear_feature_baseline import LinearFeatureBaseline
    from rllab_b200.misc import logger
    from rllab_b200.policies.gaussian_mlp_policy import GaussianMLPPolicy
    import bench
    gold = json.load(open(os.path.join(ROOT, "tests", "golden", "oracle_%s_trpo_curve.json" % env_name)))
    cfg, curve = gold["config"], gold["curve"]
    env = bench.make_env(env_name)
    policy = GaussianMLPPolicy(env.spec, hidden_sizes=tuple(cfg["hidden"]), seed=cfg["policy_seed"])
    algo = TRPO(env=env, policy=policy, baseline=LinearFeatureBaseline(env.spec),
                batch_size=cfg["lanes"] * cfg["horizon"], max_path_length=cfg["horizon"], n_itr=n_itr,
                discount=cfg["discount"], gae_lambda=cfg["gae_lambda"], step_size=cfg["step_size"], whole_paths=False,
                optimizer_args=dict(cg_iters=cfg["cg_iters"], precision=precision),
                sampler_args=dict(n_envs=cfg["lanes"], seed=cfg["seed"]))
    algo.start_worker()
    algo.init_opt()
    rets = []
    for itr in range(n_itr):
        algo.train_itr(itr)
        rets.append(logger.get_last_table()["AverageReturn"])
    return np.array(rets), np.array([c["AverageReturn"] for c in curve[:n_itr]])


def test_hopper_learning_curve_matches_oracle(dev):
    """north_star's learning check on cfg4's net: TRPO on Hopper (64,64), same lanes / horizon / Philox keys / initial
    policy as tests/golden/oracle_hopper_trpo_curve.json (float64 oracle, 40 iterations of 512 000 samples).  Iteration 0
    sees identical noise -> AverageReturn agrees to the planar-dynamics tolerance; the tail (mean of the last 5
    iterations) agrees within +-5 %."""
    gpu, ref = _curve("hopper", 40)
    assert abs(gpu[0] - ref[0]) < 0.02 * abs(ref[0]) + 0.05, (gpu[0], ref[0])
    tail_gpu, tail_ref = gpu[-5:].mean(), ref[-5:].mean()
    assert abs(tail_gpu / tail_ref - 1.0) < 0.05, (tail_gpu, tail_ref)
    assert gpu[-1] > 20 * gpu[0]                          # it learns: 5 -> ~250


def test_swimmer_learning_curve_matches_oracle(dev):
    """The same check on cfg3 (Swimmer, (32,32)) with the shipped float32 path (deterministic: same inputs -> same curve).
    Iteration 0: identical noise -> AverageReturn within the planar tolerance; the first iterations track the oracle.
    The tail does NOT reach the float64 oracle's return at iteration 40: the learning speed of TRPO on this task grows with
    the effective depth of the CG solve, and the float32 Fisher-vector product costs the 10-iteration solve about three
    iterations of depth.  Measured over 8 sampler seeds (scripts/exp_seed_sweep.py, DESIGN.md section 5): float32 kernels
    23.7 +- 2.7, float64 parity kernels 30.5 +- 1.5, float64 with cg_iters=6 21.1 +- 1.4, float32 with cg_iters=20
    36.0 +- 5.3; oracle 31.0 / 31.6 / 32.1 on its three seeds.  The band below is what the float32 path supports; the
    float64 parity kernels (which accumulate with shared-memory atomics and are therefore not run-to-run deterministic on
    a chaotic 40-iteration trajectory) are inside +-12 % of the oracle on most seeds."""
    gpu, ref = _curve("swimmer", 40)
    assert abs(gpu[0] - ref[0]) < 0.02 * abs(ref[0]) + 0.05, (gpu[0], ref[0])
    assert np.all(np.abs(gpu[:8] - ref[:8]) < 1.5), (gpu[:8], ref[:8])       # the first iterations track the oracle
    tail_gpu, tail_ref = gpu[-5:].mean(), ref[-5:].mean()
    assert 0.62 < tail_gpu / tail_ref < 1.15, (tail_gpu, tail_ref)
    assert gpu[-1] > 20.0 and gpu[3] > 0.0               # -7 -> 23+: it learns to swim forward
