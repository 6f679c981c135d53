"""GPU: the plugin API (Env / Policy / Baseline / Sampler / BatchPolopt, TRPO and VPG) end to end, and the policy
update against the CPU oracle on the very same batch: parameters within 1e-5 relative (north_star tolerance)."""
import pickle

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from oracle import optim as OPT          # noqa: E402
from oracle import policy as P           # noqa: E402
from oracle import sampler as S          # noqa: E402

PARAM_RTOL = 1e-5


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from rllab_b200 import _lib
    _lib.load()
    from rllab_b200.misc import logger
    logger.set_quiet(True)
    return torch.device("cuda:0")


def _make(env_name):
    if env_name == "half_cheetah":                 # not one of bench.py's workloads
        from rllab_b200.envs.mujoco.half_cheetah_env import HalfCheetahEnv
        from rllab_b200.envs.normalized_env import normalize
        return normalize(HalfCheetahEnv())
    import bench
    return bench.make_env(env_name)


def _algo(env_name, algo_name, n_envs, T, hidden=32, **kw):
    from rllab_b200.algos.trpo import TRPO
    from rllab_b200.algos.vpg import VPG
    from rllab_b200.baselines.linear_feature_baseline import LinearFeatureBaseline
    from rllab_b200.policies.gaussian_mlp_policy import GaussianMLPPolicy
    env = _make(env_name)
    policy = GaussianMLPPolicy(env.spec, hidden_sizes=(hidden, hidden), seed=3)
    baseline = LinearFeatureBaseline(env.spec)
    args = dict(env=env, policy=policy, baseline=baseline, batch_size=n_envs * T, max_path_length=T, n_itr=3,
                discount=0.99, sampler_args=dict(n_envs=n_envs, seed=7))
    args.update(kw)
    return (TRPO(**args) if algo_name == "trpo" else VPG(**args))


def _rel(a, b):
    return np.max(np.abs(a - b)) / np.max(np.abs(b))


def _trpo_setup(env_name, hidden, cg_iters, **opt_args):
    algo = _algo(env_name, "trpo", 1024, 50, hidden, optimizer_args=dict(cg_iters=cg_iters, **opt_args))
    algo.start_worker()
    algo.init_opt()
    paths = algo.sampler.obtain_samples(0)
    sd = algo.sampler.process_samples(0, paths)
    b = sd.lane_batch
    theta0 = algo.policy.theta32.double().cpu().numpy()
    batch = S.batch_from_traj(b.to_numpy(), b.adv.cpu().numpy(), b.valid_mask())      # whole paths only (default)
    dims = P.Dims(b.O, (hidden, hidden), b.A)
    return algo, sd, theta0, batch, dims


@pytest.mark.parametrize("env_name,hidden,cg_iters", [("cartpole", 32, 1), ("cartpole", 32, 4), ("point", 32, 4),
                                                      ("pendulum", 32, 4), ("cartpole", 64, 4),
                                                      ("swimmer", 32, 4), ("hopper", 64, 4), ("hopper", 32, 4)])
def test_trpo_update_matches_oracle(dev, env_name, hidden, cg_iters):
    """Whole TRPO step (grad -> CG -> step size -> line search) against the float64 oracle on the same batch.
    cg_iters=1 is the reference's own test setting (tests/test_algos.py:51); 4 keeps CG inside the regime where a
    float32 Hessian-vector product (rel. error ~1e-7) is not amplified past the 1e-5 parameter tolerance -- with the
    default 10 iterations CG on this ill-conditioned system (kappa ~ 1e5) amplifies 1e-8 perturbations to O(1)
    (DESIGN.md "Parity limits"), which test_trpo_default_cg_iters_behaviour covers instead."""
    algo, sd, theta0, batch, dims = _trpo_setup(env_name, hidden, cg_iters)
    algo.optimize_policy(0, sd)
    theta_dev = algo.policy.get_param_values()
    theta_ref, info = OPT.trpo_step(theta0, batch, dims, step_size=0.01, cg_iters=cg_iters)
    li = algo.optimizer.last_info
    assert li["n_iter"] == info["n_iter"] and li["rejected"] == info["rejected"]      # index work: identical
    assert not info["rejected"]
    assert _rel(theta_dev, theta_ref) < PARAM_RTOL, _rel(theta_dev, theta_ref)
    np.testing.assert_allclose(li["loss_before"], info["loss_before"], rtol=1e-4, atol=1e-7)
    np.testing.assert_allclose(li["loss"], info["loss"], rtol=1e-4, atol=1e-7)
    np.testing.assert_allclose(li["constraint_val"], info["constraint_val"], rtol=2e-4)
    assert 0 < li["constraint_val"] <= 0.01


def test_trpo_default_cg_iters_behaviour(dev):
    """cg_iters=10 (the default): the device and the float64 oracle solve H x = g to a comparable residual, and both
    accepted steps satisfy the reference's acceptance test (loss decreased, KL <= delta)."""
    from rllab_b200 import ops
    algo, sd, theta0, batch, dims = _trpo_setup("cartpole", 32, 10)
    b, pol, opt = sd.lane_batch, algo.policy, algo.optimizer
    algo.optimize_policy(0, sd)
    li = opt.last_info
    assert not li["rejected"] and li["loss"] < li["loss_before"] and 0 < li["constraint_val"] <= 0.01
    theta_ref, info = OPT.trpo_step(theta0, batch, dims, step_size=0.01, cg_iters=10)
    assert not info["rejected"]
    # the device's accepted parameters, evaluated by the ORACLE, also pass the acceptance test with the same numbers
    th_dev = pol.theta32.double().cpu().numpy()
    np.testing.assert_allclose(P.surr_loss_trpo(th_dev, batch, dims), li["loss"], rtol=1e-4, atol=1e-7)
    np.testing.assert_allclose(P.kl_stats(th_dev, batch, dims)[0], li["constraint_val"], rtol=2e-4)
    # CG quality: relative residual of the device solution (float64 oracle matvec) within 10x of the oracle's
    g = P.grad_surr(theta0, batch, dims, "trpo")
    x_dev = opt._bufs["x"].cpu().numpy()
    res = lambda x: np.linalg.norm(P.fvp(theta0, batch, x, dims, 1e-5) - g) / np.linalg.norm(g)
    assert res(x_dev) < max(10 * res(info["descent_direction"]), 0.2), (res(x_dev), res(info["descent_direction"]))
    # improvement per unit KL comparable
    assert abs(li["loss"]) > 0.5 * abs(info["loss"]) * li["constraint_val"] / info["constraint_val"]


@pytest.mark.parametrize("env_name", ["cartpole", "pendulum"])
def test_vpg_updates_match_oracle(dev, env_name):
    algo = _algo(env_name, "vpg", 1024, 50)
    algo.start_worker()
    algo.init_opt()
    dims = None
    adam = None
    theta_ref = None
    for itr in range(3):                      # Adam moments / step counter persist across iterations
        paths = algo.sampler.obtain_samples(itr)
        sd = algo.sampler.process_samples(itr, paths)
        b = sd.lane_batch
        if dims is None:
            dims = P.Dims(b.O, (32, 32), b.A)
            adam = (np.zeros(dims.P), np.zeros(dims.P), 0)
        theta0 = algo.policy.get_param_values()
        batch = S.batch_from_traj(b.to_numpy(), b.adv.cpu().numpy(), b.valid_mask())
        # the kernels see float32(theta); hand the oracle the same numbers
        th32 = algo.policy.theta32.double().cpu().numpy()
        g_ref = P.grad_surr(th32, batch, dims, "vpg")
        theta_ref, m, v, t = P.adam_step(theta0, g_ref, adam[0], adam[1], adam[2])
        adam = (m, v, t)
        algo.optimize_policy(itr, sd)
        theta_dev = algo.policy.get_param_values()
        assert _rel(theta_dev, theta_ref) < PARAM_RTOL, (itr, _rel(theta_dev, theta_ref))
        algo.policy.set_param_values(theta_ref)     # keep both sides on the same trajectory of parameters


@pytest.mark.parametrize("algo_name", ["trpo", "vpg"])
def test_train_loop_runs_and_logs(dev, algo_name):
    """Mirror of the reference's integration smoke (tests/test_algos.py:28-94): a few iterations, no NaN params,
    plus the tabular keys of sampler/base.py:170-180 and npo.py:118-122 / vpg.py:124-130."""
    from rllab_b200.misc import logger
    algo = _algo("cartpole", algo_name, 512, 100, n_itr=2)
    algo.train()
    assert not np.any(np.isnan(algo.policy.get_param_values()))
    tab = logger.get_last_table()
    keys = ["Iteration", "AverageDiscountedReturn", "AverageReturn", "ExplainedVariance", "NumTrajs", "Entropy",
            "Perplexity", "StdReturn", "MaxReturn", "MinReturn", "AveragePolicyStd", "LossBefore", "LossAfter", "MeanKL"]
    keys += ["MeanKLBefore", "dLoss"] if algo_name == "trpo" else ["MaxKL"]
    for k in keys:
        assert k in tab, k
    assert tab["Iteration"] == 1 and tab["NumTrajs"] >= 512
    assert abs(tab["Entropy"] - 1.41894) < 0.05          # docs/user/experiments.rst:88 at init (log_std ~ 0, A = 1)
    assert algo.current_itr == 2


def test_trpo_improves_cartpole_return(dev):
    algo = _algo("cartpole", "trpo", 2048, 100, n_itr=12)
    from rllab_b200.misc import logger
    rets = []
    algo.start_worker()
    algo.init_opt()
    for itr in range(12):
        algo.train_itr(itr)
        rets.append(logger.get_last_table()["AverageReturn"])
    assert rets[-1] > 2.0 * rets[0], rets


def test_samples_data_wire_format(dev):
    algo = _algo("point", "trpo", 64, 30)
    algo.start_worker()
    algo.init_opt()
    paths = algo.sampler.obtain_samples(0)
    sd = algo.sampler.process_samples(0, paths)
    b = sd.lane_batch
    valid = b.valid_mask().reshape(-1)               # whole paths only: the samples of cut paths are not samples
    nv = int(valid.sum())
    assert 0 < nv <= b.B == 64 * 30
    assert sd["observations"].shape == (nv, 2) and sd["actions"].shape == (nv, 2)
    assert sd["advantages"].shape == (nv,) and sd["agent_infos"]["mean"].shape == (nv, 2)
    assert sd["agent_infos"]["log_std"].shape == (nv, 2)
    np.testing.assert_array_equal(sd["observations"], b.obs.cpu().numpy().reshape(2, -1).T.astype(np.float64)[valid])
    plist = sd["paths"]
    assert sum(len(p["rewards"]) for p in plist) == nv
    assert abs(sd["advantages"].mean()) < 1e-5 and abs(sd["advantages"].std() - 1) < 1e-3      # centered
    p0 = plist[0]
    assert set(p0) >= {"observations", "actions", "rewards", "agent_infos", "env_infos", "advantages", "returns"}
    np.testing.assert_allclose(p0["returns"], S.discount_cumsum(p0["rewards"], 0.99), rtol=1e-5, atol=1e-5)


PROTOCOL_ENVS = ["point", "cartpole", "pendulum", "cartpole_swingup", "double_pendulum", "swimmer", "hopper",
                 "half_cheetah"]


@pytest.mark.parametrize("env_name", PROTOCOL_ENVS)
def test_env_protocol(dev, env_name):
    """tests/envs/test_envs.py:86-102: reset in obs space, action in action space, one step, scalar reward."""
    env = _make(env_name)
    ob_space, act_space = env.observation_space, env.action_space
    ob = env.reset()
    assert ob_space.contains(ob)
    a = act_space.sample()
    assert act_space.contains(a)
    res = env.step(a)
    assert ob_space.contains(res.observation) and np.isscalar(res.reward) and isinstance(res.done, bool)
    inner = env.wrapped_env
    lb, ub = inner.action_space.bounds
    inner.reset()
    r2 = inner.step(np.clip(lb + (a + 1.) * 0.5 * (ub - lb), lb, ub))     # un-normalised env takes wrapped-space actions
    assert ob_space.contains(r2.observation)
    env.terminate()


def test_vec_env_executor_semantics(dev):
    """sandbox/rocky/tf/envs/vec_env_executor.py:14-26: horizon cut and auto-reset."""
    env = _make("cartpole")
    vec = env.vec_env_executor(n_envs=16, max_path_length=5)
    obs = vec.reset()
    assert np.asarray(obs).shape == (16, 4) and vec.num_envs == 16
    for t in range(5):
        obs, rew, dones, infos = vec.step(np.zeros((16, 1)))
    assert dones.all() and (vec.ts == 0).all()               # every lane hit max_path_length on the 5th step
    assert np.all(np.abs(obs[:, 0]) <= 0.12 + 1e-6)           # returned obs is the reset obs (cartpole_env.py:31-42)


def test_policy_api_and_pickle(dev):
    from rllab_b200.policies.gaussian_mlp_policy import GaussianMLPPolicy
    env = _make("cartpole")
    pol = GaussianMLPPolicy(env.spec, seed=0)
    flat = pol.get_param_values()
    assert flat.shape == (1250,) and flat.dtype == np.float64
    a, info = pol.get_action(env.reset())
    assert a.shape == (1,) and set(info) == {"mean", "log_std"}
    acts, infos = pol.get_actions(np.zeros((7, 4)))
    assert acts.shape == (7, 1) and infos["mean"].shape == (7, 1) and np.allclose(infos["log_std"], 0.0)
    mu, _ = P.forward(pol.theta32.double().cpu().numpy(), np.zeros((7, 4)), P.Dims(4, (32, 32), 1))
    np.testing.assert_allclose(infos["mean"], mu, rtol=1e-5, atol=1e-6)
    pol.set_param_values(flat * 0.5)
    np.testing.assert_array_equal(pol.get_param_values(), flat * 0.5)
    pol2 = pickle.loads(pickle.dumps(pol))
    np.testing.assert_array_equal(pol2.get_param_values(), flat * 0.5)
    assert pol.distribution.entropy(dict(log_std=np.zeros((1, 1))))[0] == pytest.approx(1.41894, abs=1e-5)


@pytest.mark.parametrize("algo_name", ["trpo", "vpg"])
def test_snapshot_and_resume(dev, algo_name, tmp_path):
    """logger.save_itr_params + resume_from semantics (misc/logger.py:216-232, scripts/run_experiment_lite.py:111-115):
    a resumed run continues at current_itr with identical parameters (and Adam state) and produces the same next
    iterate as the uninterrupted run."""
    from rllab_b200.misc import logger
    logger.set_snapshot_dir(str(tmp_path))
    logger.set_snapshot_mode("last")
    try:
        algo = _algo("cartpole", algo_name, 256, 50, n_itr=2)
        algo.train()
        theta2 = algo.policy.get_param_values()
        data = pickle.load(open(str(tmp_path / "params.pkl"), "rb"))
    finally:
        logger.set_snapshot_mode("none")
        logger.set_snapshot_dir(None)
    assert data["itr"] == 1 and set(data) >= {"itr", "policy", "baseline", "env", "algo"}
    np.testing.assert_array_equal(data["policy"].get_param_values(), theta2)
    resumed = data["algo"]
    assert resumed.current_itr == 2
    resumed.n_itr = 3
    resumed.train()                      # runs exactly iteration 2
    # same three iterations in one process; train() re-runs init_opt on resume, which -- exactly like the reference,
    # where lasagne's Adam state lives in shared variables created by update_opt -- resets the optimizer state
    algo3 = _algo("cartpole", algo_name, 256, 50, n_itr=3)
    algo3.start_worker()
    algo3.init_opt()
    algo3.train_itr(0)
    algo3.train_itr(1)
    algo3.init_opt()
    algo3.train_itr(2)
    rel = np.max(np.abs(resumed.policy.get_param_values() - algo3.policy.get_param_values())) / \
        np.max(np.abs(algo3.policy.get_param_values()))
    assert rel < 1e-12, rel


@pytest.mark.parametrize("env_name,hidden,cg_iters,tol", [("cartpole", 32, 6, PARAM_RTOL), ("point", 32, 8, PARAM_RTOL),
                                                          ("cartpole", 64, 6, PARAM_RTOL), ("cartpole", 32, 8, 1e-4),
                                                          ("cartpole", 32, 10, 5e-3)])
def test_trpo_f64_mode_matches_oracle(dev, env_name, hidden, cg_iters, tol):
    """precision="f64": the whole TRPO step (reg 1e-5, 15 backtracks) against the float64 oracle on the same batch.
    6 CG iterations (8 on PointEnv): parameters within 1e-5 relative (the float32 path only reaches this up to 4
    iterations).  Beyond that the comparison itself becomes ill-posed -- a 1e-15 relative perturbation of Hx (one float64
    rounding; the parity kernels accumulate with float64 atomics, i.e. in a run-dependent order) moves the ORACLE's own
    result by 1e-6 at 8 iterations and 3e-5 at 10, 1e-13 by 4e-3 (tests/test_oracle_sensitivity.py) -- so 8 and 10
    iterations are held to the oracle's self-sensitivity, and the line-search index must still agree."""
    algo = _algo(env_name, "trpo", 1024, 50, hidden, optimizer_args=dict(cg_iters=cg_iters, precision="f64"))
    algo.start_worker()
    algo.init_opt()
    paths = algo.sampler.obtain_samples(0)
    sd = algo.sampler.process_samples(0, paths)
    b = sd.lane_batch
    theta0 = algo.policy.get_param_values()                     # float64 master parameters
    batch = S.batch_from_traj(b.to_numpy(), b.adv.cpu().numpy(), b.valid_mask())
    dims = P.Dims(b.O, (hidden, hidden), b.A)
    algo.optimize_policy(0, sd)
    theta_dev = algo.policy.get_param_values()
    theta_ref, info = OPT.trpo_step(theta0, batch, dims, step_size=0.01, cg_iters=cg_iters)
    li = algo.optimizer.last_info
    assert li["n_iter"] == info["n_iter"] and li["rejected"] == info["rejected"] and not info["rejected"]
    assert _rel(theta_dev, theta_ref) < tol, _rel(theta_dev, theta_ref)
    np.testing.assert_allclose(li["loss"], info["loss"], rtol=100 * tol, atol=1e-9)
    np.testing.assert_allclose(li["constraint_val"], info["constraint_val"], rtol=100 * tol)
