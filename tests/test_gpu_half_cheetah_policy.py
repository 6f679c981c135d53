"""HalfCheetah's policy network, (obs 20, act 6) at hidden 32 and 64, through every policy pass, against the float64
oracle: the checks of tests/test_gpu_update_shapes.py and tests/test_gpu_ppo.py run at this shape (loss / KL, gradient,
penalized gradient, activation cache and FVP with and without it, f64 parity kernels, masking, determinism; batch
sizes 1, 77, exact tiles and large), get_actions, one CEM population rollout bit-identical to the lane rollout, and
TRPO / VPG / PPO updates through the host API."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")

import test_gpu_cem as CEM                                                        # noqa: E402
import test_gpu_ppo as PPO                                                        # noqa: E402
import test_gpu_rollout_shapes as RS                                              # noqa: E402
import test_gpu_update_shapes as U                                                # noqa: E402
from test_gpu_update_shapes import SIZES, dev, n_sm                               # noqa: E402,F401

pytestmark = pytest.mark.gpu

SHAPES = [(20, 6, 32), (20, 6, 64)]


def _id(s):
    return "O20A6H%d" % s[2]


@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("shape", SHAPES, ids=_id)
def test_loss_kl_at_theta_old(dev, n_sm, shape, size):
    U.test_loss_kl_at_theta_old(dev, n_sm, shape, size)


@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("shape", SHAPES, ids=_id)
def test_loss_and_gradient_off_theta_old(dev, n_sm, shape, size):
    U.test_loss_and_gradient_off_theta_old(dev, n_sm, shape, size)


@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("shape", SHAPES, ids=_id)
def test_activation_cache_and_fvp(dev, n_sm, shape, size):
    U.test_activation_cache_and_fvp(dev, n_sm, shape, size)


@pytest.mark.parametrize("size", ["77", "large"])
@pytest.mark.parametrize("shape", SHAPES, ids=_id)
def test_f64_parity_kernels(dev, n_sm, shape, size):
    U.test_f64_parity_kernels(dev, n_sm, shape, size)


@pytest.mark.parametrize("shape", SHAPES, ids=_id)
def test_float32_passes_are_deterministic(dev, n_sm, shape):
    U.test_float32_passes_are_deterministic(dev, n_sm, shape)


@pytest.mark.parametrize("size", ["77", "large"])
@pytest.mark.parametrize("shape", SHAPES, ids=_id)
def test_masked_samples(dev, n_sm, shape, size):
    U.test_masked_samples(dev, n_sm, shape, size)


@pytest.mark.parametrize("size", ["77", "large"])
@pytest.mark.parametrize("shape", SHAPES, ids=_id)
def test_fvp_tile_lists(dev, n_sm, shape, size):
    U.test_fvp_tile_lists(dev, n_sm, shape, size)


@pytest.mark.parametrize("size", ["77", "large"])
@pytest.mark.parametrize("shape", SHAPES, ids=_id)
def test_min_std_clamp_per_component(dev, n_sm, shape, size):
    U.test_min_std_clamp_per_component(dev, n_sm, shape, size)


@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("shape", SHAPES, ids=_id)
def test_penalized_gradient_matches_oracle(dev, n_sm, shape, size):
    PPO.test_penalized_gradient_matches_oracle(dev, n_sm, shape, size)


@pytest.mark.parametrize("size", ["77", "large"])
@pytest.mark.parametrize("shape", SHAPES, ids=_id)
def test_penalized_gradient_masked(dev, n_sm, shape, size):
    PPO.test_penalized_gradient_masked(dev, n_sm, shape, size)


@pytest.mark.parametrize("shape", SHAPES, ids=_id)
def test_penalty_zero_and_triple_equal_grad_pass(dev, n_sm, shape):
    PPO.test_penalty_zero_and_triple_equal_grad_pass(dev, n_sm, shape)


def test_num_params():
    from rllab_b200 import _lib as L
    assert L.policy_num_params(20, 32, 32, 6) == 1932
    assert L.policy_num_params(20, 64, 64, 6) == 5900


@pytest.mark.parametrize("H", [32, 64])
def test_get_actions_philox(dev, H):
    RS.test_get_actions_philox(dev, 20, 6, H)


@pytest.mark.parametrize("H", [32, 64])
def test_cem_member_equals_lane_rollout(H):
    CEM._pop_and_lanes("half_cheetah", H, 2, 5, 40)


# --------------------------------------------------------------------------- algorithms through the host API
def _algo(algo_name, hidden=32, n_envs=512, T=50, **kw):
    from rllab_b200.algos.npo import NPO  # noqa: F401
    from rllab_b200.algos.trpo import TRPO
    from rllab_b200.algos.vpg import VPG
    from rllab_b200.baselines.linear_feature_baseline import LinearFeatureBaseline
    from rllab_b200.envs.mujoco.half_cheetah_env import HalfCheetahEnv
    from rllab_b200.envs.normalized_env import normalize
    from rllab_b200.policies.gaussian_mlp_policy import GaussianMLPPolicy
    env = normalize(HalfCheetahEnv())
    policy = GaussianMLPPolicy(env.spec, hidden_sizes=(hidden, hidden), seed=3)
    args = dict(env=env, policy=policy, baseline=LinearFeatureBaseline(env.spec), batch_size=n_envs * T,
                max_path_length=T, n_itr=2, discount=0.99, sampler_args=dict(n_envs=n_envs, seed=7))
    args.update(kw)
    if algo_name == "ppo":
        from rllab_b200.algos.ppo import PPO as PPOAlgo
        return PPOAlgo(**args)
    return TRPO(**args) if algo_name == "trpo" else VPG(**args)


@pytest.mark.parametrize("hidden", [32, 64])
def test_trpo_update_matches_oracle(dev, hidden):
    import test_gpu_algos as GA
    from oracle import optim as OPT
    from oracle import policy as P
    from oracle import sampler as S
    algo = _algo("trpo", hidden, optimizer_args=dict(cg_iters=4))
    algo.start_worker()
    algo.init_opt()
    sd = algo.sampler.process_samples(0, algo.sampler.obtain_samples(0))
    b = sd.lane_batch
    theta0 = algo.policy.theta32.double().cpu().numpy()
    batch = S.batch_from_traj(b.to_numpy(), b.adv.cpu().numpy(), b.valid_mask())
    dims = P.Dims(20, (hidden, hidden), 6)
    algo.optimize_policy(0, sd)
    theta_ref, info = OPT.trpo_step(theta0, batch, dims, step_size=0.01, cg_iters=4)
    li = algo.optimizer.last_info
    assert li["n_iter"] == info["n_iter"] and li["rejected"] == info["rejected"] and not info["rejected"]
    assert GA._rel(algo.policy.get_param_values(), theta_ref) < GA.PARAM_RTOL
    assert 0 < li["constraint_val"] <= 0.01


def test_vpg_update_matches_oracle(dev):
    import test_gpu_algos as GA
    from oracle import policy as P
    from oracle import sampler as S
    algo = _algo("vpg")
    algo.start_worker()
    algo.init_opt()
    sd = algo.sampler.process_samples(0, algo.sampler.obtain_samples(0))
    b = sd.lane_batch
    dims = P.Dims(20, (32, 32), 6)
    theta0 = algo.policy.get_param_values()
    batch = S.batch_from_traj(b.to_numpy(), b.adv.cpu().numpy(), b.valid_mask())
    g_ref = P.grad_surr(algo.policy.theta32.double().cpu().numpy(), batch, dims, "vpg")
    theta_ref, _, _, _ = P.adam_step(theta0, g_ref, np.zeros(dims.P), np.zeros(dims.P), 0)
    algo.optimize_policy(0, sd)
    assert GA._rel(algo.policy.get_param_values(), theta_ref) < GA.PARAM_RTOL


@pytest.mark.parametrize("algo_name", ["trpo", "vpg", "ppo"])
def test_training_loop_runs_and_logs(dev, algo_name):
    from rllab_b200.misc import logger
    algo = _algo(algo_name, n_envs=1024, T=100, store_paths=True)   # store_paths: the env's own diagnostics run
    algo.train()
    theta = algo.policy.get_param_values()
    assert np.isfinite(theta).all()
    tab = logger.get_last_table()
    for k in ("AverageReturn", "LossBefore", "LossAfter", "MeanKL", "AverageForwardProgress"):
        assert k in tab and np.isfinite(float(tab[k])), k
