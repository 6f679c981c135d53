"""HalfCheetah on the GPU against the float64 oracle (tests/planar_tree_oracle.py): env reset / step on lanes in free
flight, at joint limits, on their feet, upside down on the torso and head, and sunk into the floor with all 38 constraint
rows active (the compaction arrays full); the fused lane rollout at hidden 32 and
64, step by step, with the in-kernel Philox stream (action noise chunks 0 and 1) equal to injected noise."""
import numpy as np
import pytest
import torch

from oracle import policy as P
import planar_tree_oracle as T

pytestmark = pytest.mark.gpu

SEED, ITER = 1234, 7
_WORST = {}


def _mods():
    from rllab_b200 import _lib as L, ops
    L.load()
    return L, ops


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


def _mixed_states(rng, n):
    """Five groups of n lanes: airborne, hinges pushed past their limits, standing / landing, flipped onto the back, and
    sunk into the floor with every hinge past a limit (all 38 constraint rows active).  The fifth group draws from its
    own stream, so the first four and whatever the caller draws from `rng` next do not depend on it."""
    m = T.half_cheetah_model()
    q = np.zeros((9, 4 * n))
    v = rng.normal(0, 1.0, (9, 4 * n))
    q[0] = rng.uniform(-2, 2, 4 * n)
    lo = np.array([l[0] for l in m.limits[1:]])[:, None]
    hi = np.array([l[1] for l in m.limits[1:]])[:, None]
    g = [slice(k * n, (k + 1) * n) for k in range(4)]
    q[1, g[0]] = rng.uniform(0.5, 1.0, n)
    q[2, g[0]] = rng.uniform(-0.3, 0.3, n)
    q[3:, g[0]] = rng.uniform(lo + 0.05, hi - 0.05, (6, n))
    q[1, g[1]] = rng.uniform(0.5, 1.0, n)
    q[3:, g[1]] = np.where(rng.rand(6, n) < 0.5, lo - rng.uniform(0, 0.1, (6, n)), hi + rng.uniform(0, 0.1, (6, n)))
    q[1, g[2]] = rng.uniform(-0.4, -0.2, n)                       # crouched: feet and shins on the floor
    q[2, g[2]] = rng.uniform(-0.2, 0.2, n)
    q[3:, g[2]] = rng.uniform(lo, hi, (6, n))
    q[1, g[3]] = rng.uniform(-0.72, -0.6, n)                      # upside down: torso / head capsules on the floor
    q[2, g[3]] = np.pi + rng.uniform(-0.4, 0.4, n)
    q[3:, g[3]] = rng.uniform(lo, hi, (6, n))
    v[:, g[3]] *= 0.3
    g5 = np.random.RandomState(n + 5)
    q5 = np.zeros((9, n))
    q5[0] = g5.uniform(-2, 2, n)
    q5[1] = g5.uniform(-2.5, -1.0, n)                             # every end sphere below the floor
    q5[2] = g5.uniform(-0.3, 0.3, n)
    q5[3:] = np.where(g5.rand(6, n) < 0.5, lo - g5.uniform(0.01, 0.1, (6, n)), hi + g5.uniform(0.01, 0.1, (6, n)))
    v5 = g5.normal(0, 1.0, (9, n))
    return np.concatenate([np.concatenate([q, q5], axis=1), np.concatenate([v, v5], axis=1)]).astype(np.float32)


def _report(key, err):
    _WORST[key] = max(_WORST.get(key, 0.0), float(err))
    print("HALF_CHEETAH_ERR %s %.3g" % (key, _WORST[key]))


def test_env_step_matches_oracle_on_every_contact_regime(dev):
    L, ops = _mods()
    rng = np.random.RandomState(0)
    n = 512
    s0 = _mixed_states(rng, n)
    N = s0.shape[1]
    u = np.concatenate([rng.uniform(-1.5, 1.5, (6, 4 * n)), rng.uniform(-1.5, 1.5, (6, n))], axis=1).astype(np.float32)
    env = T.HalfCheetahEnv()
    # the oracle takes the device's action map (NormalizedEnv with lb, ub = -1, 1 clips) on the same float32 inputs
    s_ref, r_ref, d_ref = env.step(s0.astype(np.float64), np.clip(u.astype(np.float64), -1, 1))
    kin0 = T.dynamics(env.m, list(s0[:9].astype(np.float64)), list(s0[9:].astype(np.float64)), np.zeros((6, N)))[2]
    assert (kin0["n_active"][2 * n:3 * n] > 0).mean() > 0.85         # most crouched lanes touch the floor
    assert (kin0["n_active"][3 * n:] > 0).all()                      # every flipped lane lies on the floor
    assert (kin0["n_active"][n:2 * n] > 0).all()                     # the limit group has active limit rows
    assert (kin0["n_active"][4 * n:] == 38).mean() >= 0.99           # the sunk group fills the compaction arrays
    state = torch.tensor(s0, device=dev).contiguous()
    obs = torch.empty((20, N), dtype=torch.float32, device=dev)
    rew = torch.empty(N, dtype=torch.float32, device=dev)
    done = torch.empty(N, dtype=torch.uint8, device=dev)
    ops.env_step(L.ENV_HALF_CHEETAH, N, state, torch.tensor(u, device=dev), obs, rew, done)
    torch.cuda.synchronize()
    s1, o1, r1, d1 = state.cpu().numpy(), obs.cpu().numpy(), rew.cpu().numpy(), done.cpu().numpy()
    assert np.isfinite(s1).all() and not d1.any() and not d_ref.any()
    o_ref = env.obs(s_ref)
    # Euler: one dynamics evaluation at the step's input state, the same float32 numbers on both sides; only a lane with
    # a residual within float32 rounding of zero can take a different active set, and only those are excused
    near = (np.abs(T.constraint_residuals(env.m, list(s0[:9].astype(np.float64)))) < 1e-5).any(axis=0)
    assert near.mean() < 0.01, near.mean()
    for k, name in enumerate(["free", "limits", "feet", "flipped", "all_rows"]):
        lo_, hi_ = k * n, (k + 1) * n
        sl = slice(lo_, hi_)
        scale = 1.0 + np.abs(s_ref[:, sl])
        err = np.abs(s1[:, sl] - s_ref[:, sl]) / scale
        _report("state_" + name, err.max())
        _report("rew_" + name, np.abs(r1[sl] - r_ref[sl]).max())
        _report("obs_" + name, (np.abs(o1[:, sl] - o_ref[:, sl]) / (1.0 + np.abs(o_ref[:, sl]))).max())
        keep = ~near[sl]
        assert (err[:, keep] < 2e-4).all(), (name, err[:, keep].max())
        assert (np.abs(r1[sl] - r_ref[sl])[keep] < 2e-5).all(), name
        assert (np.abs(o1[:, sl] - o_ref[:, sl])[:, keep] / (1.0 + np.abs(o_ref[:, sl][:, keep])) < 2e-4).all(), name


def test_env_reset_matches_oracle_and_philox(dev):
    L, ops = _mods()
    N = 1000
    env = T.HalfCheetahEnv()
    raw = torch.empty((1, 18, N), dtype=torch.float32, device=dev)
    ops.fill_noise(raw, 1, 3, 18, N, 5, L.NOISE_NORMAL, SEED, ITER, 1)
    s1 = torch.empty((18, N), dtype=torch.float32, device=dev)
    o1 = torch.empty((20, N), dtype=torch.float32, device=dev)
    s2, o2 = torch.empty_like(s1), torch.empty_like(o1)
    ops.env_reset(L.ENV_HALF_CHEETAH, N, s1, o1, raw.view(18, N), SEED, ITER, 3, 5)
    ops.env_reset(L.ENV_HALF_CHEETAH, N, s2, o2, None, SEED, ITER, 3, 5)
    torch.cuda.synchronize()
    assert torch.equal(s1, s2) and torch.equal(o1, o2)
    rr = raw.view(18, N).cpu().numpy().astype(np.float64)
    s_ref = env.reset(rr)
    o_ref = env.obs(s1.cpu().numpy().astype(np.float64))
    np.testing.assert_allclose(s1.cpu().numpy(), s_ref, rtol=1e-6, atol=1e-7)
    np.testing.assert_allclose(o1.cpu().numpy(), o_ref, rtol=2e-6, atol=2e-6)
    assert np.abs(o1.cpu().numpy()[19] - 0.7).max() < 0.2           # torso COM height near the initial 0.7


def _state_from_obs(env, o):
    """(q, v) from obs = [q[1:], v, comX, 0, comZ]: rootx is comX minus the COM offset of the rest of the pose."""
    s = np.concatenate([np.zeros((1, o.shape[1])), o[:17]])
    s[0] = o[17] - env.kin(s)["comX"]
    return s


@pytest.mark.parametrize("H", [32, 64])
def test_rollout_matches_oracle_step_by_step(dev, H):
    L, ops = _mods()
    N, Tn, mpl = 300, 60, 25
    env = T.HalfCheetahEnv()
    dims = P.Dims(20, (H, H), 6)
    rng = np.random.RandomState(H)
    theta = P.init_params(dims, rng) + rng.randn(dims.P) * 0.05
    theta[-6:] = -0.5 + 0.1 * np.arange(6)
    th32 = torch.tensor(theta, dtype=torch.float32, device=dev)
    theta = th32.double().cpu().numpy()
    eps = torch.empty((Tn, 6, N), dtype=torch.float32, device=dev)
    rr = torch.empty((Tn + 1, 18, N), dtype=torch.float32, device=dev)
    ops.fill_noise(eps, Tn, 0, 6, N, 0, L.NOISE_NORMAL, SEED, ITER, 0)
    ops.fill_noise(rr, Tn + 1, 0, 18, N, 0, L.NOISE_NORMAL, SEED, ITER, 1)
    b = ops.LaneBatch(20, 6, N, Tn, dev)
    ops.rollout(L.ENV_HALF_CHEETAH, th32, H, H, 1e-6, b, mpl, eps, rr, SEED, ITER, 0)
    bp = ops.LaneBatch(20, 6, N, Tn, dev)
    ops.rollout(L.ENV_HALF_CHEETAH, th32, H, H, 1e-6, bp, mpl, None, None, SEED, ITER, 0)
    torch.cuda.synchronize()
    tr, tp = b.to_numpy(), bp.to_numpy()
    for k in tr:                                                      # in-kernel Philox == injected noise, bit for bit
        assert np.array_equal(np.asarray(tr[k]).view(np.uint8), np.asarray(tp[k]).view(np.uint8)), k
    # bookkeeping: never done; paths end at max_path_length or at the end of the buffer
    t = np.arange(Tn)[:, None]
    assert (tr["flags"] & 1 == 0).all()
    assert np.array_equal(tr["tstep"], np.broadcast_to(t % mpl, (Tn, N)))
    # policy: mean from the float64 forward on the device's obs, action = mean + std * eps
    obs = tr["obs"].astype(np.float64)
    mu, log_std = P.forward(theta, obs.reshape(20, -1).T, dims, 1e-6)
    mu = mu.T.reshape(6, Tn, N)
    np.testing.assert_allclose(tr["mean"], mu, rtol=2e-5, atol=2e-5)
    e = eps.cpu().numpy().transpose(1, 0, 2)
    np.testing.assert_allclose(tr["act"], tr["mean"] + np.exp(log_std)[:, None, None] * e, rtol=1e-5, atol=1e-5)
    # resets from reset_raw rows, and every other step replayed through the float64 oracle from the device's obs
    raw = rr.cpu().numpy().astype(np.float64)
    np.testing.assert_allclose(obs[:, 0], env.obs(env.reset(raw[0])), rtol=1e-5, atol=1e-5)
    errs, rerr = [], []
    for ti in range(Tn - 1):
        end = (tr["flags"][ti] & 2) != 0
        s = _state_from_obs(env, obs[:, ti])
        s2, r, _ = env.step(s, np.clip(tr["act"][:, ti].astype(np.float64), -1, 1))
        o2 = env.obs(s2)
        # the state is rebuilt from float32 obs; lanes with a residual within rounding of zero are excused
        near = (np.abs(T.constraint_residuals(env.m, list(s[:9]))) < 1e-5).any(axis=0)
        rerr.append(np.where(near, 0.0, np.abs(tr["rew"][ti] - r) / (1.0 + np.abs(r))))
        err = (np.abs(o2 - obs[:, ti + 1]) / (1.0 + np.abs(o2))).max(axis=0)
        errs.append(np.where(end | near, 0.0, err))
        fresh = env.obs(env.reset(raw[ti + 1]))
        if end.any():
            np.testing.assert_allclose(obs[:, ti + 1][:, end], fresh[:, end], rtol=1e-5, atol=1e-5)
    errs, rerr = np.array(errs), np.array(rerr)
    _report("rollout_obs_h%d" % H, errs.max())
    _report("rollout_rew_h%d" % H, rerr.max())
    assert errs.max() < 1e-3 and rerr.max() < 1e-3, (errs.max(), rerr.max())
