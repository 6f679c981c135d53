"""GPU: the population kernels of CEM and the CEM algorithm end to end.

- b200rl_population_sample: rows bit-identical to NumPy float64 arithmetic on the Philox stream-2 draws, for a member list
  with gaps and indices above 2^32, and the draws against the oracle's Philox restatement;
- b200rl_population_rollout: episode (m, e) bit-identical to the first path of lane e of b200rl_rollout with theta_m, for
  every env kind x hidden 32/64, n_evals 1 and 3, and populations of 1, 77 and more members than the persistent grid
  holds at once; returns and fitness against a float64 recomputation; reruns bit-identical;
- b200rl_population_topk + b200rl_rows_mean_std: the reference's elite update on its own golden rows and fitness, and a
  tie case;
- CEM.train on PointEnv and CartPole against the oracle driven by the device's fitness, the batch_size criterion, the
  snapshot, and learning progress on CartPole.
"""
import os
import pickle

import numpy as np
import pytest
import torch

import cem_oracle as K
from oracle import philox

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
DEV = torch.device("cuda", 0) if torch.cuda.is_available() else None
ENVS = ["point", "cartpole", "pendulum", "swimmer", "hopper", "cartpole_swingup", "double_pendulum", "half_cheetah"]


def _L():
    from rllab_b200 import _lib as L
    L.load()
    return L


def _eps_rows(members, P, seed, it):
    """Stream-2 draws of the given members from the library's own noise kernel (b200rl_fill_noise): [n][P] float32."""
    from rllab_b200 import ops
    L = _L()
    out = np.zeros((len(members), P), np.float32)
    buf = torch.empty((1, P, 1), dtype=torch.float32, device=DEV)
    for r, m in enumerate(members):
        ops.fill_noise(buf, 1, 0, P, 1, int(m), L.NOISE_NORMAL, seed, it, 2)
        out[r] = buf.cpu().numpy().reshape(P)
    return out


def test_sample_rows_match_numpy_restatement():
    from rllab_b200 import ops
    L = _L()
    P = L.policy_num_params(4, 32, 32, 1)
    rng = np.random.RandomState(0)
    mean = rng.randn(P)
    std = np.abs(rng.randn(P)) * 0.5
    std[::7] = 0.0
    members = np.array([0, 1, 5, 6, 1000, 77777, 2 ** 32 - 1, 2 ** 32, 2 ** 32 + 3, 3 * 2 ** 32 + 11], np.int64)
    seed, it, ev = 12345, 7, 0.37
    rows = torch.empty((len(members), P), dtype=torch.float64, device=DEV)
    ops.population_sample(torch.tensor(mean, device=DEV), torch.tensor(std, device=DEV), ev, seed, it, rows,
                          members=torch.tensor(members, device=DEV))
    eps = _eps_rows(members, P, seed, it)
    ref = eps.astype(np.float64) * np.sqrt(np.square(std) + ev) + mean
    got = rows.cpu().numpy()
    assert np.array_equal(got.view(np.uint64), ref.view(np.uint64))
    # the contiguous-range form gives the same rows as the list form
    rng_rows = torch.empty((3, P), dtype=torch.float64, device=DEV)
    ops.population_sample(torch.tensor(mean, device=DEV), torch.tensor(std, device=DEV), ev, seed, it, rng_rows,
                          member0=2 ** 32 - 1)
    assert torch.equal(rng_rows[:2], rows[6:8])
    # the draws themselves: the oracle's Philox words through the float64 Box-Muller map (the kernel's map is float32)
    Kp = (P + 3) // 4 * 4
    for r, m in enumerate(members):
        raw = philox.raw_block(1, 0, Kp, 1, int(m), seed, it, 2)
        z = philox.normal_from_raw(raw)[0, :P, 0]
        np.testing.assert_allclose(eps[r], z, rtol=0, atol=2e-5)


def _bits(t):
    """Bytes of a tensor: bit-identity that also holds for NaN (DoublePendulum diverges under some random policies, in the
    lane rollout as much as here)."""
    return t.cpu().numpy().tobytes()


def _close(got, ref, scale, where):
    if np.isnan(ref):
        assert np.isnan(got), where
    else:
        assert abs(got - ref) <= 1e-12 * (scale + 1e-300), (where, got, ref)


def _pop_and_lanes(kind_name, H, E, M, mpl, seed=11, it=3, lane0=5, check=None):
    from rllab_b200 import ops
    from oracle import policy as OP
    L = _L()
    kind = L.ENV_KINDS[kind_name]
    info = L.env_info(kind)
    O, A = info["obs_dim"], info["act_dim"]
    dims = OP.Dims(O, (H, H), A)
    mean = OP.init_params(dims, np.random.RandomState(1))
    std = np.full(dims.P, 0.3)
    rows = torch.empty((M, dims.P), dtype=torch.float64, device=DEV)
    ops.population_sample(torch.tensor(mean, device=DEV), torch.tensor(std, device=DEV), 0.0, seed, it, rows)
    res = ops.PopulationResult(M, E, O, DEV)
    ops.population_rollout(kind, rows, H, H, 1e-6, E, mpl, 0.99, seed, it, lane0, res)
    res2 = ops.PopulationResult(M, E, O, DEV)
    ops.population_rollout(kind, rows, H, H, 1e-6, E, mpl, 0.99, seed, it, lane0, res2)
    torch.cuda.synchronize()
    for name in ("ret", "undisc", "len", "obs_first", "obs_last", "member"):
        assert _bits(getattr(res, name)) == _bits(getattr(res2, name)), name      # reruns are bit-identical
    members = range(M) if check is None else check
    th32 = rows.float()
    ret, und, ln = res.ret.cpu().numpy(), res.undisc.cpu().numpy(), res.len.cpu().numpy()
    of, ol, mem = res.obs_first.cpu().numpy(), res.obs_last.cpu().numpy(), res.member.cpu().numpy()
    b = ops.LaneBatch(O, A, E, mpl, DEV)
    for m in members:
        ops.rollout(kind, th32[m].contiguous(), H, H, 1e-6, b, mpl, None, None, seed, it, lane0 + m * E)
        t = b.to_numpy()
        for e in range(E):
            end = int(np.nonzero(t["flags"][:, e] & L.FLAG_END)[0][0])
            n = end + 1
            assert ln[m, e] == n, (m, e)
            assert np.array_equal(of[m, e].view(np.uint32), t["obs"][:, 0, e].view(np.uint32)), (m, e)
            assert np.array_equal(ol[m, e].view(np.uint32), t["obs"][:, end, e].view(np.uint32)), (m, e)
            r = t["rew"][:n, e].astype(np.float64)
            g = K.discounted_return(r, 0.99)
            _close(ret[m, e], g, np.sum(np.abs(r) * 0.99 ** np.arange(n)), (m, e))
            _close(und[m, e], np.sum(r), np.sum(np.abs(r)), (m, e))
        _close(mem[m, 0], K.stderr_lb(ret[m]), np.max(np.abs(ret[m])), m)
        _close(mem[m, 1], K.stderr_lb(und[m]), np.max(np.abs(und[m])), m)
        ls = np.maximum(th32[m, -A:].cpu().numpy(), np.float32(np.log(1e-6)))
        np.testing.assert_allclose(mem[m, 2], np.mean(np.exp(ls.astype(np.float64))), rtol=1e-6)
    return ln


@pytest.mark.parametrize("M", [1, 77, 3000])
@pytest.mark.parametrize("E", [1, 3])
@pytest.mark.parametrize("H", [32, 64])
@pytest.mark.parametrize("env", ENVS)
def test_population_rollout_matches_lane_rollout(env, H, E, M):
    # CartPole: random policies fall after 3-20 steps, so a horizon of 12 both cuts and ends episodes
    mpl = {"cartpole": 12, "swimmer": 60, "hopper": 60, "half_cheetah": 60}.get(env, 80)
    check = None if M <= 77 else sorted(set(list(range(8)) + list(range(M - 8, M)) +
                                            list(np.random.RandomState(M).choice(M, 24, replace=False))))
    ln = _pop_and_lanes(env, H, E, M, mpl, check=check)
    if env == "cartpole" and M > 1:
        assert (ln < mpl).any() and (ln == mpl).any()      # some episodes terminate, some are cut by max_path_length


def test_population_rollout_rejects_unsupported():
    from rllab_b200 import ops
    L = _L()
    rows = torch.zeros((2, 1250), dtype=torch.float64, device=DEV)
    res = ops.PopulationResult(2, 1, 4, DEV)
    with pytest.raises(L.B200RLError):
        ops.population_rollout(L.ENV_CARTPOLE, rows, 16, 16, 1e-6, 1, 10, 0.99, 1, 0, 0, res)
    with pytest.raises(L.B200RLError):
        ops.population_rollout(99, rows, 32, 32, 1e-6, 1, 10, 0.99, 1, 0, 0, res)
    with pytest.raises(L.B200RLError, match=r"\(-3\)"):                    # B200RL_EUNSUPPORTED, like 16-wide
        ops.population_rollout(L.ENV_CARTPOLE, rows, 32, 64, 1e-6, 1, 10, 0.99, 1, 0, 0, res)
    with pytest.raises(ValueError):                                       # rows of the wrong width
        ops.population_rollout(L.ENV_CARTPOLE, rows[:, :1000].contiguous(), 32, 32, 1e-6, 1, 10, 0.99, 1, 0, 0, res)
    with pytest.raises(ValueError):                                       # buffers of the wrong obs_dim
        ops.population_rollout(L.ENV_PENDULUM, rows, 32, 32, 1e-6, 1, 10, 0.99, 1, 0, 0, res)


def _elite(xs, fs, k):
    from rllab_b200 import ops
    xs_d = torch.tensor(xs, dtype=torch.float64, device=DEV)
    idx = torch.empty(k, dtype=torch.int64, device=DEV)
    ops.population_topk(torch.tensor(fs, dtype=torch.float64, device=DEV), k, idx)
    rows = xs_d[idx].contiguous()
    mean = torch.empty(xs.shape[1], dtype=torch.float64, device=DEV)
    std = torch.empty_like(mean)
    ops.rows_mean_std(rows, mean, std)
    return idx.cpu().numpy(), mean.cpu().numpy(), std.cpu().numpy(), rows[0].cpu().numpy()


def test_elite_update_reproduces_reference_golden():
    g = np.load(os.path.join(HERE, "golden", "reference_cem_golden.npz"))
    cases = sorted({k.split("/")[0] for k in g.files})
    n = 0
    for c in cases:
        for it in range(int(g[c + "/n_itr"])):
            p = "%s/%d/" % (c, it)
            xs, fs, nb = g[p + "xs"], g[p + "fs"], int(g[c + "/n_best"])
            idx, mean, std, bx = _elite(xs, fs, min(nb, len(fs)))
            scale = np.max(np.abs(xs))
            assert np.max(np.abs(mean - g[p + "cur_mean"])) <= 1e-12 * scale, (c, it)
            assert np.max(np.abs(std - g[p + "cur_std"])) <= 1e-12 * scale, (c, it)
            assert np.array_equal(bx, g[p + "best_x"]), (c, it)
            n += 1
    assert n >= 9


def test_topk_ties_and_large_population():
    fs = np.array([1.0, 3.0, 3.0, -0.0, 0.0, 2.0, 3.0, np.nan, -1.0, 2.0])
    xs = np.arange(len(fs) * 3, dtype=np.float64).reshape(len(fs), 3)
    idx, mean, std, bx = _elite(xs, fs, 7)
    assert list(idx) == [1, 2, 6, 5, 9, 0, 3]
    best, m_ref, s_ref, b_ref = K.elite_update(xs, np.where(np.isnan(fs), -np.inf, fs), 7)
    assert list(best) == list(idx)
    assert np.array_equal(mean, m_ref) and np.array_equal(std, s_ref) and np.array_equal(bx, b_ref)
    rng = np.random.RandomState(3)
    for M, k in ((200000, 10000), (65536, 3276), (5000, 1), (4097, 4097)):
        f = np.round(rng.randn(M) * 50.0)          # many ties
        from rllab_b200 import ops
        idx = torch.empty(k, dtype=torch.int64, device=DEV)
        ops.population_topk(torch.tensor(f, device=DEV), k, idx)
        assert np.array_equal(idx.cpu().numpy(), np.argsort(-f, kind="stable")[:k]), (M, k)


def _cem(env_name, **kw):
    from rllab_b200.algos.cem import CEM
    from rllab_b200.envs.normalized_env import normalize
    from rllab_b200.policies.gaussian_mlp_policy import GaussianMLPPolicy
    if env_name == "point":
        from rllab_b200.envs.point_env import PointEnv
        env = normalize(PointEnv())
    elif env_name == "swimmer":
        from rllab_b200.envs.mujoco.swimmer_env import SwimmerEnv
        env = normalize(SwimmerEnv())
    else:
        from rllab_b200.envs.box2d.cartpole_env import CartpoleEnv
        env = normalize(CartpoleEnv())
    pol = GaussianMLPPolicy(env.spec, hidden_sizes=(32, 32), seed=1)
    return CEM(env, pol, **kw), env, pol


@pytest.mark.parametrize("env_name,kw", [
    ("point", dict(n_samples=200, n_evals=3, best_frac=0.05, max_path_length=40, extra_decay_time=2)),
    ("cartpole", dict(n_samples=300, n_evals=1, best_frac=0.1, max_path_length=100, extra_std=0.5)),
    ("cartpole", dict(n_samples=50, batch_size=3000, n_evals=2, best_frac=0.1, max_path_length=100)),
    ("point", dict(n_samples=10, n_evals=1, best_frac=0.01, max_path_length=30)),
    ("swimmer", dict(n_samples=24, n_evals=2, best_frac=0.25, max_path_length=20)),
])
def test_cem_train_matches_oracle(env_name, kw, tmp_path):
    from rllab_b200.misc import logger
    algo, env, pol = _cem(env_name, n_itr=3, seed=2024, **kw)
    P = pol.n_params
    cur_mean = pol.get_param_values().copy()
    cur_std = np.full(P, float(algo.init_std))
    logger.set_quiet(True)
    logger.set_snapshot_dir(str(tmp_path))
    logger.set_snapshot_mode("all")
    hist = []
    orig = algo._population

    def spy(itr, extra_var):
        out = orig(itr, extra_var)
        hist.append(out[1].copy())
        return out
    algo._population = spy
    try:
        algo.train()
    finally:
        logger.set_snapshot_mode("none")
        logger.set_snapshot_dir(None)
    table = logger.get_last_table()
    E = algo.n_evals
    nb = K.n_best(algo.n_samples, algo.best_frac)
    for itr, host in enumerate(hist):
        M = host.shape[0]
        if algo.batch_size is not None:
            assert M == K.batch_prefix(host[:, 3 + E - 1], algo.batch_size)
            assert np.sum(host[:M - 1, 3 + E - 1]) < algo.batch_size
        else:
            assert M == algo.n_samples
        eps = _eps_rows(range(M), P, algo.seed, itr)
        xs = K.theta_rows(cur_mean, cur_std, eps, itr, algo.extra_std, algo.extra_decay_time)
        best, cur_mean_ref, cur_std_ref, bx = K.elite_update(xs, host[:, 0], min(nb, M))
        with open(os.path.join(str(tmp_path), "itr_%d.pkl" % itr), "rb") as f:
            snap = pickle.load(f)
        assert np.array_equal(snap["cur_mean"], cur_mean_ref), itr
        assert np.array_equal(snap["cur_std"], cur_std_ref), itr
        assert np.array_equal(snap["policy"].get_param_values(), bx), itr
        assert snap["itr"] == itr
        cur_mean, cur_std = cur_mean_ref, cur_std_ref
    ref = K.tabular(len(hist) - 1, cur_std, hist[-1][:, 1], hist[-1][:, 0], hist[-1][:, 3:3 + E])
    for key, v in ref.items():
        assert table[key] == pytest.approx(v, rel=1e-12, abs=1e-12), key
    assert np.array_equal(pol.get_param_values(), bx)
    assert np.array_equal(algo.cur_mean.cpu().numpy(), cur_mean)
    lens = hist[-1][:, 3:3 + E]
    # the device exponentiates the float32 log_std, the oracle the float64 one
    assert table["AveragePolicyStd"] == pytest.approx(K.average_policy_std(xs, lens, pol.action_dim), rel=1e-6)
    if env_name == "swimmer":
        # SwimmerEnv.log_diagnostics from each episode's first and last observation, recomputed here from the lane rollout
        # of every member of the last iteration (its first path is the member's episode, bit for bit)
        from rllab_b200 import _lib as L, ops
        O, A, T = pol.obs_dim, pol.action_dim, int(algo.max_path_length)
        b = ops.LaneBatch(O, A, E, T, DEV)
        progs = []
        for m in range(len(xs)):
            th32 = torch.tensor(xs[m], dtype=torch.float64, device=DEV).float()
            ops.rollout(L.ENV_SWIMMER, th32, 32, 32, pol.min_std, b, T, None, None, algo.seed, len(hist) - 1, m * E)
            t = b.to_numpy()
            for e in range(E):
                end = int(np.nonzero(t["flags"][:, e] & L.FLAG_END)[0][0])
                assert end + 1 == lens[m, e]
                progs.append(float(t["obs"][O - 3, end, e]) - float(t["obs"][O - 3, 0, e]))
        for key, fn in (("Average", np.mean), ("Max", np.max), ("Min", np.min), ("Std", np.std)):
            assert table[key + "ForwardProgress"] == pytest.approx(fn(progs), rel=1e-12, abs=1e-12), key


def test_cem_cartpole_learns():
    from rllab_b200.misc import logger
    logger.set_quiet(True)
    # init_std 1 samples near-random policies (mean episode ~6 steps) whose population average barely moves in 10
    # iterations; a narrower search around the initial policy climbs (on an H100: AverageReturn 77 -> 410)
    algo, env, pol = _cem("cartpole", n_itr=10, n_samples=4000, best_frac=0.05, max_path_length=200, init_std=0.1,
                          extra_std=0.1, extra_decay_time=5, seed=7)
    returns = []
    orig = logger.dump_tabular

    def grab(*a, **k):
        orig(*a, **k)
        returns.append(logger.get_last_table()["AverageReturn"])
    logger.dump_tabular = grab
    try:
        algo.train()
    finally:
        logger.dump_tabular = orig
    assert len(returns) == 10
    assert np.mean(returns[-3:]) > 2.0 * np.mean(returns[:2]), returns


def test_cem_rejects_plot():
    from rllab_b200.algos.cem import CEM
    with pytest.raises(NotImplementedError):
        CEM(None, None, plot=True)
