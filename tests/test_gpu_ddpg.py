"""GPU: DDPG (rllab_b200/csrc/ddpg.cu) against the float64 oracle tests/ddpg_oracle.py -- the deterministic policy, the
Q function and the noise-free rollout; one do_training (b200rl_ddpg_update) in float64 and float32; the fused train loop
step by step in float64 from the device's own state; float32 against float64; independence of runs in one launch and
bit-identical reruns; the DDPG algorithm with the reference's examples/ddpg_cartpole.py body."""
import os

import numpy as np
import pytest
import torch

import ddpg_oracle as K
from rllab_b200 import _lib as L
from rllab_b200 import ops

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
BOX_KINDS = dict(point=L.ENV_POINT, cartpole=L.ENV_CARTPOLE, pendulum=L.ENV_PENDULUM,
                 cartpole_swingup=L.ENV_CARTPOLE_SWINGUP, double_pendulum=L.ENV_DOUBLE_PENDULUM)


def _hp(**kw):
    base = dict(n_updates_per_sample=1, max_path_length=30, min_pool_size=40, replay_pool_size=150,
                include_horizon_terminal_transitions=0, es_kind=L.ES_OU, discount=0.99, scale_reward=0.01,
                soft_target_tau=0.05, qf_weight_decay=0.01, qf_learning_rate=1e-3, policy_weight_decay=0.02,
                policy_learning_rate=1e-3, ou_mu=0.0, ou_theta=0.15, ou_sigma=0.3, gs_max_sigma=1.0, gs_min_sigma=0.1,
                gs_decay_period=200.0)
    base.update(kw)
    return base


def _dims(kind):
    info = L.env_info(kind)
    return K.Dims(info["obs_dim"], info["act_dim"])


def _nets(d, seed, moments=False):
    rng = np.random.RandomState(seed)
    th = np.concatenate([K.init_params(d.pshapes, rng), K.init_params(d.qshapes, rng)])
    tg = th + 0.05 * rng.randn(d.P)
    if moments:
        return np.stack([th, 1e-3 * rng.randn(d.P), 1e-6 * rng.rand(d.P), tg])
    return np.stack([th, np.zeros(d.P), np.zeros(d.P), tg])


def _scale(x):
    return max(1.0, float(np.abs(x).max()))


@pytest.mark.parametrize("name", sorted(BOX_KINDS))
def test_get_actions_get_qval_match_oracle(name):
    kind = BOX_KINDS[name]
    d = _dims(kind)
    nets = _nets(d, 3)
    n = 1000
    rng = np.random.RandomState(4)
    obs = rng.randn(n, d.O).astype(np.float32)
    act = rng.uniform(-1, 1, size=(n, d.A)).astype(np.float32)
    th32 = nets[0].astype(np.float32)
    p32 = torch.tensor(th32[:d.PP], device=DEV)
    q32 = torch.tensor(th32[d.PP:], device=DEV)
    o = torch.tensor(np.ascontiguousarray(obs.T), device=DEV)
    a = torch.tensor(np.ascontiguousarray(act.T), device=DEV)
    mu = torch.empty((d.A, n), dtype=torch.float32, device=DEV)
    q = torch.empty(n, dtype=torch.float32, device=DEV)
    ops.deterministic_get_actions(p32, d.O, d.A, o, n, mu)
    ops.qf_get_qval(q32, d.O, d.A, o, a, n, q)
    _, _, ref_mu = K.pi_forward(d, th32[:d.PP].astype(np.float64), obs.astype(np.float64))
    _, _, ref_q = K.q_forward(d, th32[d.PP:].astype(np.float64), obs.astype(np.float64), act.astype(np.float64))
    np.testing.assert_allclose(mu.cpu().numpy().T, ref_mu, rtol=0, atol=2e-6)
    np.testing.assert_allclose(q.cpu().numpy(), ref_q, rtol=0, atol=2e-6 * _scale(ref_q))


@pytest.mark.parametrize("name", sorted(BOX_KINDS))
def test_deterministic_rollout_replays_step_by_step(name):
    """Every sample of the noise-free rollout: the action is the oracle's policy output at the recorded observation,
    and the next observation / reward / done are b200rl_env_step's on the device's own state and action."""
    kind = BOX_KINDS[name]
    d = _dims(kind)
    nets = _nets(d, 5)
    N, T, mpl = 64, 40, 25
    p32 = torch.tensor(nets[0][:d.PP].astype(np.float32), device=DEV)
    b = ops.LaneBatch(d.O, d.A, N, T, DEV)
    ops.rollout_deterministic(kind, p32, b, mpl, seed=7, it=3)
    t = b.to_numpy()
    obs, act, rew, flags = t["obs"], t["act"], t["rew"], t["flags"]
    _, _, ref = K.pi_forward(d, nets[0][:d.PP].astype(np.float32).astype(np.float64),
                             obs.transpose(1, 2, 0).reshape(-1, d.O).astype(np.float64))
    np.testing.assert_allclose(act.transpose(1, 2, 0).reshape(-1, d.A), ref, rtol=0, atol=2e-6)
    # replay: reset every lane as the rollout did, then step with the recorded actions
    S = L.env_info(kind)["state_dim"]
    state = torch.empty((S, N), dtype=torch.float32, device=DEV)
    o = torch.empty((d.O, N), dtype=torch.float32, device=DEV)
    r = torch.empty(N, dtype=torch.float32, device=DEV)
    dn = torch.empty(N, dtype=torch.uint8, device=DEV)
    ops.env_reset(kind, N, state, o, seed=7, it=3, row=0, lane0=0)
    for step in range(T):
        np.testing.assert_array_equal(o.cpu().numpy(), obs[:, step, :])
        ops.env_step(kind, N, state, torch.tensor(np.ascontiguousarray(act[:, step, :]), device=DEV), o, r, dn)
        np.testing.assert_array_equal(r.cpu().numpy(), rew[step])
        np.testing.assert_array_equal(dn.cpu().numpy(), (flags[step] & L.FLAG_DONE) > 0)
        ends = np.nonzero(flags[step] & L.FLAG_END)[0]
        if len(ends) and step + 1 < T:
            st2 = torch.empty((S, N), dtype=torch.float32, device=DEV)
            o2 = torch.empty((d.O, N), dtype=torch.float32, device=DEV)
            ops.env_reset(kind, N, st2, o2, seed=7, it=3, row=step + 1, lane0=0)
            m = torch.tensor(ends, device=DEV)
            state[:, m] = st2[:, m]
            o[:, m] = o2[:, m]


def _pool(d, rows, seed):
    rng = np.random.RandomState(seed)
    return dict(obs=rng.randn(rows, d.O).astype(np.float32), act=rng.uniform(-1, 1, (rows, d.A)).astype(np.float32),
                rew=(0.1 * rng.randn(rows)).astype(np.float32), term=(rng.rand(rows) < 0.2).astype(np.uint8))


def _run_update(kind, f64, hp, pool, idx, nets, t):
    d = _dims(kind)
    g = lambda x, dt: torch.tensor(np.ascontiguousarray(x), dtype=dt, device=DEV)
    nets_t = g(nets, torch.float64)
    outs = [torch.empty(n, dtype=torch.float64, device=DEV) for n in (d.P, 32, 32, 2)]
    ops.ddpg_update(kind, f64, ops.ddpg_hparams(**hp), g(pool["obs"], torch.float32), g(pool["act"], torch.float32),
                    g(pool["rew"], torch.float32), g(pool["term"], torch.uint8), g(idx, torch.int32), nets_t, t, *outs)
    grad, q, y, loss = [x.cpu().numpy() for x in outs]
    return nets_t.cpu().numpy(), dict(grad=grad, q=q, y=y, qf_loss=loss[0], policy_surr=loss[1])


@pytest.mark.parametrize("name", ["cartpole", "point", "double_pendulum"])
def test_update_f64_matches_oracle(name):
    kind = BOX_KINDS[name]
    d = _dims(kind)
    hp = _hp()
    pool = _pool(d, 150, 11)
    idx = np.random.RandomState(12).randint(0, 149, size=32)
    nets = _nets(d, 13, moments=True)
    got_nets, got = _run_update(kind, True, hp, pool, idx, nets, 7)
    ref_nets, ref = K.do_training(d, nets, K.gather(pool, idx, 150), hp, 7)
    for k in ("grad", "q", "y"):
        np.testing.assert_allclose(got[k], ref[k], rtol=0, atol=1e-10 * _scale(ref[k]), err_msg=k)
    for k in ("qf_loss", "policy_surr"):
        assert abs(got[k] - ref[k]) <= 1e-10 * max(1.0, abs(ref[k])), (k, got[k], ref[k])
    np.testing.assert_allclose(got_nets, ref_nets, rtol=0, atol=1e-10)


def test_update_f32_close_to_oracle():
    kind = L.ENV_CARTPOLE
    d = _dims(kind)
    hp = _hp()
    pool = _pool(d, 150, 21)
    idx = np.random.RandomState(22).randint(0, 149, size=32)
    nets = _nets(d, 23, moments=True)
    _, got = _run_update(kind, False, hp, pool, idx, nets, 7)
    _, ref = K.do_training(d, nets, K.gather(pool, idx, 150), hp, 7)
    errs = {k: float(np.abs(np.asarray(got[k]) - ref[k]).max() / _scale(ref[k])) for k in ref}
    print("float32 do_training, max error / max(1, |ref|):", errs)
    # measured on an H100 80GB HBM3: grad 2.0e-8, q 3.1e-9, y 3.8e-8, qf_loss 5.4e-10, policy_surr 1.1e-11 (DESIGN §5)
    for k in ("grad", "q", "y", "qf_loss", "policy_surr"):
        assert errs[k] < 1e-6, (k, errs[k])


class _DeviceEnv(object):
    """The oracle's env callables on the device's own float32 env (b200rl_env_reset / b200rl_env_step)."""

    def __init__(self, kind, seed, run):
        self.kind, self.seed, self.run = kind, seed, run
        self.S = L.env_info(kind)["state_dim"]
        self.O = L.env_info(kind)["obs_dim"]

    def reset(self, itr):
        st = torch.empty((self.S, 1), dtype=torch.float32, device=DEV)
        o = torch.empty((self.O, 1), dtype=torch.float32, device=DEV)
        ops.env_reset(self.kind, 1, st, o, seed=self.seed, it=itr >> 28, row=itr & 0x0FFFFFFF, lane0=self.run)
        return st.cpu().numpy()[:, 0], o.cpu().numpy()[:, 0]

    def step(self, state, act):
        st = torch.tensor(np.asarray(state, np.float32).reshape(self.S, 1), device=DEV)
        o = torch.empty((self.O, 1), dtype=torch.float32, device=DEV)
        r = torch.empty(1, dtype=torch.float32, device=DEV)
        dn = torch.empty(1, dtype=torch.uint8, device=DEV)
        ops.env_step(self.kind, 1, st, torch.tensor(act.reshape(-1, 1), device=DEV), o, r, dn)
        return st.cpu().numpy()[:, 0], o.cpu().numpy()[:, 0], float(r.item()), bool(dn.item())


def _oracle_state(runs, r, d):
    s = runs.host_state()[r]
    return dict(nets=runs.nets[r].cpu().numpy().copy(), env_state=np.array(s.env_state[:8], np.float32),
                obs=np.array(s.obs[:d.O], np.float32), ou=np.array(s.ou_state[:d.A]), path_return=s.path_return,
                path_length=s.path_length, terminal=s.terminal, itr=s.itr, adam_t=s.adam_t,
                pool=dict(obs=runs.pool_obs[r].cpu().numpy().copy(), act=runs.pool_act[r].cpu().numpy().copy(),
                          rew=runs.pool_rew[r].cpu().numpy().copy(), term=runs.pool_term[r].cpu().numpy().copy()),
                top=s.top, bottom=s.bottom, size=s.size)


@pytest.mark.parametrize("name,es_kind,htt,mpl", [("cartpole", L.ES_OU, 0, 12), ("pendulum", L.ES_GAUSSIAN, 1, 30)])
def test_fused_loop_f64_per_step_parity(name, es_kind, htt, mpl):
    """n_steps = 1 launches from the device's own state, each compared with one oracle step from that state: loop
    counters, OU state, pool rows and parameters.  A 150-row pool, short paths and 320 steps cover terminal resets
    (CartPole), horizon cuts with and without their sample, the pool wrap and the full-pool rejection quirk."""
    kind = BOX_KINDS[name]
    d = _dims(kind)
    hp = _hp(es_kind=es_kind, include_horizon_terminal_transitions=htt, max_path_length=mpl)
    seed, run = 17, 0
    runs = ops.DdpgRuns(kind, d.O, d.A, 1, ops.ddpg_hparams(**hp), _nets(d, 19)[None], seed, DEV, f64=True,
                        es_cap=400)
    env = _DeviceEnv(kind, seed, run)
    stats = dict(es_returns=[], qf_loss=[], policy_surr=[], q=[], y=[])
    seen = dict(cut=0, done=0, wrap=False, quirk=False)
    for step in range(320):
        st = _oracle_state(runs, run, d)
        if st["terminal"] == 2:
            st["env_state"] = np.zeros(8, np.float32)
        st["env_state"] = st["env_state"][:env.S]
        rec = []
        K.train_step(d, st, hp, seed, run, env.reset, env.step, stats=stats, record=rec)
        runs.train(1)
        got = _oracle_state(runs, run, d)
        for k in ("path_length", "terminal", "itr", "adam_t", "top", "bottom", "size"):
            assert got[k] == st[k], (step, k, got[k], st[k])
        assert abs(got["path_return"] - st["path_return"]) <= 1e-9 * max(1.0, abs(st["path_return"])), step
        np.testing.assert_array_equal(got["obs"], st["obs"], err_msg="obs step %d" % step)
        np.testing.assert_array_equal(got["env_state"][:env.S], st["env_state"], err_msg="env step %d" % step)
        np.testing.assert_allclose(got["ou"], st["ou"], rtol=0, atol=1e-12)
        for k in ("obs", "act", "rew", "term"):
            np.testing.assert_array_equal(got["pool"][k], st["pool"][k], err_msg="pool %s step %d" % (k, step))
        np.testing.assert_allclose(got["nets"], st["nets"], rtol=0, atol=1e-10, err_msg="nets step %d" % step)
        if got["terminal"] and got["path_length"] >= hp["max_path_length"]:
            seen["cut"] += 1
        elif got["terminal"]:
            seen["done"] += 1
        seen["wrap"] |= got["size"] == hp["replay_pool_size"] and got["bottom"] > 0
        # the full-pool quirk: an update drew candidate size - 1 (not the newest row) and rejected it
        seen["quirk"] |= got["size"] == hp["replay_pool_size"] and any(
            rej and rej[0] == hp["replay_pool_size"] - 1 != (got["top"] - 1) % hp["replay_pool_size"]
            for _, _, rej in rec)
    assert seen["cut"] > 0 and seen["wrap"] and seen["quirk"], seen
    if name == "cartpole":
        assert seen["done"] > 0, seen
    s, es = runs.take_stats()
    assert int(s[0, 0]) == len(stats["qf_loss"]) and len(es[0]) == len(stats["es_returns"])
    np.testing.assert_allclose(es[0], stats["es_returns"], rtol=1e-12)
    np.testing.assert_allclose(s[0, 1], np.sum(stats["qf_loss"]), rtol=1e-9)
    np.testing.assert_allclose(s[0, 2], np.sum(stats["policy_surr"]), rtol=1e-9)
    np.testing.assert_allclose(s[0, 3], np.sum(np.concatenate(stats["q"])), rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(s[0, 5], np.sum(np.concatenate(stats["y"])), rtol=1e-9, atol=1e-12)


def _runs(kind, n_runs, f64, seed=31, hp=None, nets=None):
    d = _dims(kind)
    hp = hp or _hp()
    if nets is None:
        nets = np.stack([_nets(d, 100 + r) for r in range(n_runs)])
    return ops.DdpgRuns(kind, d.O, d.A, n_runs, ops.ddpg_hparams(**hp), nets, seed, DEV, f64=f64, es_cap=1)


def test_f32_loop_tracks_f64_over_a_short_horizon():
    kind = L.ENV_CARTPOLE
    a, b = _runs(kind, 1, False), _runs(kind, 1, True)
    a.train(80)
    b.train(80)
    (sa, _), (sb, _) = a.take_stats(), b.take_stats()
    assert sa[0, 0] == sb[0, 0] > 0
    np.testing.assert_allclose(sa[0, 1:8], sb[0, 1:8], rtol=1e-3, atol=1e-6)
    np.testing.assert_allclose(a.pool_obs.cpu().numpy(), b.pool_obs.cpu().numpy(), rtol=0, atol=1e-3)
    np.testing.assert_allclose(a.nets.cpu().numpy(), b.nets.cpu().numpy(), rtol=0, atol=1e-4)


@pytest.mark.parametrize("f64", [False, True])
def test_runs_are_independent_and_reruns_bit_identical(f64):
    kind = L.ENV_CARTPOLE
    n = 6
    together = _runs(kind, n, f64)
    together.train(120)
    again = _runs(kind, n, f64)
    again.train(120)
    assert torch.equal(together.nets, again.nets) and torch.equal(together.pool_obs, again.pool_obs)
    assert torch.equal(together.stats, again.stats) and torch.equal(together.state, again.state)
    d = _dims(kind)
    for r in (0, 4):
        # run r draws with run index r: launch it in a grid whose other runs are copies of it
        alone_grid = _runs(kind, r + 1, f64, nets=np.stack([_nets(d, 100 + r)] * (r + 1)))
        alone_grid.train(120)
        assert torch.equal(alone_grid.nets[r], together.nets[r])
        assert torch.equal(alone_grid.pool_obs[r], together.pool_obs[r])
        assert torch.equal(alone_grid.stats[r], together.stats[r])


def test_ddpg_example_run_task_and_tabular(tmp_path):
    """The run_task body of examples/ddpg_cartpole.py (import prefix changed, n_epochs reduced so that two epochs
    evaluate), then the tabular keys and the snapshot."""
    from rllab_b200.algos.ddpg import DDPG
    from rllab_b200.envs.box2d.cartpole_env import CartpoleEnv
    from rllab_b200.envs.normalized_env import normalize
    from rllab_b200.exploration_strategies.ou_strategy import OUStrategy
    from rllab_b200.policies.deterministic_mlp_policy import DeterministicMLPPolicy
    from rllab_b200.q_functions.continuous_mlp_q_function import ContinuousMLPQFunction
    from rllab_b200.misc import logger

    rows = []
    orig = logger.dump_tabular

    def capture(*a, **k):
        orig(*a, **k)
        rows.append(logger.get_last_table())

    logger.dump_tabular = capture
    try:
        env = normalize(CartpoleEnv())
        policy = DeterministicMLPPolicy(env_spec=env.spec, hidden_sizes=(32, 32))
        es = OUStrategy(env_spec=env.spec)
        qf = ContinuousMLPQFunction(env_spec=env.spec)
        algo = DDPG(env=env, policy=policy, es=es, qf=qf, batch_size=32, max_path_length=100, epoch_length=1000,
                    min_pool_size=10000, n_epochs=12, discount=0.99, scale_reward=0.01, qf_learning_rate=1e-3,
                    policy_learning_rate=1e-4)
        algo.train()
    finally:
        logger.dump_tabular = orig
    assert len(rows) == 12
    keys = {"Epoch", "AverageReturn", "StdReturn", "MaxReturn", "MinReturn", "AverageEsReturn", "StdEsReturn",
            "MaxEsReturn", "MinEsReturn", "AverageDiscountedReturn", "AverageQLoss", "AveragePolicySurr", "AverageQ",
            "AverageAbsQ", "AverageY", "AverageAbsY", "AverageAbsQYDiff", "AverageAction", "PolicyRegParamNorm",
            "QFunRegParamNorm"}
    # the pool reaches min_pool_size = 10000 at the last step of epoch 9: epochs 0-8 evaluate nothing
    for row in rows[:9]:
        assert not (keys & set(row)), row
    for epoch, row in zip(range(9, 12), rows[9:]):
        assert keys <= set(row), keys - set(row)
        assert row["Epoch"] == epoch
        assert all(np.isfinite(row[k]) for k in keys), row
        assert row["AverageQLoss"] >= 0 and row["AverageAbsQ"] >= abs(row["AverageQ"]) - 1e-12
    snap = algo.get_epoch_snapshot(11)
    assert set(snap) == {"env", "epoch", "qf", "policy", "target_qf", "target_policy", "es"}
    assert np.isfinite(algo.last_eval_returns).all()
    assert algo.runs.host_state()[0].itr == 12000


CURVE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "oracle_cartpole_ddpg_curve.json")


def _whole_path_returns(b):
    t = b.to_numpy()
    rew, flags = t["rew"], t["flags"]
    out = []
    for n in range(b.N):
        acc = 0.0
        for step in range(b.T):
            acc += float(rew[step, n])
            if flags[step, n] & L.FLAG_END:
                if not flags[step, n] & L.FLAG_CUT:
                    out.append(acc)
                acc = 0.0
    return out


def test_example_learns_within_the_oracle_band():
    """The example's configuration (tests/golden/make_cartpole_ddpg_curve.py) with the oracle's five seeds as five runs
    in one launch.  The streams differ (float32 env, run-indexed Philox draws), so bands, not values: at every evaluated
    epoch the runs' mean within the oracle's range at that epoch widened by its spread, and over the last five epochs a
    mean across runs of at least the lowest seed's mean; every run's best epoch at least the lowest seed's best less the
    seeds' spread."""
    import json
    cfg_all = json.load(open(CURVE))
    cfg = cfg_all["config"]
    curves = {int(s): {int(e): v for e, v in c.items()} for s, c in cfg_all["AverageReturn"].items()}
    seeds = sorted(curves)
    epochs = sorted(curves[seeds[0]])
    band = np.array([[curves[s][e] for e in epochs] for s in seeds])   # [seed][evaluated epoch]
    lo, hi = band.min(0), band.max(0)
    d = K.Dims(4, 1)
    nets = []
    for s in seeds:
        rng = np.random.RandomState(s)
        th = np.concatenate([K.init_params(d.pshapes, rng), K.init_params(d.qshapes, rng)])
        nets.append(np.stack([th, 0 * th, 0 * th, th]))
    hp = {k: cfg[k] for k in _hp()}
    runs = ops.DdpgRuns(L.ENV_CARTPOLE, 4, 1, len(seeds), ops.ddpg_hparams(**hp), np.stack(nets), 1, DEV)
    T = cfg["max_path_length"]
    N = -(-cfg["eval_samples"] // T)
    got = np.zeros((len(seeds), len(epochs)))
    for epoch in range(cfg["n_epochs"]):
        runs.train(cfg["epoch_length"])
        runs.take_stats()
        if epoch in epochs:
            for r in range(len(seeds)):
                b = ops.LaneBatch(4, 1, N, T, DEV)
                p32 = runs.nets[r, 0, :d.PP].float().contiguous()
                ops.rollout_deterministic(L.ENV_CARTPOLE, p32, b, T, seed=2, it=epoch, lane0=r * N)
                got[r, epochs.index(epoch)] = np.mean(_whole_path_returns(b))
    print("GPU AverageReturn per evaluated epoch:", np.round(got, 1).tolist())
    print("oracle band:", np.round(lo, 1).tolist(), np.round(hi, 1).tolist())
    # the runs' mean at each epoch within the seeds' range widened by its spread, at least 10 % of the band's top (epoch
    # 9 evaluates the initial policy: five nearly equal values, whose spread says nothing of the eval draws' noise).  A
    # single run swings by several hundred between epochs once it has learned (the oracle's own seeds do, e.g. seed 4
    # from 1000 to 557 within five epochs), so one run at one epoch is not held to a five-seed range.
    width = np.maximum(hi - lo, 0.1 * hi)
    mean = got.mean(0)
    assert (mean >= lo - width).all() and (mean <= hi + width).all(), (mean, lo - width, hi + width)
    best = band.max(1)
    assert (got.max(1) >= best.min() - (best.max() - best.min())).all()   # every run learns
    late = band[:, -5:].mean(1)
    assert got[:, -5:].mean() >= late.min()                              # and the runs' late mean holds up
