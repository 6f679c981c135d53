"""GPU: DDPG (rllab_b200/csrc/ddpg.cu) against the float64 oracle tests/ddpg_oracle.py over the grid the kernels are
compiled for -- b200rl_ddpg_update at every classic-control Box kind in both precisions, at Adam step 1 and 7 and at
saturated and nearly saturated tanh outputs; the fused train loop step by step at every kind in float64 and at Point and
DoublePendulum in float32, with several updates per sample, both exploration strategies, ou_mu != 0, clipped actions,
the step counter crossing 2^28 and a full 10^6-row pool; launch splits and a three-wave grid of runs; the evaluation
heads at odd sizes and lane offsets; and the mapping of DDPG's arguments onto b200rl_ddpg_hparams.

The float32 bounds are the worst errors measured on an H100 80GB HBM3 times about four (DESIGN §5, DDPG)."""
import numpy as np
import pytest
import torch

import ddpg_oracle as K
from ddpg_device import BOX_KINDS, DEV, _DeviceEnv, _dims, _hp, _nets, _oracle_state, _run_update
from oracle import envs as E
from oracle import philox as PH
from rllab_b200 import _lib as L
from rllab_b200 import ops

pytestmark = pytest.mark.gpu

KINDS = sorted(BOX_KINDS)
F32_EPS = float(np.finfo(np.float32).eps)
# float32 bounds, block-relative: max |device - oracle| / max |oracle|, the worst measured on an H100 80GB HBM3 (DESIGN
# §5, DDPG) in the comment
F32_QGRAD = 1e-6           # Q gradient of one update, 2.5e-7
F32_PGRAD = 2.5e-6         # policy gradient, 3.5e-7 in one update, 5.9e-7 in the float32 loop
F32_QY = 2e-6              # q 5.1e-7, y 4.6e-8
F32_LOSS = 3e-7            # qf_loss 1.7e-8, policy_surr 7.6e-8 (relative to |ref|)
F32_LOOP_QGRAD = 3.5e-5    # Q gradient in the float32 loop, 8.4e-6: y - q shrinks as the critic fits
F32_ACTION = 4e-7          # |device action - clip(mu_oracle + noise)|, absolute, 1.05e-7


def _rel(got, ref):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    err, scale = np.abs(got - ref).max(), np.abs(ref).max()
    return float(err / scale) if scale > 0 else (0.0 if err == 0 else np.inf)


def _decay(d, theta, hp):
    """The weight decay terms of the gradient ([policy | qf]), exact in both precisions (float64 on the device)."""
    wd = np.where(np.arange(d.P) < d.PP, hp["policy_weight_decay"], hp["qf_weight_decay"])
    return wd * theta * d.weight_mask()


def _actor(d, theta_p, theta_q, s, hp):
    """The actor half of do_training on a given critic: the policy gradient (with weight decay) and policy_surr."""
    a1, a2, mu = K.pi_forward(d, theta_p, s)
    px1, px2, pq = K.q_forward(d, theta_q, s, mu)
    _, dmu = K.q_backward(d, theta_q, s, px1, px2, np.full(K.BATCH, -1.0 / K.BATCH))
    g = K.pi_backward(d, theta_p, s, a1, a2, mu, dmu) + hp["policy_weight_decay"] * theta_p * d.weight_mask()[:d.PP]
    return g, -np.mean(pq)


def _adam_and_target(d, nets, g, hp, t):
    """theta, m, v, target after one Adam step on the gradient g (weight decay included) and the soft update."""
    th, m, v, tg = [x.copy() for x in nets]
    for sl, lr in ((slice(0, d.PP), hp["policy_learning_rate"]), (slice(d.PP, d.P), hp["qf_learning_rate"])):
        th[sl], m[sl], v[sl] = K.adam(th[sl], m[sl], v[sl], g[sl], lr, t)
    return np.stack([th, m, v, K.soft_update(tg, th, hp["soft_target_tau"])])


def _update_pool(d, rows, seed, scale_reward):
    """Rewards on Pendulum's scale (per-step reward down to about -16, times scale_reward), a quarter terminal rows."""
    rng = np.random.RandomState(seed)
    return dict(obs=rng.randn(rows, d.O).astype(np.float32), act=rng.uniform(-1, 1, (rows, d.A)).astype(np.float32),
                rew=(scale_reward * rng.uniform(-16.3, 0.0, rows)).astype(np.float32),
                term=(rng.rand(rows) < 0.25).astype(np.uint8))


def _update_case(name, t, seed):
    kind = BOX_KINDS[name]
    d = _dims(kind)
    hp = _hp(scale_reward=0.1, qf_weight_decay=0.01, policy_weight_decay=0.02)
    pool = _update_pool(d, 150, seed, hp["scale_reward"])
    idx = np.random.RandomState(seed + 1).randint(0, 150, size=32)
    idx[0] = 149                                   # s' of the last row is row 0
    nets = _nets(d, seed + 2, moments=t > 1)
    return kind, d, hp, pool, idx, nets


def _check_update_f64(d, hp, pool, idx, nets, t, got_nets, got):
    ref_nets, ref = K.do_training(d, nets, K.gather(pool, idx, 150), hp, t)
    for k in ("grad", "q", "y"):
        np.testing.assert_allclose(got[k], ref[k], rtol=0, atol=1e-10 * max(1.0, np.abs(ref[k]).max()), err_msg=k)
    for k in ("qf_loss", "policy_surr"):
        assert abs(got[k] - ref[k]) <= 1e-10 * max(1.0, abs(ref[k])), (k, got[k], ref[k])
    np.testing.assert_allclose(got_nets, ref_nets, rtol=0, atol=1e-10)


def _update_errors_f32(d, hp, pool, idx, nets, t, got_nets, got):
    """Block-relative float32 errors of one update, the gradients without their exact weight decay terms (which would
    otherwise set the policy block's scale).  The Q block, q, y and qf_loss against the oracle; the policy block
    and policy_surr against the oracle's actor pass on the device's own updated critic, so that a float32 Adam step
    whose sign flipped on a gradient entry at float32's noise floor (a 2 lr move of that critic entry) is not charged
    to the actor's gradient."""
    batch = K.gather(pool, idx, 150)
    _, ref = K.do_training(d, nets, batch, hp, t)
    gp, surr = _actor(d, nets[0][:d.PP], got_nets[0][d.PP:], batch["s"], hp)
    wd = _decay(d, nets[0], hp)
    errs = dict(qgrad=_rel(got["grad"][d.PP:] - wd[d.PP:], ref["grad"][d.PP:] - wd[d.PP:]),
                pgrad=_rel(got["grad"][:d.PP] - wd[:d.PP], gp - wd[:d.PP]),
                q=_rel(got["q"], ref["q"]), y=_rel(got["y"], ref["y"]),
                qf_loss=abs(got["qf_loss"] - ref["qf_loss"]) / abs(ref["qf_loss"]),
                policy_surr=abs(got["policy_surr"] - surr) / abs(surr))
    # Adam and the target update in float64 on the device's own gradient: exact up to rounding
    np.testing.assert_allclose(got_nets, _adam_and_target(d, nets, got["grad"], hp, t), rtol=0, atol=1e-12)
    return errs


@pytest.mark.parametrize("t", [1, 7])
@pytest.mark.parametrize("f64", [True, False])
@pytest.mark.parametrize("name", KINDS)
def test_update_matches_oracle_at_every_kind(name, f64, t):
    """b200rl_ddpg_update at Adam step 1 from zero moments and step 7 with moments, weight decay on both nets, terminal
    rows and rewards on Pendulum's scale."""
    kind, d, hp, pool, idx, nets = _update_case(name, t, 40 + 7 * t)
    got_nets, got = _run_update(kind, f64, hp, pool, idx, nets, t)
    if f64:
        _check_update_f64(d, hp, pool, idx, nets, t, got_nets, got)
        return
    errs = _update_errors_f32(d, hp, pool, idx, nets, t, got_nets, got)
    print("float32 update %s t=%d, block-relative errors:" % (name, t), errs)
    assert errs["qgrad"] < F32_QGRAD and errs["pgrad"] < F32_PGRAD, errs
    assert errs["q"] < F32_QY and errs["y"] < F32_QY, errs
    assert errs["qf_loss"] < F32_LOSS and errs["policy_surr"] < F32_LOSS, errs


# Pre-activations of the policy's tanh outputs: +-25 (tanh exactly +-1 in float32 and float64) and +-4 (1 - mu^2 about
# 1.3e-3, resolved by float32 to about eps / 1.3e-3).  At Point one output saturates and the other does not.
SATURATION = [("point", (25.0, 4.0)), ("point", (-4.0, -25.0)), ("pendulum", (25.0,)), ("pendulum", (-4.0,)),
              ("cartpole_swingup", (4.0,)), ("double_pendulum", (-25.0,))]


@pytest.mark.parametrize("f64", [True, False])
@pytest.mark.parametrize("name,pre", SATURATION)
def test_update_at_saturated_actions(name, pre, f64):
    kind, d, hp, pool, idx, nets = _update_case(name, 7, 71)
    PB2, PW2 = d.PP - d.A, d.PP - d.A - 32 * d.A
    for n in (0, 3):                                # theta and target: small output weights, bias at the pre-activation
        nets[n][PB2:d.PP] = pre
    batch = K.gather(pool, idx, 150)
    _, a2, _ = K.pi_forward(d, nets[0][:d.PP], batch["s"])
    z = a2 @ nets[0][PW2:PB2].reshape(32, d.A) + nets[0][PB2:d.PP]
    sat = np.abs(np.asarray(pre)) > 20
    assert (np.abs(z[:, sat]) > 20).all() and (np.abs(z[:, ~sat]) < 6).all(), z
    got_nets, got = _run_update(kind, f64, hp, pool, idx, nets, 7)
    assert np.isfinite(got_nets).all() and np.isfinite(got["grad"]).all()
    # no gradient passes a saturated output: its output-layer column and bias carry the weight decay term only
    w = got["grad"][PW2:PB2].reshape(32, d.A)
    np.testing.assert_array_equal(w[:, sat], hp["policy_weight_decay"] * nets[0][PW2:PB2].reshape(32, d.A)[:, sat])
    np.testing.assert_array_equal(got["grad"][PB2:d.PP][sat], 0.0)
    if f64:
        _check_update_f64(d, hp, pool, idx, nets, 7, got_nets, got)
        return
    errs = _update_errors_f32(d, hp, pool, idx, nets, 7, got_nets, got)
    # float32 resolves 1 - mu^2 to about eps / (1 - mu^2) relative, 9e-5 at a pre-activation of 4: the bound near
    # saturation (measured worst 0.21 of it).  With every output saturated the policy's loss gradient is exactly 0.
    one_m = 1.0 - np.tanh(z[:, ~sat]) ** 2
    res = F32_EPS / one_m.min() if one_m.size else 0.0
    print("float32 saturated update %s pre=%s: errors %s, eps / min(1 - mu^2) = %.2e" % (name, pre, errs, res))
    assert errs["qgrad"] < F32_QGRAD and errs["pgrad"] < max(F32_PGRAD, res), errs
    assert errs["q"] < F32_QY and errs["y"] < F32_QY, errs


# ---------------------------------------------------------------- the fused loop, step by step from the device's state
def _runs(kind, n_runs, f64, hp, nets, seed=31, es_cap=1):
    d = _dims(kind)
    return ops.DdpgRuns(kind, d.O, d.A, n_runs, ops.ddpg_hparams(**hp), nets, seed, DEV, f64=f64, es_cap=es_cap)


def _oracle_from_device(runs, run, d, env):
    st = _oracle_state(runs, run, d)
    if st["terminal"] == 2:
        st["env_state"] = np.zeros(8, np.float32)
    st["env_state"] = st["env_state"][:env.S]
    return st


def _assert_loop_state(got, st, env, step):
    """Counters, env state, OU state and pool rows of the device after one step against the oracle's."""
    for k in ("path_length", "terminal", "itr", "adam_t", "top", "bottom", "size"):
        assert got[k] == st[k], (step, k, got[k], st[k])
    assert abs(got["path_return"] - st["path_return"]) <= 1e-9 * max(1.0, abs(st["path_return"])), step
    np.testing.assert_array_equal(got["obs"], st["obs"], err_msg="obs step %d" % step)
    np.testing.assert_array_equal(got["env_state"][:env.S], st["env_state"], err_msg="env step %d" % step)
    # the oracle's Box-Muller takes cos / sin of 2 pi u, the kernel sincospi(2 u): last-bit differences
    np.testing.assert_allclose(got["ou"], st["ou"], rtol=0, atol=1e-12, err_msg="ou step %d" % step)
    for k in ("obs", "act", "rew", "term"):
        np.testing.assert_array_equal(got["pool"][k], st["pool"][k], err_msg="pool %s step %d" % (k, step))


def _note(seen, got, hp, rec, added_act):
    rows = hp["replay_pool_size"]
    if got["terminal"] and got["path_length"] >= hp["max_path_length"]:
        seen["cut"] += 1
    elif got["terminal"]:
        seen["done"] += 1
    seen["wrap"] |= got["size"] == rows and got["bottom"] > 0
    seen["quirk"] |= got["size"] == rows and any(
        rej and rej[0] == rows - 1 != (got["top"] - 1) % rows for _, _, rej in rec)
    seen["clip"] += int(added_act is not None and (np.abs(added_act) == 1.0).any())
    seen["updates"] += len(rec)


def _f64_loop(kind, hp, n_steps, seed=17, prepare=None, check=None):
    """n_steps single-step launches of a float64 run, each against one oracle step from the device's state."""
    d = _dims(kind)
    runs = _runs(kind, 1, True, hp, _nets(d, 19)[None], seed=seed, es_cap=n_steps + 1)
    if prepare is not None:
        prepare(runs, d)
    env = _DeviceEnv(kind, seed, 0)
    stats = dict(es_returns=[], qf_loss=[], policy_surr=[], q=[], y=[])
    seen = dict(cut=0, done=0, wrap=False, quirk=False, clip=0, updates=0)
    for step in range(n_steps):
        st = _oracle_from_device(runs, 0, d, env)
        top, size0 = st["top"], st["size"]
        rec = []
        K.train_step(d, st, hp, seed, 0, env.reset, env.step, stats=stats, record=rec)
        runs.train(1)
        got = _oracle_from_device(runs, 0, d, env)
        _assert_loop_state(got, st, env, step)
        np.testing.assert_allclose(got["nets"], st["nets"], rtol=0, atol=1e-10, err_msg="nets step %d" % step)
        added = got["top"] != top or got["size"] != size0
        _note(seen, got, hp, rec, got["pool"]["act"][top] if added else None)
        if check is not None:
            check(step, got, rec)
    return runs, stats, seen


LOOP_CASES = {
    "point": dict(es_kind=L.ES_OU, ou_mu=0.2, ou_sigma=0.5, n_updates_per_sample=3,
                  include_horizon_terminal_transitions=1, max_path_length=25),
    "cartpole": dict(es_kind=L.ES_GAUSSIAN, gs_decay_period=150.0, n_updates_per_sample=1, max_path_length=12),
    "pendulum": dict(es_kind=L.ES_OU, ou_mu=-0.2, ou_sigma=0.6, n_updates_per_sample=3, max_path_length=20),
    "cartpole_swingup": dict(es_kind=L.ES_GAUSSIAN, gs_max_sigma=1.5, gs_decay_period=100.0, n_updates_per_sample=3,
                             include_horizon_terminal_transitions=1, max_path_length=30),
    "double_pendulum": dict(es_kind=L.ES_OU, ou_mu=0.2, ou_sigma=0.6, n_updates_per_sample=1,
                            include_horizon_terminal_transitions=1, max_path_length=15),
}


@pytest.mark.parametrize("name", KINDS)
def test_fused_loop_f64_per_step_at_every_kind(name):
    """320 one-step launches against one oracle step each: 1 or 3 updates per sample, OU with ou_mu != 0 and sigma
    large enough to clip, Gaussian with its sigma decaying to the floor within the run (decay periods 100 and 150),
    horizon samples kept and dropped, the wrap of a 150-row pool and the full-pool rejection quirk."""
    kind = BOX_KINDS[name]
    hp = _hp(**LOOP_CASES[name])
    runs, stats, seen = _f64_loop(kind, hp, 320)
    assert seen["cut"] > 0 and seen["wrap"] and seen["quirk"], seen
    if name == "cartpole":
        assert seen["done"] > 0, seen
    if hp["es_kind"] == L.ES_OU:
        assert seen["clip"] > 0, seen                 # OU noise pushed mu + x past +-1: the pool holds +-1.0f
    s, es = runs.take_stats()
    assert int(s[0, 0]) == len(stats["qf_loss"]) == seen["updates"] and len(es[0]) == len(stats["es_returns"])
    np.testing.assert_allclose(es[0], stats["es_returns"], rtol=1e-12)
    np.testing.assert_allclose(s[0, 1], np.sum(stats["qf_loss"]), rtol=1e-9)
    np.testing.assert_allclose(s[0, 2], np.sum(stats["policy_surr"]), rtol=1e-9)
    np.testing.assert_allclose(s[0, 3], np.sum(np.concatenate(stats["q"])), rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(s[0, 5], np.sum(np.concatenate(stats["y"])), rtol=1e-9, atol=1e-12)


def _prefill(runs, d, size, top, bottom, seed):
    """Random pool rows 0 .. size - 1 (terminal one in five) and the pool pointers, written straight into the run."""
    rng = np.random.RandomState(seed)
    rows = runs.pool_rew.shape[1]
    runs.pool_obs[0, :size] = torch.tensor(rng.randn(size, d.O).astype(np.float32))
    runs.pool_act[0, :size] = torch.tensor(rng.uniform(-1, 1, (size, d.A)).astype(np.float32))
    runs.pool_rew[0, :size] = torch.tensor((0.1 * rng.randn(size)).astype(np.float32))
    runs.pool_term[0, :size] = torch.tensor((rng.rand(size) < 0.2).astype(np.uint8))
    st = runs.host_state()
    st[0].top, st[0].bottom, st[0].size = top % rows, bottom, size
    return st


def test_fused_loop_f64_across_itr_2_28():
    """itr from 2^28 - 40 to 2^28 + 40: the Philox key's high word changes from 0 to 1 mid-run, with resets and updates
    on both sides (the pool starts with 100 rows so that updates run from the first step)."""
    kind = L.ENV_CARTPOLE
    hp = _hp(n_updates_per_sample=2, max_path_length=10, include_horizon_terminal_transitions=1)
    start = 2 ** 28 - 40

    def prepare(runs, d):
        st = _prefill(runs, d, 100, 100, 0, 5)
        st[0].itr = start
        runs.set_host_state(st)

    sides = dict(reset=[0, 0], update=[0, 0])

    def check(step, got, rec):
        side = int(got["itr"] - 1 >= 2 ** 28)
        sides["update"][side] += len(rec)
        sides["reset"][side] += int(got["path_length"] == 1)

    _, _, seen = _f64_loop(kind, hp, 80, prepare=prepare, check=check)
    assert min(sides["update"]) > 0 and min(sides["reset"]) > 0, sides


def test_fused_loop_f64_full_wrapped_million_row_pool():
    """replay_pool_size = 10^6, the pool full and wrapped (top = bottom != 0), two updates per sample: index draws over
    the whole pool from a non-zero bottom, the bottom advancing with every sample."""
    kind = L.ENV_POINT
    rows = 10 ** 6
    hp = _hp(replay_pool_size=rows, min_pool_size=1000, n_updates_per_sample=2, include_horizon_terminal_transitions=1)

    def prepare(runs, d):
        runs.set_host_state(_prefill(runs, d, rows, 654321, 654321, 6))

    def check(step, got, rec):
        assert got["size"] == rows and got["bottom"] == (654321 + step + 1) % rows and len(rec) == 2
        assert any((idx < 654321).any() for idx, _, _ in rec) and any((idx > 654321).any() for idx, _, _ in rec)

    _f64_loop(kind, hp, 12, prepare=prepare, check=check)


def test_fused_loop_without_updates():
    """n_updates_per_sample = 0: the loop fills the pool and ends paths but never trains."""
    kind = L.ENV_PENDULUM
    d = _dims(kind)
    hp = _hp(n_updates_per_sample=0, include_horizon_terminal_transitions=1, max_path_length=20)
    nets = _nets(d, 19)[None]
    for f64 in (True, False):
        runs = _runs(kind, 1, f64, hp, nets)
        runs.train(100)
        s, es = runs.take_stats()
        st = runs.host_state()[0]
        assert (s[0, :8] == 0).all() and len(es[0]) == 4 and st.adam_t == 0 and st.size == 100, (s, st.size)
        np.testing.assert_array_equal(runs.nets[0].cpu().numpy(), nets[0])


@pytest.mark.parametrize("name,es_kind", [("point", L.ES_OU), ("double_pendulum", L.ES_GAUSSIAN)])
def test_fused_loop_f32_per_step(name, es_kind):
    """Float32 one-step launches from the device's own state.  Every sample is stored, so the device's action is read
    from the pool: it lies within F32_ACTION of the oracle's clip(mu + noise); stepping the oracle's env with it gives
    bit-identical env state, pool rows and counters.  The device's gradient is recovered from its float64 Adam
    moments, g = (m_new - 0.9 m_old) / 0.1, and held to the oracle's at the update's block-relative bounds; theta, v
    and the target follow from it by Adam and the soft update."""
    kind = BOX_KINDS[name]
    d = _dims(kind)
    hp = _hp(es_kind=es_kind, ou_mu=0.1, ou_sigma=0.5, gs_decay_period=100.0, n_updates_per_sample=1,
             include_horizon_terminal_transitions=1, max_path_length=25)
    seed = 23
    runs = _runs(kind, 1, False, hp, _nets(d, 29)[None], seed=seed, es_cap=400)
    env = _DeviceEnv(kind, seed, 0)
    worst = dict(action=0.0, qgrad=0.0, pgrad=0.0)
    seen = dict(cut=0, done=0, wrap=False, quirk=False, clip=0, updates=0)
    for step in range(200):
        st = _oracle_from_device(runs, 0, d, env)
        nets0 = st["nets"].copy()
        top = st["top"]
        runs.train(1)
        got = _oracle_from_device(runs, 0, d, env)
        act = got["pool"]["act"][top].copy()
        rec, explored = [], []
        K.train_step(d, st, hp, seed, 0, env.reset, env.step, record=rec, action=act, explored=explored)
        _assert_loop_state(got, st, env, step)
        worst["action"] = max(worst["action"], float(np.abs(act - explored[0]).max()))
        _note(seen, got, hp, rec, act)
        if not rec:
            np.testing.assert_array_equal(got["nets"], nets0)
            continue
        (idx, info, _), = rec
        t = got["adam_t"]
        th0, m0, v0, tg0 = nets0
        th1, m1, v1, tg1 = got["nets"]
        g = (m1 - K.B1 * m0) / (1.0 - K.B1)
        batch = K.gather(st["pool"], idx, hp["replay_pool_size"])
        gp, _ = _actor(d, th0[:d.PP], th1[d.PP:], batch["s"], hp)
        wd = _decay(d, th0, hp)
        worst["qgrad"] = max(worst["qgrad"], _rel(g[d.PP:] - wd[d.PP:], info["grad"][d.PP:] - wd[d.PP:]))
        worst["pgrad"] = max(worst["pgrad"], _rel(g[:d.PP] - wd[:d.PP], gp - wd[:d.PP]))
        np.testing.assert_allclose(v1, K.B2 * v0 + (1.0 - K.B2) * g * g, rtol=1e-9, atol=1e-15, err_msg="v %d" % step)
        for sl, lr in ((slice(0, d.PP), hp["policy_learning_rate"]), (slice(d.PP, d.P), hp["qf_learning_rate"])):
            a_t = lr * np.sqrt(1.0 - K.B2 ** t) / (1.0 - K.B1 ** t)
            np.testing.assert_allclose(th1[sl], th0[sl] - a_t * m1[sl] / (np.sqrt(v1[sl]) + K.EPS), rtol=0,
                                       atol=1e-12, err_msg="theta step %d" % step)
        np.testing.assert_allclose(tg1, K.soft_update(tg0, th1, hp["soft_target_tau"]), rtol=0, atol=1e-12)
    print("float32 loop %s, worst over 200 steps:" % name, worst, seen)
    assert seen["updates"] > 100 and seen["cut"] > 0 and seen["wrap"], seen
    if es_kind == L.ES_OU:
        assert seen["clip"] > 0, seen
    assert worst["action"] < F32_ACTION and worst["qgrad"] < F32_LOOP_QGRAD and worst["pgrad"] < F32_PGRAD, worst


# ---------------------------------------------------------------- launch splits and grids
def _split_hp():
    return _hp(es_kind=L.ES_OU, ou_mu=0.1, n_updates_per_sample=2, include_horizon_terminal_transitions=1,
               max_path_length=23)


def _same_runs(a, b, runs=slice(None)):
    for x, y in ((a.nets, b.nets), (a.pool_obs, b.pool_obs), (a.pool_act, b.pool_act), (a.pool_rew, b.pool_rew),
                 (a.pool_term, b.pool_term), (a.stats, b.stats)):
        if not torch.equal(x[runs], y[runs]):
            return False
    state = lambda r: r.state.view(r.n_runs, -1)[runs]
    return torch.equal(state(a), state(b))


@pytest.mark.parametrize("f64", [False, True])
@pytest.mark.parametrize("name", ["point", "double_pendulum"])
def test_launch_splits_are_bit_identical(name, f64):
    """train(320) in one launch against 320 one-step launches and against splits at the first update (size reaches
    min_pool_size = 40 at step 39), mid-path, at a terminal step and at the pool wrap (step 150); the same splits with
    take_stats between launches add up to the one launch's statistics and Es returns."""
    kind = BOX_KINDS[name]
    d = _dims(kind)
    hp = _split_hp()
    nets = _nets(d, 41)[None]
    one = _runs(kind, 1, f64, hp, nets)
    one.train(320)
    steps = _runs(kind, 1, f64, hp, nets)
    terminal = []
    for i in range(320):
        steps.train(1)
        if steps.host_state()[0].terminal:
            terminal.append(i + 1)
    assert _same_runs(one, steps)
    cuts = sorted({39, 40, 101, terminal[3], terminal[3] + 1, 149, 150, 151, 320})
    assert terminal[3] not in (39, 40, 101, 149, 150, 151)
    split = _runs(kind, 1, f64, hp, nets)
    taken = _runs(kind, 1, f64, hp, nets)
    sums, es = np.zeros(L.DDPG_NSTAT), []
    prev = 0
    for c in cuts:
        split.train(c - prev)
        taken.train(c - prev)
        s, e = taken.take_stats()
        sums += s[0]
        es.extend(e[0])
        prev = c
    assert _same_runs(one, split)
    s_one, es_one = one.take_stats()
    np.testing.assert_array_equal(np.asarray(es), es_one[0])
    assert sums[0] == s_one[0, 0] > 0 and sums[8] == s_one[0, 8] == len(es_one[0]) > 0
    np.testing.assert_allclose(sums[1:8], s_one[0, 1:8], rtol=1e-12, atol=1e-15)
    for a, b in ((taken.nets, one.nets), (taken.pool_obs, one.pool_obs), (taken.pool_act, one.pool_act)):
        assert torch.equal(a, b)


@pytest.mark.parametrize("f64", [False, True])
def test_three_wave_grid_runs_are_independent(f64):
    """300 runs in one launch (one CTA per SM: three waves on 132 SMs): runs 0, 131, 132 and 299 each equal the same run
    in a grid whose other members are copies of it."""
    kind = L.ENV_DOUBLE_PENDULUM
    d = _dims(kind)
    hp = _split_hp()
    nets = np.stack([_nets(d, 100 + r) for r in range(300)])
    together = _runs(kind, 300, f64, hp, nets)
    together.train(100)
    assert together.host_state()[299].adam_t > 0
    for r in (0, 131, 132, 299):
        alone = _runs(kind, r + 1, f64, hp, np.stack([nets[r]] * (r + 1)))
        alone.train(100)
        for x, y in ((alone.nets, together.nets), (alone.pool_obs, together.pool_obs), (alone.stats, together.stats),
                     (alone.pool_act, together.pool_act)):
            assert torch.equal(x[r], y[r]), r
        assert torch.equal(alone.state.view(r + 1, -1)[r], together.state.view(300, -1)[r]), r


# ---------------------------------------------------------------- evaluation heads
# n = 2^20 + 3 at the smallest and the largest observation
@pytest.mark.parametrize("name,n", [(k, n) for k in KINDS for n in (1, 127, 129)] +
                         [("point", 2 ** 20 + 3), ("double_pendulum", 2 ** 20 + 3)])
def test_get_actions_get_qval_at_odd_sizes(name, n):
    kind = BOX_KINDS[name]
    d = _dims(kind)
    th32 = _nets(d, 3)[0].astype(np.float32)
    rng = np.random.RandomState(n)
    obs = rng.randn(n, d.O).astype(np.float32)
    act = rng.uniform(-1, 1, size=(n, d.A)).astype(np.float32)
    o = torch.tensor(np.ascontiguousarray(obs.T), device=DEV)
    a = torch.tensor(np.ascontiguousarray(act.T), device=DEV)
    mu = torch.full((d.A, n), np.nan, dtype=torch.float32, device=DEV)
    q = torch.full((n,), np.nan, dtype=torch.float32, device=DEV)
    ops.deterministic_get_actions(torch.tensor(th32[:d.PP], device=DEV), d.O, d.A, o, n, mu)
    ops.qf_get_qval(torch.tensor(th32[d.PP:], device=DEV), d.O, d.A, o, a, n, q)
    _, _, ref_mu = K.pi_forward(d, th32[:d.PP].astype(np.float64), obs.astype(np.float64))
    _, _, ref_q = K.q_forward(d, th32[d.PP:].astype(np.float64), obs.astype(np.float64), act.astype(np.float64))
    np.testing.assert_allclose(mu.cpu().numpy().T, ref_mu, rtol=0, atol=2e-6)
    np.testing.assert_allclose(q.cpu().numpy(), ref_q, rtol=0, atol=2e-6 * max(1.0, np.abs(ref_q).max()))


@pytest.mark.parametrize("given_raw", [False, True])
@pytest.mark.parametrize("name", KINDS)
def test_deterministic_rollout_at_a_lane_offset(name, given_raw):
    """N = 300 lanes from lane0 = 1000, T = 60 > max_path_length = 25: every path start's observation is the oracle's
    reset from the raw draws of its lane (raw_block at lane0 + n, or the given reset_raw row), the actions are the
    oracle policy's, and the transitions replay on b200rl_env_step."""
    kind = BOX_KINDS[name]
    d = _dims(kind)
    env32 = E.make(name, np.float32)
    N, T, mpl, lane0, seed, it = 300, 60, 25, 1000, 7, 5
    p32 = torch.tensor(_nets(d, 5)[0][:d.PP].astype(np.float32), device=DEV)
    if given_raw:
        rng = np.random.RandomState(8)
        raw = (rng.rand(T + 1, env32.K, N) if env32.noise_kind == "uniform" else rng.randn(T + 1, env32.K, N))
        raw = raw.astype(np.float32)
        rr = torch.tensor(raw, device=DEV)
    else:
        words = PH.raw_block(T + 1, 0, env32.K + env32.K % 2, N, lane0, seed, it, 1)
        raw = PH.uniform_from_raw(words) if env32.noise_kind == "uniform" else PH.normal_from_raw(words)
        raw, rr = raw[:, :env32.K], None
    b = ops.LaneBatch(d.O, d.A, N, T, DEV)
    ops.rollout_deterministic(kind, p32, b, mpl, reset_raw=rr, seed=seed, it=it, lane0=lane0)
    t = b.to_numpy()
    obs, act, rew, flags = t["obs"], t["act"], t["rew"], t["flags"]
    starts = np.zeros((T, N), bool)
    starts[0] = True
    starts[1:] = (flags[:-1] & L.FLAG_END) > 0
    assert starts[1:].sum() >= N * (T // mpl)
    exact = given_raw or env32.noise_kind == "uniform"
    for step in range(T):
        lanes = np.nonzero(starts[step])[0]
        ref = env32.obs(env32.reset(np.asarray(raw[step][:, lanes], np.float32)))
        tol = dict(rtol=0, atol=1e-6) if exact else dict(rtol=5e-5, atol=2e-5)
        np.testing.assert_allclose(obs[:, step, lanes], ref, err_msg="reset obs at step %d" % step, **tol)
    _, _, ref_mu = K.pi_forward(d, p32.cpu().numpy().astype(np.float64),
                                obs.transpose(1, 2, 0).reshape(-1, d.O).astype(np.float64))
    np.testing.assert_allclose(act.transpose(1, 2, 0).reshape(-1, d.A), ref_mu, rtol=0, atol=2e-6)
    S = L.env_info(kind)["state_dim"]
    state = torch.empty((S, N), dtype=torch.float32, device=DEV)
    o = torch.empty((d.O, N), dtype=torch.float32, device=DEV)
    r = torch.empty(N, dtype=torch.float32, device=DEV)
    dn = torch.empty(N, dtype=torch.uint8, device=DEV)
    row_raw = lambda row: None if rr is None else rr[row].contiguous()
    ops.env_reset(kind, N, state, o, reset_raw=row_raw(0), seed=seed, it=it, row=0, lane0=lane0)
    for step in range(T):
        np.testing.assert_array_equal(o.cpu().numpy(), obs[:, step, :])
        ops.env_step(kind, N, state, torch.tensor(np.ascontiguousarray(act[:, step, :]), device=DEV), o, r, dn)
        np.testing.assert_array_equal(r.cpu().numpy(), rew[step])
        np.testing.assert_array_equal(dn.cpu().numpy(), (flags[step] & L.FLAG_DONE) > 0)
        ends = np.nonzero(flags[step] & L.FLAG_END)[0]
        if len(ends) and step + 1 < T:
            st2 = torch.empty((S, N), dtype=torch.float32, device=DEV)
            o2 = torch.empty((d.O, N), dtype=torch.float32, device=DEV)
            ops.env_reset(kind, N, st2, o2, reset_raw=row_raw(step + 1), seed=seed, it=it, row=step + 1, lane0=lane0)
            m = torch.tensor(ends, device=DEV)
            state[:, m] = st2[:, m]
            o[:, m] = o2[:, m]


# ---------------------------------------------------------------- the host mapping
def _point_algo(es, **kw):
    from rllab_b200.algos.ddpg import DDPG
    from rllab_b200.envs.normalized_env import normalize
    from rllab_b200.envs.point_env import PointEnv
    from rllab_b200.policies.deterministic_mlp_policy import DeterministicMLPPolicy
    from rllab_b200.q_functions.continuous_mlp_q_function import ContinuousMLPQFunction
    env = normalize(PointEnv())
    policy = DeterministicMLPPolicy(env_spec=env.spec, hidden_sizes=(32, 32))
    qf = ContinuousMLPQFunction(env_spec=env.spec)
    return DDPG(env=env, policy=policy, qf=qf, es=es(env.spec), **kw)


ALGO_ARGS = dict(n_updates_per_sample=3, max_path_length=41, min_pool_size=55, replay_pool_size=333,
                 include_horizon_terminal_transitions=True, discount=0.97, scale_reward=0.3, soft_target_tau=0.007,
                 qf_weight_decay=0.011, qf_learning_rate=2e-3, policy_weight_decay=0.021, policy_learning_rate=3e-4)


def test_hparams_pass_every_non_default_value():
    from rllab_b200.exploration_strategies.gaussian_strategy import GaussianStrategy
    from rllab_b200.exploration_strategies.ou_strategy import OUStrategy
    host = dict(ALGO_ARGS, include_horizon_terminal_transitions=1)
    hp = _point_algo(lambda spec: OUStrategy(spec, mu=0.25, theta=0.3, sigma=0.45), **ALGO_ARGS).hparams()
    for k, v in dict(host, es_kind=L.ES_OU, ou_mu=0.25, ou_theta=0.3, ou_sigma=0.45).items():
        assert getattr(hp, k) == v, (k, getattr(hp, k), v)
    hp = _point_algo(lambda spec: GaussianStrategy(spec, max_sigma=0.8, min_sigma=0.05, decay_period=1234),
                     **ALGO_ARGS).hparams()
    for k, v in dict(host, es_kind=L.ES_GAUSSIAN, gs_max_sigma=0.8, gs_min_sigma=0.05, gs_decay_period=1234).items():
        assert getattr(hp, k) == v, (k, getattr(hp, k), v)


def test_point_gaussian_train_tabular():
    """A short DDPG.train on normalize(PointEnv()) with GaussianStrategy: paths of at most 50 steps, horizon samples
    dropped, so epoch 0 stores at most 100 rows and evaluates nothing, and epochs 1 and 2 (at least 196 rows >= 150)
    log the whole tabular."""
    from rllab_b200.exploration_strategies.gaussian_strategy import GaussianStrategy
    from rllab_b200.misc import logger
    rows = []
    orig = logger.dump_tabular

    def capture(*a, **k):
        orig(*a, **k)
        rows.append(logger.get_last_table())

    logger.dump_tabular = capture
    try:
        algo = _point_algo(lambda spec: GaussianStrategy(spec, decay_period=150), n_epochs=3, epoch_length=100,
                           min_pool_size=150, max_path_length=50, eval_samples=200, seed=3)
        algo.train()
    finally:
        logger.dump_tabular = orig
    keys = {"Epoch", "AverageReturn", "StdReturn", "MaxReturn", "MinReturn", "AverageEsReturn", "StdEsReturn",
            "MaxEsReturn", "MinEsReturn", "AverageDiscountedReturn", "AverageQLoss", "AveragePolicySurr", "AverageQ",
            "AverageAbsQ", "AverageY", "AverageAbsY", "AverageAbsQYDiff", "AverageAction", "PolicyRegParamNorm",
            "QFunRegParamNorm"}
    assert len(rows) == 3 and not (keys & set(rows[0])), rows
    for epoch, row in zip((1, 2), rows[1:]):
        assert keys <= set(row), keys - set(row)
        assert row["Epoch"] == epoch and all(np.isfinite(row[k]) for k in keys), row
        assert row["AverageQLoss"] >= 0 and row["MaxReturn"] <= 0
    assert algo.runs.host_state()[0].itr == 300
