"""CPU: tests/ddpg_oracle.py against fixtures generated from the reference's own code (tests/golden/make_ddpg_golden.py):
SimpleReplayPool through the wrap and the full-pool rejection quirk, OUStrategy / GaussianStrategy, the control flow of
DDPG.train, the y and soft-update arithmetic of DDPG.do_training, and the constructor surfaces and layer order."""
import inspect
import json
import os

import numpy as np
import pytest

import ddpg_oracle as K

HERE = os.path.dirname(os.path.abspath(__file__))
G = dict(np.load(os.path.join(HERE, "golden", "reference_ddpg_golden.npz")))
API = json.load(open(os.path.join(HERE, "golden", "reference_api_ddpg.json")))


def _pool_state(rows, O, A):
    return dict(pool=dict(obs=np.zeros((rows, O), np.float32), act=np.zeros((rows, A), np.float32),
                          rew=np.zeros(rows, np.float32), term=np.zeros(rows, np.uint8)), top=0, bottom=0, size=0)


@pytest.mark.parametrize("tag,n_added", [("part", 10), ("full", 27)])
def test_pool_add_and_random_batch_match_reference(tag, n_added):
    rows = 20
    st = _pool_state(rows, 3, 1)
    for i in range(n_added):
        K.pool_add(st, rows, G["pool_obs_in"][i], G["pool_act_in"][i], G["pool_rew_in"][i], G["pool_term_in"][i])
    assert [st["top"], st["bottom"], st["size"]] == G["pool_%s_state" % tag].tolist()
    np.testing.assert_array_equal(st["pool"]["obs"], G["pool_%s_obs" % tag])
    np.testing.assert_array_equal(st["pool"]["term"], G["pool_%s_term" % tag])
    n_rejected = 0
    for s in range(12):
        # the reference's candidates: np.random.randint(bottom, bottom + size) under the same seed, as offsets
        np.random.seed(100 + s)
        cand = (np.random.randint(st["bottom"], st["bottom"] + st["size"]) - st["bottom"] for _ in iter(int, 1))
        rejected = []
        idx = K.accept_indices(cand, st["bottom"], st["size"], rows, batch=8, rejected=rejected)
        n_rejected += len(rejected)
        b = K.gather(st["pool"], idx, rows)
        key = "pool_%s_b%d_" % (tag, s)
        np.testing.assert_array_equal(b["s"], G[key + "observations"])
        np.testing.assert_array_equal(b["s2"], G[key + "next_observations"])
        np.testing.assert_array_equal(b["a"], G[key + "actions"])
        np.testing.assert_array_equal(b["r"], G[key + "rewards"])
        np.testing.assert_array_equal(b["term"], G[key + "terminals"])
    if tag == "full":
        # the quirk: the rejected index is size - 1 = 19, not the newest sample (row top - 1 = 6)
        assert n_rejected > 0 and st["top"] - 1 != st["size"] - 1


def test_exploration_strategies_match_reference():
    np.random.seed(3)
    x = np.full(2, 0.2)
    for t in range(10):
        if t == 5:
            x = np.full(2, 0.2)
        x = K.ou_step(x, 0.2, 0.15, 0.3, np.random.randn(2))
        np.testing.assert_allclose(x, G["ou_states"][t], rtol=0, atol=1e-15)
        np.testing.assert_allclose(np.clip(np.array([0.5, -0.9]) + x, -1, 1), G["ou_actions"][t], rtol=0, atol=1e-15)
    np.random.seed(4)
    for t in range(12):
        a = np.array([0.5, -0.9]) + np.random.normal(size=2) * K.gaussian_sigma(t, 1.0, 0.1, 8)
        np.testing.assert_allclose(np.clip(a, -1, 1), G["gs_actions"][t], rtol=0, atol=1e-15)


@pytest.mark.parametrize("htt", [0, 1])
def test_train_loop_control_flow_matches_reference(htt):
    """The oracle's train_step driven by the reference golden's scripted env: which samples enter the pool (obs, scaled
    reward, terminal), when training runs, and the Es path returns."""
    cfg = {k[len("loop_cfg_"):]: v.item() for k, v in G.items() if k.startswith("loop_cfg_")}
    lengths = G["loop_lengths"].tolist()
    d = K.Dims(3, 1)
    rows = cfg["replay_pool_size"]
    hp = dict(n_updates_per_sample=1, max_path_length=cfg["max_path_length"], min_pool_size=cfg["min_pool_size"],
              replay_pool_size=rows, include_horizon_terminal_transitions=htt, es_kind=0, discount=0.99,
              scale_reward=cfg["scale_reward"], soft_target_tau=0.001, qf_weight_decay=0.0, qf_learning_rate=1e-3,
              policy_weight_decay=0.0, policy_learning_rate=1e-4, ou_mu=0.0, ou_theta=0.15, ou_sigma=0.3,
              gs_max_sigma=1.0, gs_min_sigma=0.1, gs_decay_period=1e6)
    rng = np.random.RandomState(0)
    th = np.concatenate([K.init_params(d.pshapes, rng), K.init_params(d.qshapes, rng)])
    st = dict(_pool_state(rows, 3, 1), nets=np.stack([th, 0 * th, 0 * th, th]), env_state=None, obs=None,
              ou=np.zeros(1), path_return=0.0, path_length=0, terminal=2, itr=0, adam_t=0)
    env = dict(t=0, path=-1, k=0)
    resets = []

    def env_reset(itr):
        env["path"] += 1
        env["k"] = 0
        resets.append(itr)
        return None, np.array([env["t"], env["path"], 0.5], np.float32)

    def env_step(s, act):
        env["t"] += 1
        env["k"] += 1
        return None, np.array([env["t"], env["path"], 0.5], np.float32), 1.0 + 0.1 * env["t"], \
            env["k"] >= lengths[env["path"] % len(lengths)]

    stats = dict(es_returns=[], qf_loss=[], policy_surr=[], q=[], y=[])
    trained = []
    for _ in range(cfg["n_epochs"] * cfg["epoch_length"]):
        t0, itr = st["adam_t"], st["itr"]
        K.train_step(d, st, hp, 1, 0, env_reset, env_step, stats=stats)
        if st["adam_t"] > t0:
            trained.append(itr)
    key = "loop%d_" % htt
    assert trained == G[key + "trained"].tolist()
    # the reference's first reset precedes the loop (no es.reset); the golden records, for each es.reset, the itr of the
    # last get_action before it, i.e. the reset happens at the next itr
    assert resets[1:] == [i + 1 for i in G[key + "resets"].tolist()]
    np.testing.assert_allclose(stats["es_returns"], G[key + "es_returns"], rtol=1e-6)
    assert [st["top"], st["bottom"], st["size"]] == G[key + "pool_state"].tolist()
    np.testing.assert_array_equal(st["pool"]["obs"], G[key + "pool_obs"])
    np.testing.assert_allclose(st["pool"]["rew"], G[key + "pool_rew"], rtol=1e-6)
    np.testing.assert_array_equal(st["pool"]["term"], G[key + "pool_term"])


def test_do_training_y_and_soft_update_match_reference():
    o2, term, r = G["dt_b_next_observations"], G["dt_b_terminals"].astype(np.float64), G["dt_b_rewards"]
    q_next = o2 @ G["dt_wq"] + G["dt_cq"] * np.tanh(o2 @ G["dt_Wp"])[:, 0]
    np.testing.assert_allclose(K.targets_y(r, term, float(G["dt_discount"]), q_next), G["dt_ys"], rtol=0, atol=1e-14)
    tau = float(G["dt_tau"])
    np.testing.assert_allclose(K.soft_update(G["dt_tp0"], G["dt_p0"], tau), G["dt_tp1"], rtol=0, atol=1e-15)
    np.testing.assert_allclose(K.soft_update(G["dt_tq0"], G["dt_q0"], tau), G["dt_tq1"], rtol=0, atol=1e-15)


def _params(fn):
    return [n for n in inspect.signature(fn).parameters if n not in ("self", "kwargs")]


def test_constructor_surfaces_and_layer_order_match_reference():
    pytest.importorskip("torch")
    from rllab_b200.algos.ddpg import DDPG
    from rllab_b200.exploration_strategies.gaussian_strategy import GaussianStrategy
    from rllab_b200.exploration_strategies.ou_strategy import OUStrategy
    from rllab_b200.policies.deterministic_mlp_policy import DeterministicMLPPolicy
    from rllab_b200.q_functions.continuous_mlp_q_function import ContinuousMLPQFunction
    for cls in (DDPG, OUStrategy, GaussianStrategy, DeterministicMLPPolicy, ContinuousMLPQFunction):
        ref = [n for n, _ in API[cls.__name__]]
        assert _params(cls.__init__)[:len(ref)] == ref, cls.__name__
    # numeric defaults agree
    for cls in (DDPG, OUStrategy, GaussianStrategy):
        ours = inspect.signature(cls.__init__).parameters
        for n, dflt in API[cls.__name__]:
            if dflt is not None and dflt not in ("'adam'",):
                assert float(eval(dflt)) == float(ours[n].default), (cls.__name__, n)
    # both nets: dense layers h*, then output; the flat order is [W, b] per layer in that order
    assert API["DeterministicMLPPolicy_dense_layer_names"] == ["'h%d' % idx", "'output'"]
    assert API["ContinuousMLPQFunction_dense_layer_names"] == ["'h%d' % (idx + 1)", "'output'"]
    d = K.Dims(4, 1)
    assert d.pshapes == [(4, 32), (32,), (32, 32), (32,), (32, 1), (1,)]
    assert d.qshapes == [(4, 32), (32,), (33, 32), (32,), (32, 1), (1,)]
