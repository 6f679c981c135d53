"""CPU: CategoricalGRUPolicy's host surface and oracle against fixtures generated from the reference's own code
(tests/golden/make_categorical_gru_golden.py): RecurrentCategorical on padded arrays, the input get_action composes
(obs + one-hot previous action, zero at a path start) and its prev_action agent_info, the recurrent samples_data layout
with prob agent_infos and its Entropy statistic, and the parameter order and constructor surface."""
import json
import os

import numpy as np
import pytest

import categorical_gru_oracle as C
import categorical_oracle as CO
import gru_oracle as G

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = np.load(os.path.join(HERE, "golden", "reference_categorical_gru_golden.npz"))
API = json.load(open(os.path.join(HERE, "golden", "reference_api_categorical_gru.json")))


def test_distribution_matches_reference():
    from rllab_b200.distributions.recurrent_categorical import RecurrentCategorical
    d = RecurrentCategorical(2)
    p0, p1 = dict(prob=GOLD["dist_p0"]), dict(prob=GOLD["dist_p1"])
    np.testing.assert_allclose(d.kl(p0, p1), GOLD["dist_kl"], rtol=1e-13, atol=1e-15)
    np.testing.assert_allclose(d.entropy(p1), GOLD["dist_entropy"], rtol=1e-13, atol=1e-15)
    assert d.dist_info_keys == API["dist_info_keys"]
    if "dist_loglik" in GOLD.files:
        np.testing.assert_allclose(d.log_likelihood(GOLD["dist_x"], p1), GOLD["dist_loglik"], rtol=1e-13)
    else:   # the reference's numeric log_likelihood calls its graph builder; ours is log(p[x] + TINY) per cell
        x, p = GOLD["dist_x"], GOLD["dist_p1"]
        np.testing.assert_allclose(d.log_likelihood(x, p1), np.log(np.sum(p * x, axis=-1) + 1e-8), rtol=1e-13)


def _lanes_from_actions(key):
    """One lane holding the fixture's observations and actions, paths starting at the fixture's reset steps."""
    obs, acts, starts = GOLD[key + "obs"], GOLD[key + "actions"], list(GOLD[key + "starts"])
    T = len(obs)
    tstep = np.zeros((T, 1), np.uint16)
    for t in range(1, T):
        tstep[t] = 0 if t in starts else tstep[t - 1] + 1
    return dict(obs=obs.T[:, :, None].astype(np.float32), act=np.eye(2)[acts].T[:, :, None], tstep=tstep)


@pytest.mark.parametrize("inc", [True, False])
def test_input_and_prev_action_match_reference_get_action(inc):
    """The oracle's (and so the kernels') x_t is the input the reference's get_action feeds its step function."""
    key = "act_inc%d_" % int(inc)
    lanes = _lanes_from_actions(key)
    dims = C.CatGruDims(4, 32, 2, inc)
    xs = np.stack([G.inputs(lanes, dims, t)[0][0] for t in range(len(GOLD[key + "obs"]))])
    np.testing.assert_allclose(xs, GOLD[key + "inputs"], rtol=0, atol=1e-6)
    if inc:
        # the wire format's prev_action rule (lanes_to_paths): zeros at a path start, then the previous one-hot action
        acts = np.eye(2)[GOLD[key + "actions"]]
        starts = list(GOLD[key + "starts"])
        pa = np.array([np.zeros(2) if t in starts else acts[t - 1] for t in range(len(acts))])
        np.testing.assert_array_equal(pa, GOLD[key + "prev_action"])


@pytest.mark.parametrize("inc", [True, False])
def test_policy_step_matches_reference_get_action(inc, monkeypatch):
    """CategoricalGRUPolicy.get_action with its device step replaced by the fixture's stand-in (prob (0.3, 0.7), hidden
    + 1): the same inputs, the same host draws from np.random, the same prev_action agent_infos."""
    from rllab_b200 import _lib as L
    if not os.path.exists(L.LIB_PATH):
        pytest.skip("library not built")
    from rllab_b200.envs.gym_env import GymEnv
    from rllab_b200.envs.normalized_env import normalize
    from rllab_b200.policies.categorical_gru_policy import CategoricalGRUPolicy
    key = "act_inc%d_" % int(inc)
    pol = CategoricalGRUPolicy(normalize(GymEnv("CartPole-v0")).spec, state_include_action=inc)
    seen = []

    def step(flat_obs, prev, hid):
        seen.append(np.concatenate([flat_obs[0], prev[0]]) if inc else flat_obs[0].copy())
        return np.array([[0.3, 0.7]]), np.asarray(hid) + 1.0
    monkeypatch.setattr(pol, "_step", step)
    np.random.seed(5)
    acts, pas = [], []
    for t, o in enumerate(GOLD[key + "obs"]):
        if t in list(GOLD[key + "starts"]):
            pol.reset()
        a, info = pol.get_action(o)
        acts.append(a)
        pas.append(info.get("prev_action"))
    np.testing.assert_array_equal(acts, GOLD[key + "actions"])
    np.testing.assert_allclose(np.stack(seen), GOLD[key + "inputs"], rtol=0, atol=0)
    if inc:
        np.testing.assert_array_equal(np.stack(pas), GOLD[key + "prev_action"])


def _golden_paths():
    n = int(GOLD["ps_n_paths"])
    valids = GOLD["ps_valids"]
    paths = []
    for i in range(n):
        L = int(valids[i].sum())
        paths.append(dict(observations=GOLD["ps_in%d_observations" % i], actions=GOLD["ps_in%d_actions" % i],
                          rewards=GOLD["ps_in%d_rewards" % i], returns=GOLD["ps_returns"][i, :L],
                          advantages=GOLD["ps_advantages"][i, :L], env_infos=dict(),
                          agent_infos={a: GOLD["ps_in%d_%s" % (i, a)] for a in ("prob", "prev_action")}))
    return paths


def test_recurrent_samples_data_matches_reference_layout():
    from rllab_b200.sampler.lane_sampler import recurrent_samples_entry
    paths = _golden_paths()
    for key in ("observations", "actions", "rewards", "returns", "advantages", "valids"):
        v = recurrent_samples_entry(paths, key)
        assert v.shape == GOLD["ps_" + key].shape, key
        np.testing.assert_allclose(v, GOLD["ps_" + key], rtol=1e-12, atol=1e-12, err_msg=key)
    ai = recurrent_samples_entry(paths, "agent_infos")
    assert sorted(ai) == sorted(k[9:] for k in GOLD.files if k.startswith("ps_agent_")) == ["prev_action", "prob"]
    for k, v in ai.items():
        np.testing.assert_array_equal(v, GOLD["ps_agent_" + k])


def test_entropy_statistic_matches_reference():
    """The sampler's categorical Entropy (sum of entropy(prob) over the valid samples / their number, as
    b200rl_categorical_entropy reduces it) and the oracle's are the reference's recurrent-branch Entropy."""
    from rllab_b200.sampler.lane_sampler import LaneSampler
    v = GOLD["ps_valids"] == 1
    prob = GOLD["ps_agent_prob"]

    class _P(object):
        def __init__(self, x):
            self.x = x

        def get(self):
            return self.x
    s = np.zeros(16)
    s[2], s[3] = 1.0, 1.0
    e = np.array([CO.entropy(prob[v]).sum(), v.sum()])
    st = LaneSampler._resolve_stats(0, _P(s), _P(np.zeros(4)), _P(e), True)
    np.testing.assert_allclose(st["Entropy"], GOLD["ps_entropy"], rtol=1e-12)
    lanes = dict(mean=np.moveaxis(prob, -1, 0), valid=v, tstep=np.zeros(v.shape))
    np.testing.assert_allclose(C.entropy_mean(lanes), GOLD["ps_entropy"], rtol=1e-12)


def test_parameter_order_and_surface_match_reference():
    """GRULayer's add_param order (h0 untrainable: hidden_init_trainable is False in GRUNetwork) then the softmax output
    layer's W and b is the flat layout of the policy and the oracle; the constructor takes the reference's arguments."""
    import inspect
    from rllab_b200.policies.categorical_gru_policy import CategoricalGRUPolicy
    names = [n for n, _ in API["gru_layer_params"]]
    assert names[0] == "h0" and API["gru_layer_params"][0][1] == "hidden_init_trainable"
    dims = C.CatGruDims(4, 32, 2, True)
    assert dims.names == names[1:] + ["W_out", "b_out"]
    assert API["output_nonlinearity_softmax"]
    sig = inspect.signature(CategoricalGRUPolicy.__init__)
    params = list(sig.parameters)[1:]
    assert params[:len(API["ctor_args"])] == API["ctor_args"]
    for k, v in API["ctor_defaults"].items():
        d = sig.parameters[k].default
        assert (v == "NL.tanh" and d is None) or repr(d) == v, (k, v, d)
    assert API["state_info_keys"] == ["prev_action"]
