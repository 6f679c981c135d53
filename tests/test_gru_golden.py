"""CPU: the GRU oracle, the host policy and the recurrent wire format against outputs of the reference's own code
(tests/golden/make_gru_golden.py -> reference_gru_golden.npz, reference_api_gru.json): GRULayer.step, the
RecurrentDiagonalGaussian functions, BaseSampler.process_samples' recurrent branch (padding, valids, centred
advantages, agent_infos with prev_action, Entropy), and the parameter order and constructor surface."""
import json
import os

import numpy as np
import pytest

import gru_oracle as G

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
GOLD = np.load(os.path.join(HERE, "reference_gru_golden.npz"))
API = json.load(open(os.path.join(HERE, "reference_api_gru.json")))


def test_cell_matches_reference_step():
    p = {k[5:]: GOLD[k] for k in GOLD.files if k.startswith("step_") and k not in ("step_x", "step_h")}
    xs, hs = GOLD["step_x"], GOLD["step_h"]
    h = np.zeros_like(hs[0])
    for t in range(len(xs)):
        h, _, _, _, _ = G.cell(p, xs[t], h)
        np.testing.assert_allclose(h, hs[t], rtol=1e-13, atol=1e-14)


def test_distribution_matches_reference():
    from rllab_b200.distributions.recurrent_diagonal_gaussian import RecurrentDiagonalGaussian
    d = RecurrentDiagonalGaussian(2)
    old = dict(mean=GOLD["dist_m0"], log_std=GOLD["dist_l0"])
    new = dict(mean=GOLD["dist_m1"], log_std=GOLD["dist_l1"])
    np.testing.assert_allclose(d.kl(old, new), GOLD["dist_kl"], rtol=1e-13)
    np.testing.assert_allclose(d.log_likelihood(GOLD["dist_x"], new), GOLD["dist_loglik"], rtol=1e-13)
    np.testing.assert_allclose(d.entropy(new), GOLD["dist_entropy"], rtol=1e-13)


def _golden_paths():
    """The golden's input paths with the device's centring of the advantages (process_samples + center_advantages:
    mean and population std + 1e-8 over the valid samples) and the returns the reference computed."""
    n = int(GOLD["ps_n_paths"])
    valids = GOLD["ps_valids"]
    raw = GOLD["ps_raw_advantages"]
    adv = (raw - raw.mean()) / (raw.std() + 1e-8)
    paths, k = [], 0
    for i in range(n):
        L = int(valids[i].sum())
        paths.append(dict(observations=GOLD["ps_in%d_observations" % i], actions=GOLD["ps_in%d_actions" % i],
                          rewards=GOLD["ps_in%d_rewards" % i], returns=GOLD["ps_returns"][i, :L],
                          advantages=adv[k:k + L], env_infos=dict(),
                          agent_infos={a: GOLD["ps_in%d_%s" % (i, a)] for a in ("mean", "log_std", "prev_action")}))
        k += L
    return paths


def test_recurrent_samples_data_matches_reference_layout():
    from rllab_b200.sampler.lane_sampler import recurrent_samples_entry
    paths = _golden_paths()
    for key in ("observations", "actions", "rewards", "returns", "advantages", "valids"):
        v = recurrent_samples_entry(paths, key)
        assert v.shape == GOLD["ps_" + key].shape, key
        np.testing.assert_allclose(v, GOLD["ps_" + key], rtol=1e-12, atol=1e-12, err_msg=key)
    ai = recurrent_samples_entry(paths, "agent_infos")
    assert sorted(ai) == sorted(k[9:] for k in GOLD.files if k.startswith("ps_agent_"))
    for k, v in ai.items():
        np.testing.assert_array_equal(v, GOLD["ps_agent_" + k])
    assert recurrent_samples_entry(paths, "env_infos") == dict()


def test_entropy_statistic_matches_reference():
    """The sampler's Entropy for a Gaussian policy, sum(log_std + log sqrt(2 pi e)), is the reference's valid-weighted
    mean of the per-sample entropy (the entropy does not depend on the state)."""
    from rllab_b200.sampler.lane_sampler import LaneSampler

    class _P(object):
        def __init__(self, v):
            self.v = v

        def get(self):
            return self.v
    s = np.zeros(16)
    s[2], s[3] = 1.0, 1.0
    ls = GOLD["ps_in0_log_std"][0].astype(np.float32)
    st = LaneSampler._resolve_stats(0, _P(s), _P(np.zeros(4)), _P(ls), False)
    np.testing.assert_allclose(st["Entropy"], GOLD["ps_entropy"], rtol=1e-6)


def test_parameter_order_and_surface_match_reference():
    """GRULayer's add_param order with h0 left out (GRUNetwork builds it with hidden_init_trainable=False), then the
    output DenseLayer's W, b and the log_std ParamLayer: the oracle's and the policy's flat layout."""
    params = API["gru_layer_params"]
    assert params[0] == ["h0", "hidden_init_trainable"] and API["gru_network_hidden_init_trainable"] == ["False"]
    gru = [n for n, t in params if t == "True"]
    assert gru + ["W_out", "b_out", "log_std"] == G.GruDims(4, 32, 1).names
    assert API["ctor_args"] == ["env_spec", "hidden_sizes", "state_include_action", "hidden_nonlinearity", "learn_std",
                                "init_std", "output_nonlinearity"]
    import inspect
    from rllab_b200.policies.gaussian_gru_policy import GaussianGRUPolicy
    sig = inspect.signature(GaussianGRUPolicy.__init__)
    assert list(sig.parameters)[1:len(API["ctor_args"]) + 1] == API["ctor_args"]
    for k, v in API["ctor_defaults"].items():
        if k == "hidden_nonlinearity":
            continue                                   # NL.tanh; None means the same tanh here
        assert repr(sig.parameters[k].default) == v, k
    for m in API["methods"]:
        if m == "dist_info_sym":
            continue                                   # the Theano graph builder: its compiled functions are kernels
        assert hasattr(GaussianGRUPolicy, m), m


def test_policy_rejects_a_row_count_it_holds_no_state_for():
    from rllab_b200 import _lib
    try:
        _lib.load()
    except _lib.B200RLError:
        pytest.skip("libb200rl.so not built")
    from rllab_b200.envs.box2d.cartpole_env import CartpoleEnv
    from rllab_b200.envs.normalized_env import normalize
    from rllab_b200.policies.gaussian_gru_policy import GaussianGRUPolicy
    pol = GaussianGRUPolicy(env_spec=normalize(CartpoleEnv()).spec)
    with pytest.raises(ValueError):
        pol.get_actions(np.zeros((3, 4)))
