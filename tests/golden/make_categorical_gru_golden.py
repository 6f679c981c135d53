"""Generate tests/golden/reference_categorical_gru_golden.npz and tests/golden/reference_api_categorical_gru.json from
the reference's own code, run through oracle/ref_shims.py on fixed inputs:
  * rllab/distributions/recurrent_categorical.py  kl / log_likelihood / entropy on padded (paths, time, n) arrays
                                          (keys dist_*)
  * rllab/policies/categorical_gru_policy.py CategoricalGRUPolicy.get_action  the method body, taken out with `ast` and
                                          exec'd with a NumPy `self` whose f_step_prob records its input: the input
                                          obs + one-hot prev action it composes and the prev_action agent_info, over a
                                          fixed action sequence with reset() (keys act_*)
  * rllab/sampler/base.py BaseSampler.process_samples, recurrent branch with RecurrentCategorical: fixed paths with
                                          prob / prev_action agent_infos (keys ps_*: padding, valids, centred
                                          advantages, agent_infos, Entropy)
  * the parameter order (GRULayer.__init__'s add_param calls, then the softmax output layer's W and b) and the
    constructor signature (reference_api_categorical_gru.json).
The GRU cell itself is pinned by make_gru_golden.py (the same GRULayer.step).

Run:  python tests/golden/make_categorical_gru_golden.py   (needs the reference tree; the tests only read the
committed files)
"""
import ast
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from oracle import ref_shims  # noqa: E402

O, N_ACT, H = 4, 2, 32


def _method(path, cls_name, name, ns):
    import make_gru_golden as MG
    cls = MG._class_node(path, cls_name)
    fn = next(n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name == name)
    fn.decorator_list = []
    exec(compile(ast.Module(body=[fn], type_ignores=[]), "%s.%s" % (cls_name, name), "exec"), ns)
    return ns[name]


def main():
    ref_shims.install()
    import make_gru_golden as MG
    ref = ref_shims.REFERENCE_ROOT
    rng = np.random.RandomState(13)
    out = {}

    # RecurrentCategorical on padded arrays
    from rllab.distributions.recurrent_categorical import RecurrentCategorical
    d = RecurrentCategorical(N_ACT)
    p0 = rng.dirichlet(np.ones(N_ACT), size=(3, 5))
    p1 = rng.dirichlet(np.ones(N_ACT), size=(3, 5))
    p1[0, 0] = [1.0 - 1e-9, 1e-9]
    x = np.eye(N_ACT)[rng.randint(0, N_ACT, size=(3, 5))]
    out.update(dist_p0=p0, dist_p1=p1, dist_x=x, dist_kl=d.kl(dict(prob=p0), dict(prob=p1)),
               dist_entropy=d.entropy(dict(prob=p1)))
    try:
        out["dist_loglik"] = np.asarray(d.log_likelihood(x, dict(prob=p1)), dtype=np.float64)
    except Exception as e:                        # log_likelihood goes through the flat *_sym graph builder
        print("RecurrentCategorical.log_likelihood not evaluable through the shims:", repr(e))

    # CategoricalGRUPolicy.get_action: the composed input and the prev_action agent_info
    from rllab.spaces import Box, Discrete
    path = os.path.join(ref, "rllab", "policies", "categorical_gru_policy.py")
    import rllab.misc.special as special
    get_action = _method(path, "CategoricalGRUPolicy", "get_action", {"np": np, "special": special})
    reset = _method(path, "CategoricalGRUPolicy", "reset", {"np": np})

    class _Net(object):
        class hid_init_param(object):
            @staticmethod
            def get_value():
                return np.zeros(H)

    class _Self(object):
        def __init__(self, inc):
            self.state_include_action = inc
            self.action_space = Discrete(N_ACT)
            self.observation_space = Box(-np.inf, np.inf, (O,))
            self.prob_network = _Net()
            self.inputs = []

        def f_step_prob(self, inp, hid):
            self.inputs.append(np.asarray(inp[0], dtype=np.float64))
            return [np.array([[0.3, 0.7]]), np.asarray(hid, dtype=np.float64).reshape(1, -1) + 1.0]

    obs = rng.randn(6, O)
    starts = [0, 3]
    for inc in (True, False):
        s = _Self(inc)
        infos, acts = [], []
        np.random.seed(5)
        for t in range(len(obs)):
            if t in starts:
                reset(s)
            a, info = get_action(s, obs[t])
            acts.append(a)
            infos.append(info)
        key = "act_inc%d_" % int(inc)
        out[key + "obs"] = obs
        out[key + "starts"] = np.array(starts)
        out[key + "actions"] = np.array(acts)
        out[key + "inputs"] = np.stack(s.inputs)
        if inc:
            out[key + "prev_action"] = np.stack([i["prev_action"] for i in infos])

    # BaseSampler.process_samples, recurrent branch, categorical agent_infos
    from rllab.sampler.base import BaseSampler
    import rllab.misc.logger as logger
    logger.record_tabular = lambda *a, **k: None
    logger.log = lambda *a, **k: None
    lens = [4, 1, 7, 3]
    paths = []
    for L in lens:
        act = np.eye(N_ACT)[rng.randint(0, N_ACT, L)]
        paths.append(dict(observations=rng.randn(L, O), actions=act, rewards=rng.randn(L),
                          agent_infos=dict(prob=rng.dirichlet(np.ones(N_ACT), size=L),
                                           prev_action=np.concatenate([np.zeros((1, N_ACT)), act[:-1]])),
                          env_infos=dict()))

    class _Baseline(object):
        def predict(self, path):
            return np.zeros(len(path["rewards"]))

        def fit(self, paths):
            pass

    class _Policy(object):
        recurrent = True
        distribution = RecurrentCategorical(N_ACT)

    class _Algo(object):
        baseline, policy = _Baseline(), _Policy()
        discount, gae_lambda, center_adv, positive_adv = 0.99, 1.0, True, False

    import copy
    sd = BaseSampler(_Algo()).process_samples(0, copy.deepcopy(paths))
    for i, p in enumerate(paths):
        for k in ("observations", "actions", "rewards"):
            out["ps_in%d_%s" % (i, k)] = p[k]
        for k in ("prob", "prev_action"):
            out["ps_in%d_%s" % (i, k)] = p["agent_infos"][k]
    out["ps_n_paths"] = len(paths)
    for k in ("observations", "actions", "rewards", "returns", "advantages", "valids"):
        out["ps_" + k] = sd[k]
    for k, v in sd["agent_infos"].items():
        out["ps_agent_" + k] = v
    # the Entropy statistic of the recurrent branch (base.py): mean of entropy over the valid samples
    out["ps_entropy"] = np.sum(_Algo.policy.distribution.entropy(sd["agent_infos"]) * sd["valids"]) / np.sum(sd["valids"])
    np.savez(os.path.join(HERE, "reference_categorical_gru_golden.npz"), **out)

    # API surface
    pol = MG._class_node(path, "CategoricalGRUPolicy")
    init = next(n for n in pol.body if isinstance(n, ast.FunctionDef) and n.name == "__init__")
    args = [a.arg for a in init.args.args][1:]
    defaults = [ast.unparse(v) for v in init.args.defaults]
    src = open(path).read()
    api = dict(ctor_args=args, ctor_defaults=dict(zip(args[len(args) - len(defaults):], defaults)),
               gru_layer_params=MG.gru_param_order(ref),
               output_nonlinearity_softmax="output_nonlinearity=TT.nnet.softmax" in src,
               output_layer="GRUNetwork's output DenseLayer: W (hidden, n), b (n)",
               state_info_keys=["prev_action"], dist_info_keys=["prob"])
    with open(os.path.join(HERE, "reference_api_categorical_gru.json"), "w") as f:
        json.dump(api, f, indent=1)


if __name__ == "__main__":
    main()
