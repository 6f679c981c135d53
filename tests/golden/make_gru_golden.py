"""Generate tests/golden/reference_gru_golden.npz and tests/golden/reference_api_gru.json from the reference's own code,
run through oracle/ref_shims.py on fixed inputs:
  * rllab/core/network.py GRULayer.step   the method body, taken out with `ast` and exec'd with a NumPy `self` (the
                                          module itself cannot be imported: its classes subclass the lasagne stand-ins);
                                          hidden sequences over fixed inputs (keys step_*)
  * rllab/distributions/recurrent_diagonal_gaussian.py  kl / log_likelihood / entropy on padded (paths, time, dim)
                                          arrays (keys dist_*)
  * rllab/sampler/base.py BaseSampler.process_samples, recurrent branch: fixed paths, a shim algo whose policy has
                                          recurrent = True and a zero baseline (keys ps_*: padding, valids, centred
                                          advantages, agent_infos incl. prev_action, Entropy)
  * the parameter order: GRULayer.__init__'s add_param calls in source order, their trainable flags, and the policy's
    constructor signature, recurrent / state_info_keys surface (reference_api_gru.json).

Run:  python tests/golden/make_gru_golden.py   (needs the reference tree; the tests only read the committed files)
"""
import ast
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import ref_shims  # noqa: E402

O, A, H = 4, 1, 32
I = O + A


def _class_node(path, name):
    tree = ast.parse(open(path).read())
    return next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == name)


def gru_step_fn(ref):
    cls = _class_node(os.path.join(ref, "rllab", "core", "network.py"), "GRULayer")
    fn = next(n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name == "step")
    import theano                                   # the shim: config.floatX = "float64" (the step's final cast)
    ns = {"np": np, "theano": theano}
    exec(compile(ast.Module(body=[fn], type_ignores=[]), "GRULayer.step", "exec"), ns)
    return ns["step"]


def gru_param_order(ref):
    """(name, trainable expression) of every add_param call in GRULayer.__init__, in source order."""
    cls = _class_node(os.path.join(ref, "rllab", "core", "network.py"), "GRULayer")
    init = next(n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name == "__init__")
    out = []
    for node in ast.walk(init):
        if isinstance(node, ast.Call) and getattr(node.func, "attr", "") == "add_param":
            kw = {k.arg: k.value for k in node.keywords}
            name = kw["name"].value
            trainable = ast.unparse(kw["trainable"]) if "trainable" in kw else "True"
            out.append((node.lineno, name, trainable))
    return [(n, t) for _, n, t in sorted(out)]


class _Self(object):
    def __init__(self, p):
        for k, v in p.items():
            setattr(self, k, v)
        self.gate_nonlinearity = lambda x: 1.0 / (1.0 + np.exp(-x))
        self.nonlinearity = np.tanh


def main():
    ref_shims.install()
    ref = ref_shims.REFERENCE_ROOT
    rng = np.random.RandomState(11)
    shapes = dict(W_xr=(I, H), W_hr=(H, H), b_r=(H,), W_xu=(I, H), W_hu=(H, H), b_u=(H,), W_xc=(I, H), W_hc=(H, H),
                  b_c=(H,))
    p = {k: rng.randn(*s) * (0.4 if len(s) == 2 else 0.2) for k, s in shapes.items()}
    step = gru_step_fn(ref)
    # a (T, n, I) input sequence from h0 = 0
    T, n = 9, 7
    xs = rng.randn(T, n, I)
    h = np.zeros((n, H))
    hs = []
    for t in range(T):
        h = step(_Self(p), xs[t], h)
        hs.append(h)
    out = {"step_" + k: v for k, v in p.items()}
    out.update(step_x=xs, step_h=np.stack(hs))

    # RecurrentDiagonalGaussian on padded arrays
    from rllab.distributions.recurrent_diagonal_gaussian import RecurrentDiagonalGaussian
    d = RecurrentDiagonalGaussian(2)
    m0, m1 = rng.randn(3, 5, 2), rng.randn(3, 5, 2)
    l0, l1 = rng.randn(3, 5, 2) * 0.3, rng.randn(3, 5, 2) * 0.3
    xa = rng.randn(3, 5, 2)
    out.update(dist_m0=m0, dist_m1=m1, dist_l0=l0, dist_l1=l1, dist_x=xa,
               dist_kl=d.kl(dict(mean=m0, log_std=l0), dict(mean=m1, log_std=l1)),
               dist_loglik=d.log_likelihood(xa, dict(mean=m1, log_std=l1)),
               dist_entropy=d.entropy(dict(mean=m1, log_std=l1)))

    # BaseSampler.process_samples, recurrent branch
    from rllab.sampler.base import BaseSampler
    from rllab.distributions.diagonal_gaussian import DiagonalGaussian
    import rllab.misc.logger as logger
    logger.record_tabular = lambda *a, **k: None
    logger.log = lambda *a, **k: None
    lens = [4, 1, 7, 3]
    paths = []
    ls = np.array([-0.4])
    for L in lens:
        act = rng.randn(L, A)
        paths.append(dict(observations=rng.randn(L, O), actions=act, rewards=rng.randn(L),
                          agent_infos=dict(mean=rng.randn(L, A), log_std=np.tile(ls, (L, 1)),
                                           prev_action=np.concatenate([np.zeros((1, A)), act[:-1]])),
                          env_infos=dict()))

    class _Baseline(object):
        def predict(self, path):
            return np.zeros(len(path["rewards"]))

        def fit(self, paths):
            pass

    class _Policy(object):
        recurrent = True
        distribution = DiagonalGaussian(A)

    class _Algo(object):
        baseline, policy = _Baseline(), _Policy()
        discount, gae_lambda, center_adv, positive_adv = 0.99, 1.0, True, False

    import copy
    sd = BaseSampler(_Algo()).process_samples(0, copy.deepcopy(paths))
    for i, path in enumerate(paths):
        for k in ("observations", "actions", "rewards"):
            out["ps_in%d_%s" % (i, k)] = path[k]
        for k in ("mean", "log_std", "prev_action"):
            out["ps_in%d_%s" % (i, k)] = path["agent_infos"][k]
    out["ps_n_paths"] = len(paths)
    for k in ("observations", "actions", "rewards", "returns", "advantages", "valids"):
        out["ps_" + k] = sd[k]
    for k, v in sd["agent_infos"].items():
        out["ps_agent_" + k] = v
    out["ps_raw_advantages"] = np.concatenate([p_["advantages"] for p_ in sd["paths"]])
    ent = np.sum(_Algo.policy.distribution.entropy(sd["agent_infos"]) * sd["valids"]) / np.sum(sd["valids"])
    out["ps_entropy"] = ent
    np.savez(os.path.join(HERE, "reference_gru_golden.npz"), **out)

    # API surface
    pol = _class_node(os.path.join(ref, "rllab", "policies", "gaussian_gru_policy.py"), "GaussianGRUPolicy")
    init = next(n for n in pol.body if isinstance(n, ast.FunctionDef) and n.name == "__init__")
    args = [a.arg for a in init.args.args][1:]
    defaults = [ast.unparse(v) for v in init.args.defaults]
    methods = sorted(n.name for n in pol.body if isinstance(n, ast.FunctionDef) and not n.name.startswith("_"))
    net = _class_node(os.path.join(ref, "rllab", "core", "network.py"), "GRUNetwork")
    h0_trainable = [ast.unparse(k.value) for node in ast.walk(net) if isinstance(node, ast.Call)
                    for k in node.keywords if k.arg == "hidden_init_trainable"]
    api = dict(ctor_args=args, gru_network_hidden_init_trainable=h0_trainable, ctor_defaults=dict(zip(args[len(args) - len(defaults):], defaults)),
               methods=methods, gru_layer_params=gru_param_order(ref),
               mean_network_output="DenseLayer(W, b) on the GRU layer's output (network.py GRUNetwork)",
               policy_params="LasagnePowered([l_mean, l_log_std]): GRU params, then output W, b, then log_std")
    with open(os.path.join(HERE, "reference_api_gru.json"), "w") as f:
        json.dump(api, f, indent=1)


if __name__ == "__main__":
    main()
