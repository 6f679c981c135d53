"""Generate tests/golden/reference_ddpg_golden.npz and tests/golden/reference_api_ddpg.json from the reference's own code,
run through oracle/ref_shims.py on fixed inputs:
  * rllab/algos/ddpg.py SimpleReplayPool   add_sample through the wrap, random_batch under a seeded np.random before and
                                           after the pool is full (keys pool_*)
  * rllab/exploration_strategies/ou_strategy.py, gaussian_strategy.py  get_action with a stub policy under a seeded
                                           np.random, with a reset mid-way (keys ou_*, gs_*)
  * DDPG.train                             the method body, taken out with `ast` and exec'd with a stub env (scripted
                                           path lengths), a stub es / policy and a recording do_training / evaluate:
                                           which samples enter the pool, when training runs, es_path_returns
                                           (keys loop<h>_*, h = include_horizon_terminal_transitions)
  * DDPG.do_training                       the method body with NumPy stand-ins for the nets: y and the soft update
                                           (keys dt_*)
  * the constructor signatures and the layer order of the two nets (reference_api_ddpg.json).

Run:  python tests/golden/make_ddpg_golden.py   (needs the reference tree; the tests only read the committed files)
"""
import ast
import inspect
import json
import os
import pickle
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from oracle import ref_shims  # noqa: E402

# scripted env of the loop golden: path k lasts LENGTHS[k % len] steps unless max_path_length cuts it first
LENGTHS = [3, 9, 5, 12, 2, 7, 4, 10]
LOOP = dict(n_epochs=3, epoch_length=50, min_pool_size=40, max_path_length=7, scale_reward=0.5, replay_pool_size=60)


def _method(path, cls_name, name, ns):
    import make_gru_golden as MG
    cls = MG._class_node(path, cls_name)
    fn = next(n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name == name)
    fn.decorator_list = []
    exec(compile(ast.Module(body=[fn], type_ignores=[]), "%s.%s" % (cls_name, name), "exec"), ns)
    return ns[name]


class StubPolicy(object):
    def reset(self):
        pass

    def get_param_values(self):
        return np.zeros(1)

    def set_param_values(self, v):
        pass

    def terminate(self):
        pass


class ScriptedEnv(object):
    """obs = [global step, path index, 0.5]; reward = 1 + 0.1 * global step; done after LENGTHS[path] steps."""

    def __init__(self):
        self.t, self.path, self.k = 0, -1, 0

    def reset(self):
        self.path += 1
        self.k = 0
        return np.array([self.t, self.path, 0.5])

    def step(self, action):
        self.t += 1
        self.k += 1
        r = 1.0 + 0.1 * self.t
        return np.array([self.t, self.path, 0.5]), r, self.k >= LENGTHS[self.path % len(LENGTHS)], {}

    def terminate(self):
        pass


def main():
    ref_shims.install()
    ref = ref_shims.REFERENCE_ROOT
    from rllab.algos.ddpg import DDPG, SimpleReplayPool
    from rllab.exploration_strategies.gaussian_strategy import GaussianStrategy
    from rllab.exploration_strategies.ou_strategy import OUStrategy
    from rllab.misc import ext
    from rllab.misc.ext import AttrDict
    from rllab.spaces import Box
    out = dict(loop_lengths=np.array(LENGTHS), **{"loop_cfg_" + k: np.array(v) for k, v in LOOP.items()})
    rng = np.random.RandomState(13)

    # SimpleReplayPool
    rows, O, A = 20, 3, 1
    pool = SimpleReplayPool(rows, O, A)
    obs = rng.randn(27, O).astype(np.float32).astype(np.float64)
    act = rng.uniform(-1, 1, (27, A)).astype(np.float32).astype(np.float64)
    rew = rng.randn(27).astype(np.float32).astype(np.float64)
    term = (rng.rand(27) < 0.3).astype(np.uint8)
    out.update(pool_obs_in=obs, pool_act_in=act, pool_rew_in=rew, pool_term_in=term)
    for lo, hi, tag in ((0, 10, "part"), (10, 27, "full")):
        for i in range(lo, hi):
            pool.add_sample(obs[i], act[i], rew[i], term[i])
        out["pool_%s_state" % tag] = np.array([pool._top, pool._bottom, pool._size])
        out["pool_%s_obs" % tag] = pool._observations.copy()
        out["pool_%s_term" % tag] = pool._terminals.copy()
        for s in range(12):
            np.random.seed(100 + s)
            b = pool.random_batch(8)
            for k in ("observations", "actions", "rewards", "terminals", "next_observations"):
                out["pool_%s_b%d_%s" % (tag, s, k)] = b[k]

    # exploration strategies with a stub policy
    class Pol(object):
        def get_action(self, o):
            return np.array([0.5, -0.9]), {}

    spec = AttrDict(action_space=Box(-1.0, 1.0, (2,)))
    ou = OUStrategy(spec, mu=0.2, theta=0.15, sigma=0.3)
    np.random.seed(3)
    acts, states = [], []
    for t in range(10):
        if t == 5:
            ou.reset()
        acts.append(ou.get_action(t, None, Pol()))
        states.append(ou.state.copy())
    out.update(ou_actions=np.array(acts), ou_states=np.array(states))
    gs = GaussianStrategy(spec, max_sigma=1.0, min_sigma=0.1, decay_period=8)
    np.random.seed(4)
    out["gs_actions"] = np.array([gs.get_action(t, None, Pol()) for t in range(12)])

    # DDPG.train control flow
    path = os.path.join(ref, "rllab", "algos", "ddpg.py")

    class Log(object):
        def __getattr__(self, name):
            return lambda *a, **k: None

    class Prog(object):
        @staticmethod
        def prog_bar(x):
            return x

    for htt in (0, 1):
        ns = {"np": np, "pickle": pickle, "logger": Log(), "pyprind": Prog(), "SimpleReplayPool": SimpleReplayPool}
        train = _method(path, "DDPG", "train", ns)
        trained, evals, resets = [], [], []

        class Es(object):
            def reset(self):
                resets.append(self_.itr_now)

            def get_action(self, itr, o, policy):
                self_.itr_now = itr
                return np.array([0.25])

        class Self(object):
            pass
        self_ = Self()
        self_.itr_now = 0
        env = ScriptedEnv()
        env.observation_space = AttrDict(flat_dim=O)
        env.action_space = AttrDict(flat_dim=A)
        self_.env, self_.es, self_.policy, self_.plot = env, Es(), StubPolicy(), False
        for k, v in LOOP.items():
            setattr(self_, k, v)
        self_.include_horizon_terminal_transitions = bool(htt)
        self_.n_updates_per_sample, self_.batch_size = 1, 32
        self_.es_path_returns = []
        self_.start_worker = lambda: None
        self_.init_opt = lambda: None
        self_.get_epoch_snapshot = lambda epoch: None
        pools = []

        def do_training(itr, batch):
            trained.append(itr)

        def evaluate(epoch, pool):
            evals.append(list(self_.es_path_returns))
            self_.es_path_returns = []
            pools.append(pool)
        self_.do_training, self_.evaluate = do_training, evaluate
        np.random.seed(5)
        train(self_)
        p = pools[-1]
        key = "loop%d_" % htt
        out[key + "trained"] = np.array(trained)
        out[key + "resets"] = np.array(resets)
        out[key + "es_returns"] = np.array(sum(evals, []) + list(self_.es_path_returns))
        out[key + "n_eval_returns"] = np.array([len(e) for e in evals])
        out[key + "pool_obs"] = p._observations.copy()
        out[key + "pool_rew"] = p._rewards.copy()
        out[key + "pool_term"] = p._terminals.copy()
        out[key + "pool_state"] = np.array([p._top, p._bottom, p._size])

    # DDPG.do_training with NumPy stand-ins for the nets
    do_training = _method(path, "DDPG", "do_training", {"ext": ext, "np": np})
    Wp = rng.randn(O, A)
    wq, cq = rng.randn(O), 0.7

    class Flat(object):
        def __init__(self, v):
            self.v = v

        def get_param_values(self):
            return self.v.copy()

        def set_param_values(self, v):
            self.v = np.asarray(v).copy()

    class TPol(Flat):
        def get_actions(self, o):
            return np.tanh(o @ Wp), {}

    class TQf(Flat):
        def get_qval(self, o, a):
            return o @ wq + cq * a[:, 0]

    rec = {}

    def f_train_qf(ys, o, a):
        rec["ys"] = ys
        return 0.0, np.zeros(len(ys))
    S = type("S", (), {})()
    S.discount, S.soft_target_tau = 0.97, 0.3
    tp0, tq0, p0, q0 = rng.randn(5), rng.randn(6), rng.randn(5), rng.randn(6)
    S.opt_info = dict(target_policy=TPol(tp0), target_qf=TQf(tq0), f_train_qf=f_train_qf, f_train_policy=lambda o: 0.0)
    S.policy, S.qf = Flat(p0), Flat(q0)
    S.qf_loss_averages, S.policy_surr_averages, S.q_averages, S.y_averages = [], [], [], []
    batch = dict(observations=rng.randn(8, O), actions=rng.randn(8, A), rewards=rng.randn(8),
                 next_observations=rng.randn(8, O), terminals=(rng.rand(8) < 0.5).astype(np.uint8))
    do_training(S, 0, batch)
    out.update(dt_Wp=Wp, dt_wq=wq, dt_cq=np.array(cq), dt_discount=np.array(S.discount),
               dt_tau=np.array(S.soft_target_tau), dt_tp0=tp0, dt_tq0=tq0, dt_p0=p0, dt_q0=q0,
               dt_ys=rec["ys"], dt_tp1=S.opt_info["target_policy"].v, dt_tq1=S.opt_info["target_qf"].v,
               **{"dt_b_" + k: v for k, v in batch.items()})
    np.savez(os.path.join(HERE, "reference_ddpg_golden.npz"), **out)

    # constructor surfaces and layer order
    def sig(fn):
        return [[n, (repr(p.default) if p.default is not inspect.Parameter.empty else None)]
                for n, p in inspect.signature(fn).parameters.items() if n not in ("self", "kwargs")]

    def ast_sig_and_layers(rel, cls_name):
        import make_gru_golden as MG
        cls = MG._class_node(os.path.join(ref, rel), cls_name)
        init = next(n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name == "__init__")
        args = init.args.args[1:]
        defaults = [None] * (len(args) - len(init.args.defaults)) + [ast.unparse(d) for d in init.args.defaults]
        calls = sorted((n for n in ast.walk(init) if isinstance(n, ast.Call) and "DenseLayer" in ast.unparse(n.func)),
                       key=lambda n: n.lineno)
        names = [ast.unparse(k.value) for n in calls for k in n.keywords if k.arg == "name"]
        return [[a.arg, d] for a, d in zip(args, defaults)], names

    api = dict(DDPG=sig(DDPG.__init__), SimpleReplayPool=sig(SimpleReplayPool.__init__),
               OUStrategy=sig(OUStrategy.__init__), GaussianStrategy=sig(GaussianStrategy.__init__))
    for rel, cls_name in (("rllab/policies/deterministic_mlp_policy.py", "DeterministicMLPPolicy"),
                          ("rllab/q_functions/continuous_mlp_q_function.py", "ContinuousMLPQFunction")):
        api[cls_name], api[cls_name + "_dense_layer_names"] = ast_sig_and_layers(rel, cls_name)
    with open(os.path.join(HERE, "reference_api_ddpg.json"), "w") as f:
        json.dump(api, f, indent=1)


if __name__ == "__main__":
    main()
