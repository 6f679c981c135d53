"""DeterministicMLPPolicy (API of rllab/policies/deterministic_mlp_policy.py): MLP(obs_dim -> 32 -> 32 -> act_dim), ReLU
hidden units, tanh output; flat layout [h0.W, h0.b, h1.W, h1.b, output.W, output.b].  HeUniform hidden weights (lasagne
0.2, gain 1: U(+-sqrt(3 / fan_in)), fan_in = rows of W), zero hidden biases, Uniform(-3e-3, 3e-3) output W and b.

The parameters are a float64 host vector; get_actions runs b200rl_deterministic_get_actions on a float32 copy.  DDPG
trains the policy inside its fused kernel and writes the result back through set_param_values.
"""
import numpy as np

from ..spaces import Box

HIDDEN = (32, 32)


def _require_mlp(cls_name, hidden_sizes, hidden_nonlinearity, bn, extra=()):
    if bn:
        raise NotImplementedError("%s: batch normalization (bn=True) is not built" % cls_name)
    if tuple(hidden_sizes) != HIDDEN:
        raise NotImplementedError("%s: the DDPG kernels are compiled for hidden_sizes=(32, 32) (got %r)"
                                  % (cls_name, tuple(hidden_sizes)))
    if hidden_nonlinearity not in (None, "rectify", "relu"):
        raise NotImplementedError("%s: the DDPG kernels implement ReLU hidden units" % cls_name)
    for name, ok in extra:
        if not ok:
            raise NotImplementedError("%s: %s is not built" % (cls_name, name))


def init_values(shapes, rng):
    """HeUniform hidden weights, zero hidden biases, Uniform(-3e-3, 3e-3) output W and b."""
    vals = []
    for i, s in enumerate(shapes):
        if i >= len(shapes) - 2:
            vals.append(rng.uniform(-3e-3, 3e-3, size=s).reshape(-1))
        elif len(s) == 2:
            a = np.sqrt(3.0 / s[0])
            vals.append(rng.uniform(-a, a, size=s).reshape(-1))
        else:
            vals.append(np.zeros(s))
    return np.concatenate(vals)


class FlatParams(object):
    """Parameterized (rllab/core/parameterized.py) over a float64 host vector with `_shapes()`; pickles as the
    constructor arguments plus the flat values."""

    def get_param_values(self, regularizable=None, **tags):
        if regularizable:
            return np.concatenate([p.reshape(-1) for p, s in zip(self.flat_to_params(self._theta), self._shapes())
                                   if len(s) == 2])
        return self._theta.copy()

    def set_param_values(self, flattened_params, **tags):
        flat = np.asarray(flattened_params, dtype=np.float64).reshape(-1)
        assert flat.size == self.n_params, (flat.size, self.n_params)
        self._theta = flat.copy()

    def get_param_shapes(self, **tags):
        return self._shapes()

    def flat_to_params(self, flattened_params, **tags):
        out, k = [], 0
        for s in self._shapes():
            n = int(np.prod(s))
            out.append(np.asarray(flattened_params[k:k + n]).reshape(s))
            k += n
        return out

    def _device_params(self):
        import torch
        return torch.as_tensor(self._theta, dtype=torch.float32).cuda()

    def __getstate__(self):
        return dict(env_spec=self._env_spec, ctor=self._ctor, params=self.get_param_values())

    def __setstate__(self, d):
        self.__init__(d["env_spec"], **d["ctor"])
        self.set_param_values(d["params"])


class DeterministicMLPPolicy(FlatParams):
    def __init__(self, env_spec, hidden_sizes=(32, 32), hidden_nonlinearity=None, hidden_W_init=None,
                 hidden_b_init=None, output_nonlinearity=None, output_W_init=None, output_b_init=None, bn=False,
                 seed=None):
        """hidden_nonlinearity / output_nonlinearity: None means the reference's defaults (ReLU, tanh); the *_init
        arguments must be None (the reference's initialisers).  seed: RandomState seed of the initial values (None: the
        global np.random)."""
        _require_mlp("DeterministicMLPPolicy", hidden_sizes, hidden_nonlinearity, bn,
                     [("output_nonlinearity other than tanh", output_nonlinearity in (None, "tanh")),
                      ("a custom initialiser", all(x is None for x in (hidden_W_init, hidden_b_init, output_W_init,
                                                                        output_b_init)))])
        if not isinstance(env_spec.action_space, Box):
            raise NotImplementedError("DeterministicMLPPolicy needs a Box action space")
        from .. import _lib as L
        self._env_spec = env_spec
        self._ctor = dict(hidden_sizes=tuple(hidden_sizes))
        self.obs_dim = int(env_spec.observation_space.flat_dim)
        self.action_dim = int(env_spec.action_space.flat_dim)
        self.n_params = L.ddpg_num_params(self.obs_dim, self.action_dim)[0]   # raises if not compiled in
        rng = np.random if seed is None else np.random.RandomState(seed)
        self._theta = init_values(self._shapes(), rng)

    def _shapes(self):
        O, A, h = self.obs_dim, self.action_dim, HIDDEN[0]
        return [(O, h), (h,), (h, h), (h,), (h, A), (A,)]

    @property
    def observation_space(self):
        return self._env_spec.observation_space

    @property
    def action_space(self):
        return self._env_spec.action_space

    @property
    def recurrent(self):
        return False

    @property
    def vectorized(self):
        return True

    @property
    def state_info_keys(self):
        return list()

    def reset(self, dones=None):
        pass

    def terminate(self):
        pass

    def log_diagnostics(self, paths):
        pass

    def get_actions(self, observations):
        import torch
        from .. import ops
        flat = np.asarray(observations, np.float32).reshape(-1, self.obs_dim)
        n = flat.shape[0]
        obs = torch.as_tensor(np.ascontiguousarray(flat.T)).cuda()
        act = torch.empty((self.action_dim, n), dtype=torch.float32, device=obs.device)
        ops.deterministic_get_actions(self._device_params(), self.obs_dim, self.action_dim, obs, n, act)
        return act.t().double().cpu().numpy(), dict()

    def get_action(self, observation):
        actions, _ = self.get_actions([observation])
        return actions[0], dict()
