"""CategoricalMLPPolicy with device-resident parameters (API of rllab/policies/categorical_mlp_policy.py +
rllab/policies/base.py + rllab/core/parameterized.py).

Net: MLP(obs_dim -> 32 -> 32 -> n), tanh hidden units, softmax output (core/network.py:36-81); flat layout
[W0, b0, W1, b1, Wout, bout] (core/lasagne_powered.py:16-20), GlorotUniform weights and zero biases.  Parameters live on
the GPU as a float64 master vector plus the float32 shadow the kernels read, as GaussianMLPPolicy's.  get_actions runs
b200rl_categorical_get_actions for the probabilities and draws each action on the host with weighted_sample on
np.random.rand(), one draw per observation in order, as the reference does (categorical_mlp_policy.py:88-92); the fused
sampler draws from the in-kernel Philox stream instead.
"""
import numpy as np

from .. import _lib as L
from ..distributions.categorical import Categorical
from ..spaces import Discrete


class CategoricalMLPPolicy(object):
    def __init__(self, env_spec, hidden_sizes=(32, 32), hidden_nonlinearity=None, num_seq_inputs=1, prob_network=None,
                 seed=None):
        assert isinstance(env_spec.action_space, Discrete)
        if prob_network is not None:
            raise NotImplementedError("only the MLP prob network is on the B200 hot path (prob_network must be None)")
        if hidden_nonlinearity is not None:
            raise NotImplementedError("B200 kernels implement tanh hidden units (hidden_nonlinearity must be None)")
        if num_seq_inputs != 1:
            raise NotImplementedError("num_seq_inputs != 1 is not built (the kernels read one observation per sample)")
        if tuple(hidden_sizes) != (32, 32):
            raise NotImplementedError("the categorical kernels are compiled for hidden_sizes=(32, 32) (got %r)"
                                      % (tuple(hidden_sizes),))
        self._ctor = dict(hidden_sizes=tuple(hidden_sizes))
        self._env_spec = env_spec
        self.obs_dim = int(env_spec.observation_space.flat_dim)
        self.action_dim = int(env_spec.action_space.n)
        self.h1, self.h2 = 32, 32
        self.min_std = None
        self.n_params = L.categorical_num_params(self.obs_dim, self.h1, self.h2, self.action_dim)  # raises if unsupported
        self._dist = Categorical(self.action_dim)
        self._theta64 = None
        self._theta32 = None
        self._pin = None
        self.version = 0
        rng = np.random if seed is None else np.random.RandomState(seed)
        self._host_init = self._init_values(rng)

    @property
    def dims(self):
        from ..ops import CategoricalDims
        return CategoricalDims(self.obs_dim, self.h1, self.h2, self.action_dim)

    def _shapes(self):
        O, h1, h2, n = self.obs_dim, self.h1, self.h2, self.action_dim
        return [(O, h1), (h1,), (h1, h2), (h2,), (h2, n), (n,)]

    def _init_values(self, rng):
        """GlorotUniform weights / zero biases (core/network.py:38-39)."""
        vals = []
        for s in self._shapes():
            if len(s) == 2:
                a = np.sqrt(6.0 / (s[0] + s[1]))
                vals.append(rng.uniform(-a, a, size=s).reshape(-1))
            else:
                vals.append(np.zeros(s))
        return np.concatenate(vals)

    # the parameter storage is GaussianMLPPolicy's: float64 master + float32 shadow on the device
    from .gaussian_mlp_policy import GaussianMLPPolicy as _G
    _ensure_device = _G._ensure_device
    theta64 = _G.theta64
    theta32 = _G.theta32
    bump_version = _G.bump_version
    get_param_values = _G.get_param_values
    set_param_values = _G.set_param_values
    set_param_values_device = _G.set_param_values_device
    flat_to_params = _G.flat_to_params
    observation_space = _G.observation_space
    action_space = _G.action_space
    recurrent = _G.recurrent
    vectorized = _G.vectorized
    state_info_keys = _G.state_info_keys
    distribution = _G.distribution
    reset = _G.reset
    terminate = _G.terminate
    del _G

    def get_param_shapes(self, **tags):
        return self._shapes()

    def _probs(self, observations):
        import torch
        from .. import ops
        flat_obs = self.observation_space.flatten_n(observations)
        n = flat_obs.shape[0]
        th32 = self._ensure_device()[1]
        dev = th32.device
        obs = torch.as_tensor(np.ascontiguousarray(flat_obs.T), dtype=torch.float32).to(dev)
        u = torch.zeros(n, dtype=torch.float32, device=dev)
        act = torch.empty(n, dtype=torch.int32, device=dev)
        prob = torch.empty((self.action_dim, n), dtype=torch.float32, device=dev)
        ops.categorical_get_actions(th32, self.dims, obs, n, u, 0, 0, 0, 0, act, prob)
        return prob.t().double().cpu().numpy()

    def get_actions(self, observations):
        probs = self._probs(observations)
        actions = np.array([self.action_space.weighted_sample(p) for p in probs], dtype=int)
        return actions, dict(prob=probs)

    def get_action(self, observation, deterministic=False):
        prob = self._probs([observation])[0]
        action = int(np.argmax(prob)) if deterministic else self.action_space.weighted_sample(prob)
        return action, dict(prob=prob)

    def dist_info(self, obs, state_infos=None):
        return dict(prob=self._probs(obs))

    def log_diagnostics(self, paths):
        pass

    def __getstate__(self):
        return dict(env_spec=self._env_spec, ctor=self._ctor, params=self.get_param_values())

    def __setstate__(self, d):
        self.__init__(d["env_spec"], **d["ctor"])
        self.set_param_values(d["params"])
