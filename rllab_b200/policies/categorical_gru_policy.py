"""CategoricalGRUPolicy with device-resident parameters (API of rllab/policies/categorical_gru_policy.py +
rllab/core/network.py GRUNetwork with output_nonlinearity=softmax).

Net: one GRU layer (tanh candidate, sigmoid gates) over x_t = [obs_t, one-hot prev_action_t] (state_include_action=True)
or obs_t, and a softmax output layer over the n actions.  h_0 is the constant zero vector (hidden_init_trainable=False),
so it is not a parameter.  Flat layout (in add_param order): [W_xr, W_hr, b_r, W_xu, W_hu, b_u, W_xc, W_hc, b_c, W_out,
b_out]; GlorotUniform weights and zero biases.  Parameters live on the GPU as the MLP policies' float64 master + float32
shadow.

get_action / get_actions run b200rl_categorical_gru_get_actions for the probabilities and the next hidden state on the
policy's own per-row state (prev_action, hidden), and draw each action on the host with weighted_sample on
np.random.rand(), as the reference does; reset(dones) clears the rows of finished paths.  The fused sampler carries the
same state per lane inside b200rl_rollout_categorical_gru and draws from the in-kernel Philox stream instead.
"""
import numpy as np

from .. import _lib as L
from ..distributions.recurrent_categorical import RecurrentCategorical
from ..spaces import Discrete


class CategoricalGRUPolicy(object):
    def __init__(self, env_spec, hidden_dim=32, feature_network=None, state_include_action=True,
                 hidden_nonlinearity=None, seed=None):
        """hidden_nonlinearity: tanh (None means tanh, the reference's default NL.tanh)."""
        assert isinstance(env_spec.action_space, Discrete)
        if feature_network is not None:
            raise NotImplementedError("feature networks are not built for the categorical GRU kernels "
                                      "(feature_network must be None)")
        if hidden_nonlinearity is not None and getattr(hidden_nonlinearity, "__name__", "") != "tanh":
            raise NotImplementedError("the GRU kernels implement a tanh candidate (hidden_nonlinearity must be tanh)")
        self._ctor = dict(hidden_dim=int(hidden_dim), state_include_action=bool(state_include_action))
        self._env_spec = env_spec
        self.obs_dim = int(env_spec.observation_space.flat_dim)
        self.action_dim = int(env_spec.action_space.n)
        self.hidden = self.hidden_dim = int(hidden_dim)
        self.state_include_action = bool(state_include_action)
        self.input_dim = self.obs_dim + (self.action_dim if self.state_include_action else 0)
        # h1 / h2 size the batch's activation cache: [hidden][T][N], h_t of every sample
        self.h1, self.h2 = self.hidden, 0
        self.min_std = None
        self.n_params = L.categorical_gru_num_params(self.obs_dim, self.hidden, self.action_dim,
                                                     self.state_include_action)   # raises if unsupported
        self._dist = RecurrentCategorical(self.action_dim)
        self._theta64 = None
        self._theta32 = None
        self._pin = None
        self.version = 0
        rng = np.random if seed is None else np.random.RandomState(seed)
        self._host_init = self._init_values(rng)
        self._prev_actions = None
        self._prev_hiddens = None
        self.reset()

    @property
    def dims(self):
        from ..ops import CategoricalGRUDims
        return CategoricalGRUDims(self.obs_dim, self.hidden, self.action_dim, self.state_include_action)

    def _shapes(self):
        I, H, n = self.input_dim, self.hidden, self.action_dim
        return [(I, H), (H, H), (H,)] * 3 + [(H, n), (n,)]

    def _init_values(self, rng):
        """GlorotUniform weights / zero biases (core/network.py GRULayer and the softmax DenseLayer)."""
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
    vectorized = _G.vectorized
    distribution = _G.distribution
    terminate = _G.terminate
    del _G

    def get_param_shapes(self, **tags):
        return self._shapes()

    @property
    def recurrent(self):
        return True

    @property
    def state_info_keys(self):
        return ["prev_action"] if self.state_include_action else []

    def reset(self, dones=None):
        """Clear the state of the rows whose path ended (all rows, and one row, when dones is None)."""
        if dones is None:
            dones = [True]
        dones = np.asarray(dones, dtype=bool).reshape(-1)
        if self._prev_actions is None or len(dones) != len(self._prev_actions):
            self._prev_actions = np.zeros((len(dones), self.action_dim))
            self._prev_hiddens = np.zeros((len(dones), self.hidden))
        self._prev_actions[dones] = 0.0
        self._prev_hiddens[dones] = 0.0

    def _step(self, flat_obs, prev_actions, prev_hiddens):
        """(prob (n, n_actions), h_out (n, H)) of one GRU step on the device."""
        import torch
        from .. import ops
        n = flat_obs.shape[0]
        th32 = self._ensure_device()[1]
        dev = th32.device

        def t(a):
            return torch.as_tensor(np.ascontiguousarray(np.asarray(a).T), dtype=torch.float32).to(dev)
        # the entry point also draws an action (here with u = 0, always action 0); it is discarded: the action is drawn
        # on the host with np.random, as the reference does
        act = torch.empty(n, dtype=torch.int32, device=dev)
        prob = torch.empty((self.action_dim, n), dtype=torch.float32, device=dev)
        h_out = torch.empty((self.hidden, n), dtype=torch.float32, device=dev)
        ops.categorical_gru_get_actions(th32, self.dims, t(flat_obs), t(prev_actions) if self.state_include_action
                                        else None, t(prev_hiddens), n, torch.zeros(n, dtype=torch.float32, device=dev),
                                        0, 0, 0, 0, act, prob, h_out)
        return prob.t().double().cpu().numpy(), h_out.t().double().cpu().numpy()

    def get_actions(self, observations):
        flat_obs = self.observation_space.flatten_n(observations)
        n = flat_obs.shape[0]
        if len(self._prev_actions) != n:
            raise ValueError("get_actions got %d observations but the policy holds the state of %d rows: call "
                             "reset(dones) with one entry per row first" % (n, len(self._prev_actions)))
        prev = self._prev_actions.copy()
        probs, hidden = self._step(flat_obs, prev, self._prev_hiddens)
        actions = np.array([self.action_space.weighted_sample(p) for p in probs], dtype=int)
        self._prev_actions = self.action_space.flatten_n(actions)
        self._prev_hiddens = hidden
        info = dict(prob=probs)
        if self.state_include_action:
            info["prev_action"] = prev
        return actions, info

    def get_action(self, observation):
        actions, info = self.get_actions([observation])
        return actions[0], {k: v[0] for k, v in info.items()}

    def log_diagnostics(self, paths):
        pass

    def __getstate__(self):
        return dict(env_spec=self._env_spec, ctor=self._ctor, params=self.get_param_values())

    def __setstate__(self, d):
        self.__init__(d["env_spec"], **d["ctor"])
        self.set_param_values(d["params"])
