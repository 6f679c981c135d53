"""GaussianGRUPolicy with device-resident parameters (API of rllab/policies/gaussian_gru_policy.py +
rllab/core/network.py:104-270 GRUNetwork).

Net: one GRU layer (tanh candidate, sigmoid gates) over x_t = [obs_t, prev_action_t] (state_include_action=True) or
obs_t, a linear mean head and a state-independent log_std.  h_0 is the constant zero vector (GRUNetwork's
hidden_init_trainable=False), so it is not a parameter.  Flat layout (LasagnePowered over [l_mean, l_log_std], in
add_param order): [W_xr, W_hr, b_r, W_xu, W_hu, b_u, W_xc, W_hc, b_c, W_out, b_out, log_std]; GlorotUniform weights,
zero biases, log_std = log(init_std).  Parameters live on the GPU as the MLP policies' float64 master + float32 shadow.

get_action / get_actions run b200rl_gru_get_actions on the policy's own per-row state (prev_action, hidden), with the
noise drawn from np.random on the host like the reference; reset(dones) clears the rows of finished paths.  The fused
sampler carries the same state per lane inside b200rl_rollout_gru instead.
"""
import numpy as np

from .. import _lib as L
from ..distributions.recurrent_diagonal_gaussian import RecurrentDiagonalGaussian
from ..spaces import Box


class GaussianGRUPolicy(object):
    def __init__(self, env_spec, hidden_sizes=(32,), state_include_action=True, hidden_nonlinearity=None,
                 learn_std=True, init_std=1.0, output_nonlinearity=None, seed=None):
        assert isinstance(env_spec.action_space, Box)
        if len(hidden_sizes) != 1:
            raise ValueError("GaussianGRUPolicy has one recurrent layer (hidden_sizes must have one entry)")
        if hidden_nonlinearity is not None and getattr(hidden_nonlinearity, "__name__", "") != "tanh":
            raise NotImplementedError("the GRU kernels implement a tanh candidate (hidden_nonlinearity must be tanh)")
        if output_nonlinearity is not None:
            raise NotImplementedError("the GRU kernels implement a linear mean head (output_nonlinearity must be None)")
        if not learn_std:
            raise NotImplementedError("the GRU kernels implement a learnt log_std (learn_std must be True)")
        self._ctor = dict(hidden_sizes=tuple(hidden_sizes), state_include_action=bool(state_include_action),
                          init_std=init_std)
        self._env_spec = env_spec
        self.obs_dim = int(env_spec.observation_space.flat_dim)
        self.action_dim = int(env_spec.action_space.flat_dim)
        self.hidden = int(hidden_sizes[0])
        self.state_include_action = bool(state_include_action)
        self.input_dim = self.obs_dim + (self.action_dim if self.state_include_action else 0)
        # h1 / h2 size the batch's activation cache: [hidden][T][N], h_t of every sample
        self.h1, self.h2 = self.hidden, 0
        self.min_std = None
        self.n_params = L.gru_num_params(self.obs_dim, self.hidden, self.action_dim, self.state_include_action)
        self._dist = RecurrentDiagonalGaussian(self.action_dim)
        self._theta64 = None
        self._theta32 = None
        self._pin = None
        self.version = 0
        rng = np.random if seed is None else np.random.RandomState(seed)
        self._host_init = self._init_values(rng, init_std)
        self._prev_actions = None
        self._prev_hiddens = None
        self.reset()

    @property
    def dims(self):
        from ..ops import GRUDims
        return GRUDims(self.obs_dim, self.hidden, self.action_dim, self.state_include_action)

    def _shapes(self):
        I, H, A = self.input_dim, self.hidden, self.action_dim
        gate = [(I, H), (H, H), (H,)]
        return gate * 3 + [(H, A), (A,), (A,)]

    def _init_values(self, rng, init_std):
        """GlorotUniform weights / zero biases / log(init_std) (core/network.py GRULayer, gaussian_gru_policy.py)."""
        vals = []
        for s in self._shapes()[:-1]:
            if len(s) == 2:
                a = np.sqrt(6.0 / (s[0] + s[1]))
                vals.append(rng.uniform(-a, a, size=s).reshape(-1))
            else:
                vals.append(np.zeros(s))
        vals.append(np.full((self.action_dim,), np.log(init_std)))
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
    log_diagnostics = _G.log_diagnostics
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

    def get_actions(self, observations):
        import torch
        from .. import ops
        flat_obs = self.observation_space.flatten_n(observations)
        n = flat_obs.shape[0]
        if len(self._prev_actions) != n:
            raise ValueError("get_actions got %d observations but the policy holds the state of %d rows: call "
                             "reset(dones) with one entry per row first" % (n, len(self._prev_actions)))
        th32 = self._ensure_device()[1]
        dev = th32.device

        def t(a):
            return torch.as_tensor(np.ascontiguousarray(np.asarray(a).T), dtype=torch.float32).to(dev)
        rnd = np.random.normal(size=(n, self.action_dim))
        act = torch.empty((self.action_dim, n), dtype=torch.float32, device=dev)
        mean = torch.empty_like(act)
        h_out = torch.empty((self.hidden, n), dtype=torch.float32, device=dev)
        ls = torch.empty((self.action_dim,), dtype=torch.float32, device=dev)
        prev = self._prev_actions.copy()
        ops.gru_get_actions(th32, self.dims, t(flat_obs), t(prev) if self.state_include_action else None,
                            t(self._prev_hiddens), n, t(rnd), 0, 0, 0, 0, act, mean, h_out, ls)
        actions = act.t().double().cpu().numpy()
        means = mean.t().double().cpu().numpy()
        log_stds = np.tile(ls.double().cpu().numpy().reshape(1, -1), (n, 1))
        self._prev_actions = actions.copy()
        self._prev_hiddens = h_out.t().double().cpu().numpy()
        info = dict(mean=means, log_std=log_stds)
        if self.state_include_action:
            info["prev_action"] = prev
        return actions, info

    def get_action(self, observation):
        actions, info = self.get_actions([observation])
        return actions[0], {k: v[0] for k, v in info.items()}

    def __getstate__(self):
        return dict(env_spec=self._env_spec, ctor=self._ctor, params=self.get_param_values())

    def __setstate__(self, d):
        self.__init__(d["env_spec"], **d["ctor"])
        self.set_param_values(d["params"])
