"""GaussianMLPPolicy with device-resident parameters (API of rllab/policies/gaussian_mlp_policy.py:20-161 +
rllab/policies/base.py:4-77 + rllab/core/parameterized.py:54-84).

Parameters live on the GPU as a float64 master vector plus the float32 shadow the kernels read; the flat layout is the
reference's ([W0,b0,W1,b1,Wout,bout,log_std], core/lasagne_powered.py:16-20).  get_action / get_actions run
b200rl_policy_get_actions; the Gaussian noise comes from np.random on the host exactly like the reference
(gaussian_mlp_policy.py:128,135) -- the fused sampler uses the in-kernel Philox stream instead.
"""
import numpy as np

from .. import _lib as L
from ..distributions.diagonal_gaussian import DiagonalGaussian
from ..misc import logger
from ..spaces import Box


class GaussianMLPPolicy(object):
    def __init__(self, env_spec, hidden_sizes=(32, 32), learn_std=True, init_std=1.0, adaptive_std=False,
                 std_share_network=False, std_hidden_sizes=(32, 32), min_std=1e-6, std_hidden_nonlinearity=None,
                 hidden_nonlinearity=None, output_nonlinearity=None, mean_network=None, std_network=None,
                 dist_cls=DiagonalGaussian, seed=None):
        assert isinstance(env_spec.action_space, Box)
        if adaptive_std or std_share_network or mean_network is not None or std_network is not None:
            raise NotImplementedError("only the state-independent log_std ParamLayer head is on the B200 hot path")
        if hidden_nonlinearity is not None or output_nonlinearity is not None or not learn_std:
            raise NotImplementedError("B200 kernels implement tanh hidden units, a linear output and a learnt log_std")
        self._ctor = dict(hidden_sizes=tuple(hidden_sizes), init_std=init_std, min_std=min_std)
        self._env_spec = env_spec
        self.obs_dim = int(env_spec.observation_space.flat_dim)
        self.action_dim = int(env_spec.action_space.flat_dim)
        if len(hidden_sizes) != 2:
            raise NotImplementedError("B200 kernels implement two hidden layers (got %r)" % (hidden_sizes,))
        self.h1, self.h2 = int(hidden_sizes[0]), int(hidden_sizes[1])
        self.min_std = min_std
        self.n_params = L.policy_num_params(self.obs_dim, self.h1, self.h2, self.action_dim)   # raises if unsupported
        self._dist = dist_cls(self.action_dim)
        self._theta64 = None
        self._theta32 = None
        self._pin = None
        self.version = 0          # bumped whenever the parameters change (optimizers cache loss/KL per version)
        rng = np.random if seed is None else np.random.RandomState(seed)
        self._host_init = self._init_values(rng, init_std)

    # ---- construction helpers
    @property
    def dims(self):
        return (self.obs_dim, self.h1, self.h2, self.action_dim)

    def _shapes(self):
        O, h1, h2, A = self.dims
        return [(O, h1), (h1,), (h1, h2), (h2,), (h2, A), (A,), (A,)]

    def _init_values(self, rng, init_std):
        """GlorotUniform weights / zero biases / log(init_std)  (core/network.py:38-39, gaussian_mlp_policy.py:88-94)."""
        vals = []
        for s in self._shapes()[:-1]:
            if len(s) == 2:
                a = np.sqrt(6.0 / (s[0] + s[1]))
                vals.append(rng.uniform(-a, a, size=s).reshape(-1))
            else:
                vals.append(np.zeros(s))
        vals.append(np.full((self.action_dim,), np.log(init_std)))
        return np.concatenate(vals)

    def _ensure_device(self):
        if self._theta64 is None:
            import torch
            if not torch.cuda.is_available():
                raise L.B200RLError("GaussianMLPPolicy needs a CUDA device (no CPU fallback)")
            dev = torch.device("cuda", torch.cuda.current_device())
            self._theta64 = torch.as_tensor(self._host_init, dtype=torch.float64).to(dev)
            self._theta32 = self._theta64.to(torch.float32)
            self._pin = torch.empty(self.n_params, dtype=torch.float64).pin_memory()   # page-locked H2D staging
        return self._theta64, self._theta32

    @property
    def theta64(self):
        return self._ensure_device()[0]

    @property
    def theta32(self):
        return self._ensure_device()[1]

    def bump_version(self):
        self.version += 1

    # ---- Parameterized
    def get_param_values(self, **tags):
        if self._theta64 is None:
            return self._host_init.copy()
        return self._theta64.cpu().numpy()

    def set_param_values(self, flattened_params, **tags):
        flat = np.asarray(flattened_params, dtype=np.float64).reshape(-1)
        assert flat.size == self.n_params, (flat.size, self.n_params)
        self.version += 1
        if self._theta64 is None:
            self._host_init = flat.copy()
            return
        import torch
        if getattr(self, "_pin", None) is None:
            self._pin = torch.empty(self.n_params, dtype=torch.float64).pin_memory()   # page-locked staging buffer
        # the single pinned staging buffer may still be the source of an earlier, queued host->device copy: wait for that
        # copy (an event recorded right behind it) before overwriting the buffer
        ev = getattr(self, "_pin_event", None)
        if ev is not None:
            ev.synchronize()
        self._pin.copy_(torch.as_tensor(flat))
        self._theta64.copy_(self._pin, non_blocking=True)
        self._pin_event = torch.cuda.Event()
        self._pin_event.record()
        from .. import ops
        ops.f64_to_f32(self._theta64, self._theta32)  # value.astype(dtype), parameterized.py:68

    def set_param_values_device(self, theta64):
        """set_param_values from a float64 device tensor [P], without a host round trip (CEM's best row)."""
        from .. import ops
        th64, th32 = self._ensure_device()
        th64.copy_(theta64.reshape(-1))
        ops.f64_to_f32(th64, th32)
        self.version += 1

    def get_param_shapes(self, **tags):
        return self._shapes()

    def flat_to_params(self, flattened_params, **tags):
        out, k = [], 0
        for s in self._shapes():
            n = int(np.prod(s))
            out.append(np.asarray(flattened_params[k:k + n]).reshape(s))
            k += n
        return out

    # ---- Policy
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

    @property
    def distribution(self):
        return self._dist

    def reset(self, dones=None):
        pass

    def terminate(self):
        pass

    def get_actions(self, observations):
        import torch
        from .. import ops
        flat_obs = self.observation_space.flatten_n(observations)
        n = flat_obs.shape[0]
        th64, th32 = self._ensure_device()
        dev = th32.device
        obs = torch.as_tensor(np.ascontiguousarray(flat_obs.T), dtype=torch.float32).to(dev)
        rnd = np.random.normal(size=(n, self.action_dim))
        eps = torch.as_tensor(np.ascontiguousarray(rnd.T), dtype=torch.float32).to(dev)
        act = torch.empty((self.action_dim, n), dtype=torch.float32, device=dev)
        mean = torch.empty_like(act)
        ls = torch.empty((self.action_dim,), dtype=torch.float32, device=dev)
        O, h1, h2, A = self.dims
        ops.policy_get_actions(th32, O, h1, h2, A, self.min_std, obs, n, eps, 0, 0, 0, 0, act, mean, ls)
        means = mean.t().double().cpu().numpy()
        log_stds = np.tile(ls.double().cpu().numpy().reshape(1, -1), (n, 1))
        actions = act.t().double().cpu().numpy()
        return actions, dict(mean=means, log_std=log_stds)

    def get_action(self, observation):
        actions, info = self.get_actions([observation])
        return actions[0], {k: v[0] for k, v in info.items()}

    def dist_info(self, obs, state_infos=None):
        _, info = self.get_actions(obs)
        return info

    def log_diagnostics(self, paths):
        log_stds = np.vstack([path["agent_infos"]["log_std"] for path in paths])
        logger.record_tabular('AveragePolicyStd', np.mean(np.exp(log_stds)))

    # ---- Serializable (core/serializable.py:36-42 + parameterized.py:75-84): ctor args + flat params
    def __getstate__(self):
        return dict(env_spec=self._env_spec, ctor=self._ctor, params=self.get_param_values())

    def __setstate__(self, d):
        self.__init__(d["env_spec"], **d["ctor"])
        self.set_param_values(d["params"])
