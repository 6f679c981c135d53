"""ContinuousMLPQFunction (API of rllab/q_functions/continuous_mlp_q_function.py) with the reference's defaults:
obs -> 32 ReLU -> concat(hidden, action) -> 32 ReLU -> 1 linear (action_merge_layer=-2); flat layout [h1.W (O,32),
h1.b, h2.W (32+A,32) (hidden rows first), h2.b, output.W (32,1), output.b].  Initialisation as DeterministicMLPPolicy's.
get_qval runs b200rl_qf_get_qval on a float32 copy of the parameters.
"""
import numpy as np

from ..policies.deterministic_mlp_policy import HIDDEN, FlatParams, _require_mlp, init_values
from ..spaces import Box
from .base import QFunction


class ContinuousMLPQFunction(QFunction, FlatParams):
    def __init__(self, env_spec, hidden_sizes=(32, 32), hidden_nonlinearity=None, hidden_W_init=None,
                 hidden_b_init=None, action_merge_layer=-2, output_nonlinearity=None, output_W_init=None,
                 output_b_init=None, bn=False, seed=None):
        n_layers = len(hidden_sizes) + 1
        _require_mlp("ContinuousMLPQFunction", hidden_sizes, hidden_nonlinearity, bn,
                     [("action_merge_layer other than -2", (action_merge_layer % n_layers + n_layers) % n_layers == 1),
                      ("an output nonlinearity", output_nonlinearity is None),
                      ("a custom initialiser", all(x is None for x in (hidden_W_init, hidden_b_init, output_W_init,
                                                                        output_b_init)))])
        if not isinstance(env_spec.action_space, Box):
            raise NotImplementedError("ContinuousMLPQFunction needs a Box action space")
        from .. import _lib as L
        self._env_spec = env_spec
        self._ctor = dict(hidden_sizes=tuple(hidden_sizes))
        self.obs_dim = int(env_spec.observation_space.flat_dim)
        self.action_dim = int(env_spec.action_space.flat_dim)
        self.n_params = L.ddpg_num_params(self.obs_dim, self.action_dim)[1]
        rng = np.random if seed is None else np.random.RandomState(seed)
        self._theta = init_values(self._shapes(), rng)

    def _shapes(self):
        O, A, h = self.obs_dim, self.action_dim, HIDDEN[0]
        return [(O, h), (h,), (h + A, h), (h,), (h, 1), (1,)]

    def get_qval(self, observations, actions):
        import torch
        from .. import ops
        obs = np.asarray(observations, np.float32).reshape(-1, self.obs_dim)
        act = np.asarray(actions, np.float32).reshape(-1, self.action_dim)
        n = obs.shape[0]
        o = torch.as_tensor(np.ascontiguousarray(obs.T)).cuda()
        a = torch.as_tensor(np.ascontiguousarray(act.T)).cuda()
        q = torch.empty(n, dtype=torch.float32, device=o.device)
        ops.qf_get_qval(self._device_params(), self.obs_dim, self.action_dim, o, a, n, q)
        return q.double().cpu().numpy()
