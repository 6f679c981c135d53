"""Device-backed environments.  One class per env kind of include/b200rl.h; each exposes

  * the reference's single-environment protocol  Env.reset() / Env.step(action)  (rllab/envs/base.py:6-100) backed by a
    one-lane device state (API parity: `rollout()`-style callers keep working; not the fast path), and
  * the reference's batched-lane hook  env.vectorized / env.vec_env_executor(n_envs, max_path_length)
    (sandbox/rocky/tf/samplers/vectorized_sampler.py:26-37, sandbox/rocky/tf/envs/vec_env_executor.py:6-46),
  * `env_kind`, which the fused sampler (rllab_b200/sampler/lane_sampler.py) hands to b200rl_rollout.

There is no CPU fallback: constructing an env needs libb200rl.so, stepping it needs a CUDA device.
"""
import numpy as np

from .. import _lib as L
from ..spaces import Box, Discrete
from .base import Env, Step

BIG = 1e6


def _device():
    import torch
    if not torch.cuda.is_available():
        raise L.B200RLError("a CUDA device is required to step rllab_b200 environments (no CPU fallback)")
    return torch.device("cuda", torch.cuda.current_device())


def require_defaults(cls_name, given, supported):
    """The device kernels implement the reference envs at their default construction arguments; anything else is
    rejected loudly rather than silently ignored."""
    for k, v in given.items():
        if k not in supported:
            raise TypeError("%s() got an unexpected keyword argument %r" % (cls_name, k))
        if v is not None and v != supported[k]:
            raise NotImplementedError("%s(%s=%r): only the reference default %r is built into the CUDA dynamics"
                                      % (cls_name, k, v, supported[k]))


class LaneEnv(Env):
    """Base of the device-backed envs.  Subclasses set ENV_NAME and (optionally) HORIZON."""
    ENV_NAME = None
    HORIZON = None

    def __init__(self):
        self.env_kind = L.ENV_KINDS[self.ENV_NAME] if self.ENV_NAME in L.ENV_KINDS else L.DISCRETE_ENV_KINDS[self.ENV_NAME]
        self._info = L.env_info(self.env_kind)
        self._n_actions = L.env_num_actions(self.env_kind)
        self._one = None          # lazily created one-lane device buffers
        self._normalized = False  # toggled by NormalizedEnv

    # ---- static description
    @property
    def observation_space(self):
        ub = BIG * np.ones(self._info["obs_dim"])
        return Box(-ub, ub)

    @property
    def action_space(self):
        if self._n_actions > 0:             # the action is an index: env_step reads it as one float
            return Discrete(self._n_actions)
        return Box(np.array(self._info["lb"], dtype=np.float64), np.array(self._info["ub"], dtype=np.float64))

    @property
    def action_bounds(self):
        return self.action_space.bounds

    @property
    def horizon(self):
        if self.HORIZON is None:
            raise NotImplementedError
        return self.HORIZON

    # ---- noise plumbing shared by the scalar and the vector API: np.random drives the reset, like the reference
    def _raw_reset_noise(self, n):
        K = self._info["reset_dim"]
        if self._info["noise_kind"] == L.NOISE_UNIFORM:
            return np.random.uniform(size=(K, n)).astype(np.float32)
        return np.random.normal(size=(K, n)).astype(np.float32)

    # ---- single-environment protocol
    def _buffers(self):
        if self._one is None:
            self._one = LaneState(self, 1)
        return self._one

    def reset(self):
        st = self._buffers()
        return st.reset()[0]

    def step(self, action):
        st = self._buffers()
        obs, rew, done = st.step(np.asarray(action, dtype=np.float64).reshape(1, -1), self._normalized)
        return Step(observation=obs[0], reward=float(rew[0]), done=bool(done[0]))

    # ---- batched-lane hook
    vectorized = True

    def vec_env_executor(self, n_envs, max_path_length):
        return VecEnvExecutor(self, n_envs, max_path_length)

    def __getstate__(self):
        d = dict(self.__dict__)
        d["_one"] = None
        return d


class LaneState(object):
    """n lanes of device state for the step-at-a-time API."""

    def __init__(self, env, n):
        import torch
        self.env, self.n = env, n
        dev = _device()
        info = env._info
        self.state = torch.zeros((info["state_dim"], n), dtype=torch.float32, device=dev)
        self.obs = torch.zeros((info["obs_dim"], n), dtype=torch.float32, device=dev)
        self.act = torch.zeros((info["act_dim"], n), dtype=torch.float32, device=dev)
        self.rew = torch.zeros((n,), dtype=torch.float32, device=dev)
        self.done = torch.zeros((n,), dtype=torch.uint8, device=dev)
        self.dev = dev

    def reset(self, mask=None):
        """Reset all lanes (mask None) or the masked lanes; returns obs (n, O) float64 on the host."""
        import torch
        from .. import ops
        raw = torch.as_tensor(self.env._raw_reset_noise(self.n), device=self.dev)
        if mask is None:
            ops.env_reset(self.env.env_kind, self.n, self.state, self.obs, raw)
        else:
            st2, ob2 = torch.empty_like(self.state), torch.empty_like(self.obs)
            ops.env_reset(self.env.env_kind, self.n, st2, ob2, raw)
            m = torch.as_tensor(np.asarray(mask, dtype=bool), device=self.dev)
            self.state[:, m] = st2[:, m]
            self.obs[:, m] = ob2[:, m]
        return self.obs.t().double().cpu().numpy()

    def step(self, actions, normalized):
        import torch
        from .. import ops
        a = np.ascontiguousarray(np.asarray(actions, dtype=np.float32).T)       # (A, n)
        self.act.copy_(torch.as_tensor(a))
        ops.env_step(self.env.env_kind, self.n, self.state, self.act, self.obs, self.rew, self.done, normalized)
        return (self.obs.t().double().cpu().numpy(), self.rew.double().cpu().numpy(),
                self.done.cpu().numpy().astype(bool))


class VecEnvExecutor(object):
    """sandbox/rocky/tf/envs/vec_env_executor.py:6-46 over device lanes: step(action_n) -> (obs, rewards, dones,
    env_infos) with the horizon cut and auto-reset (the returned obs of a finished lane is its reset obs)."""

    def __init__(self, env, n_envs, max_path_length):
        inner = env
        normalized = False
        while hasattr(inner, "wrapped_env"):
            normalized = True
            inner = inner.wrapped_env
        self._env = env
        self._inner = inner
        self._normalized = normalized
        self._st = LaneState(inner, n_envs)
        self.ts = np.zeros(n_envs, dtype="int")
        self.max_path_length = max_path_length

    def step(self, action_n):
        obs, rewards, dones = self._st.step(np.asarray(action_n), self._normalized)
        self.ts += 1
        if self.max_path_length is not None:
            dones[self.ts >= self.max_path_length] = True
        if dones.any():
            obs_reset = self._st.reset(mask=dones)
            obs[dones] = obs_reset[dones]
            self.ts[dones] = 0
        return obs, rewards, dones, dict()

    def reset(self):
        self.ts[:] = 0
        return self._st.reset()

    @property
    def num_envs(self):
        return self._st.n

    @property
    def action_space(self):
        return self._env.action_space

    @property
    def observation_space(self):
        return self._env.observation_space

    def terminate(self):
        pass
