"""GaussianStrategy (rllab/exploration_strategies/gaussian_strategy.py): action = clip(policy(obs) + sigma N(0, 1), low,
high) with sigma = max_sigma - (max_sigma - min_sigma) min(1, t / decay_period).  DDPG runs it inside its fused kernel on
the Philox stream of include/b200rl.h."""
import numpy as np

from ..spaces import Box
from .base import ExplorationStrategy


class GaussianStrategy(ExplorationStrategy):
    ES_KIND = 1

    def __init__(self, env_spec, max_sigma=1.0, min_sigma=0.1, decay_period=1000000):
        assert isinstance(env_spec.action_space, Box)
        assert len(env_spec.action_space.shape) == 1
        self._env_spec = env_spec
        self._max_sigma, self._min_sigma, self._decay_period = max_sigma, min_sigma, decay_period
        self._action_space = env_spec.action_space

    def sigma(self, t):
        return self._max_sigma - (self._max_sigma - self._min_sigma) * min(1.0, t * 1.0 / self._decay_period)

    def get_action(self, t, observation, policy, **kwargs):
        action, _ = policy.get_action(observation)
        return np.clip(action + np.random.normal(size=len(action)) * self.sigma(t), self._action_space.low,
                       self._action_space.high)

    def __getstate__(self):
        return dict(env_spec=self._env_spec, max_sigma=self._max_sigma, min_sigma=self._min_sigma,
                    decay_period=self._decay_period)

    def __setstate__(self, d):
        self.__init__(d["env_spec"], d["max_sigma"], d["min_sigma"], d["decay_period"])
