"""OUStrategy (rllab/exploration_strategies/ou_strategy.py): x <- x + theta (mu - x) + sigma N(0, 1), reset to mu at every
path start; action = clip(policy(obs) + x, low, high).  get_action here draws from np.random like the reference; DDPG
runs the same process inside its fused kernel on the Philox stream of include/b200rl.h."""
import numpy as np

from ..spaces import Box
from .base import ExplorationStrategy


class OUStrategy(ExplorationStrategy):
    ES_KIND = 0

    def __init__(self, env_spec, mu=0, theta=0.15, sigma=0.3, **kwargs):
        assert isinstance(env_spec.action_space, Box)
        assert len(env_spec.action_space.shape) == 1
        self._env_spec = env_spec
        self.mu, self.theta, self.sigma = mu, theta, sigma
        self.action_space = env_spec.action_space
        self.reset()

    def reset(self):
        self.state = np.ones(self.action_space.flat_dim) * self.mu

    def evolve_state(self):
        x = self.state
        self.state = x + (self.theta * (self.mu - x) + self.sigma * np.random.randn(len(x)))
        return self.state

    def get_action(self, t, observation, policy, **kwargs):
        action, _ = policy.get_action(observation)
        ou_state = self.evolve_state()
        return np.clip(action + ou_state, self.action_space.low, self.action_space.high)

    def __getstate__(self):
        return dict(env_spec=self._env_spec, mu=self.mu, theta=self.theta, sigma=self.sigma, state=self.state)

    def __setstate__(self, d):
        self.__init__(d["env_spec"], mu=d["mu"], theta=d["theta"], sigma=d["sigma"])
        self.state = d["state"]
