"""Discrete space, API of rllab/spaces/discrete.py (without the Theano tensor-variable factory): the actions {0, ..., n-1},
flattened to one-hot vectors of length n."""
import numpy as np


class Discrete(object):
    def __init__(self, n):
        self._n = int(n)

    @property
    def n(self):
        return self._n

    def sample(self):
        return np.random.randint(self.n)

    def contains(self, x):
        x = np.asarray(x)
        return x.shape == () and x.dtype.kind == 'i' and 0 <= x < self.n

    def __repr__(self):
        return "Discrete(%d)" % self.n

    def __eq__(self, other):
        return isinstance(other, Discrete) and self.n == other.n

    def __hash__(self):
        return hash(self.n)

    def flatten(self, x):
        ret = np.zeros(self.n)
        ret[x] = 1
        return ret

    def unflatten(self, x):
        return np.nonzero(x)[0][0]

    def flatten_n(self, x):
        x = np.asarray(x, dtype=int).reshape(-1)
        ret = np.zeros((len(x), self.n))
        ret[np.arange(len(x)), x] = 1
        return ret

    def unflatten_n(self, x):
        if len(x) == 0:
            return []
        return np.nonzero(x)[1]

    @property
    def flat_dim(self):
        return self.n

    def weighted_sample(self, weights):
        """special.weighted_sample: the first index whose cumulative weight reaches np.random.rand(), clipped to n-1."""
        idx = int(np.sum(np.cumsum(weights) < np.random.rand()))
        return min(idx, self.n - 1)

    @property
    def default_value(self):
        return 0
