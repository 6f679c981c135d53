"""Categorical, host-side numeric API of rllab/distributions/categorical.py (kl / log_likelihood / entropy /
dist_info_keys).  The *_sym graph builders have no counterpart: their compiled functions are the CUDA kernels of
csrc/categorical.cu (b200rl_categorical_loss_kl / _grad / _fvp)."""
import numpy as np

TINY = 1e-8


def from_onehot(x_var):
    ret = np.zeros((len(x_var),), 'int32')
    nonzero_n, nonzero_a = np.nonzero(x_var)
    ret[nonzero_n] = nonzero_a
    return ret


class Categorical(object):
    def __init__(self, dim):
        self._dim = dim

    @property
    def dim(self):
        return self._dim

    def kl(self, old_dist_info, new_dist_info):
        old_prob, new_prob = old_dist_info["prob"], new_dist_info["prob"]
        return np.sum(old_prob * (np.log(old_prob + TINY) - np.log(new_prob + TINY)), axis=-1)

    def log_likelihood(self, xs, dist_info):
        probs = dist_info["prob"]
        N = probs.shape[0]
        return np.log(probs[np.arange(N), from_onehot(np.asarray(xs))] + TINY)

    def entropy(self, info):
        probs = info["prob"]
        return -np.sum(probs * np.log(probs + TINY), axis=1)

    @property
    def dist_info_keys(self):
        return ["prob"]
