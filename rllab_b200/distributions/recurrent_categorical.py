"""RecurrentCategorical, host-side numeric API of rllab/distributions/recurrent_categorical.py (kl / log_likelihood /
entropy / dist_info_keys) on the padded (n_paths, max_len, n) arrays of a recurrent samples_data.  The *_sym graph
builders have no counterpart: their compiled functions are the CUDA kernels of csrc/gru.cu
(b200rl_categorical_gru_loss_kl / _grad / _fvp)."""
import numpy as np

from .categorical import TINY, Categorical


class RecurrentCategorical(object):
    def __init__(self, dim):
        self._cat = Categorical(dim)
        self._dim = dim

    @property
    def dim(self):
        return self._dim

    def kl(self, old_dist_info, new_dist_info):
        old_prob, new_prob = old_dist_info["prob"], new_dist_info["prob"]
        return np.sum(old_prob * (np.log(old_prob + TINY) - np.log(new_prob + TINY)), axis=2)

    def log_likelihood(self, xs, dist_info):
        """log(p[x] + TINY) per (path, step); xs one-hot (n_paths, max_len, n), as the reference's flat
        log_likelihood_sym over the reshaped arrays."""
        probs = np.asarray(dist_info["prob"])
        a_dim = probs.shape[-1]
        flat = self._cat.log_likelihood(np.asarray(xs).reshape((-1, a_dim)), dict(prob=probs.reshape((-1, a_dim))))
        return flat.reshape(probs.shape[:2])

    def entropy(self, dist_info):
        probs = dist_info["prob"]
        return -np.sum(probs * np.log(probs + TINY), axis=2)

    @property
    def dist_info_keys(self):
        return ["prob"]
