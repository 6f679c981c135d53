"""Generate tests/golden/reference_categorical_golden.npz: the reference's own NumPy code for the categorical policy's
distribution, run verbatim through oracle/ref_shims.py on fixed inputs:
  * rllab/distributions/categorical.py  Categorical.kl / log_likelihood / entropy   (keys kl, loglik, entropy)
  * rllab/misc/special.py              weighted_sample_n after np.random.seed(SEED) (key ws_idx; the uniforms it drew
                                        are recorded as ws_u by re-seeding)
  * rllab/spaces/discrete.py           Discrete(n).flatten_n                          (key onehot)
on probability rows that include exact 0 / 1 entries and rows summing to slightly less than 1, so TINY's placement and
weighted_sample's comparison and clipping are pinned.

Run:  python tests/golden/make_categorical_golden.py   (needs the reference tree; the tests only read the committed file)
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import ref_shims  # noqa: E402

SEED = 123


def inputs():
    rng = np.random.RandomState(7)
    n, B = 3, 64
    z = rng.randn(B, n) * 2.0
    p = np.exp(z - z.max(axis=1, keepdims=True))
    p /= p.sum(axis=1, keepdims=True)
    q = np.exp(-z)
    q /= q.sum(axis=1, keepdims=True)
    p[0] = [1.0, 0.0, 0.0]
    q[1] = [0.0, 1.0, 0.0]
    p[2] = [0.3, 0.3, 0.3999999]              # sums below 1: the clip to n - 1
    idx = rng.randint(0, n, B)
    return p, q, idx, n


def main():
    ref_shims.install()
    from rllab.distributions.categorical import Categorical
    from rllab.misc import special
    from rllab.spaces.discrete import Discrete
    p, q, idx, n = inputs()
    d = Categorical(n)
    onehot = Discrete(n).flatten_n(idx)
    out = dict(p=p, q=q, idx=idx, n=n, onehot=onehot,
               kl=d.kl(dict(prob=q), dict(prob=p)), loglik=d.log_likelihood(onehot, dict(prob=p)),
               entropy=d.entropy(dict(prob=p)))
    np.random.seed(SEED)
    out["ws_idx"] = special.weighted_sample_n(p, np.arange(n))
    np.random.seed(SEED)
    out["ws_u"] = np.random.rand(p.shape[0])
    np.savez(os.path.join(HERE, "reference_categorical_golden.npz"), **out)


if __name__ == "__main__":
    main()
