"""Float64 restatement of the cross-entropy method's host arithmetic (rllab/algos/cem.py), for the CEM tests.

Per-episode statistics (discounted and undiscounted return), the member fitness (mean - stderr over the evals), the
std schedule, the batch_size criterion, the elite update and the tabular values.  Pinned to the reference's own
CEM.train by tests/golden/reference_cem_golden.npz (tests/golden/make_cem_golden.py).

One deliberate difference: elites are ordered by a STABLE sort of -f (ties to the lower member index), where the reference
uses numpy's default quicksort.  They agree whenever the fitness values are distinct.
"""
import numpy as np


def discounted_return(rewards, discount):
    """discount_cumsum(rewards, discount)[0] (rllab/misc/special.py)."""
    r = np.asarray(rewards, np.float64)
    return float(np.sum(r * discount ** np.arange(len(r))))


def stderr_lb(x):
    """_get_stderr_lb (cem.py:15-18) of a 1-D list of per-eval values; equals _get_stderr_lb_varyinglens(...)[0] for the
    returns at time index 0, which every eval has."""
    x = np.asarray(x, np.float64)
    return float(np.mean(x) - np.std(x, ddof=1 if len(x) > 1 else 0) / np.sqrt(len(x)))


def extra_var(itr, extra_std, extra_decay_time):
    return float(np.square(extra_std) * max(1.0 - itr / extra_decay_time, 0))


def sample_std(cur_std, itr, extra_std, extra_decay_time):
    """cem.py:117-118."""
    return np.sqrt(np.square(cur_std) + extra_var(itr, extra_std, extra_decay_time))


def theta_rows(cur_mean, cur_std, eps, itr, extra_std, extra_decay_time):
    """cem.py:34 for a batch of members: eps [n][P] standard normal draws."""
    return np.asarray(eps, np.float64) * sample_std(cur_std, itr, extra_std, extra_decay_time) + cur_mean


def n_best(n_samples, best_frac):
    return max(1, int(n_samples * best_frac))


def batch_prefix(last_lens, batch_size):
    """Members collected by run_collect with the 'samples' criterion: the shortest prefix whose last-episode lengths
    (cem.py:51) add up to batch_size."""
    c = np.cumsum(np.asarray(last_lens, np.float64))
    hit = np.nonzero(c >= batch_size)[0]
    assert len(hit), "population too short for batch_size"
    return int(hit[0]) + 1


def elite_update(xs, fs, nb):
    """cem.py:138-142: (best indices, cur_mean, cur_std, best_x)."""
    xs = np.asarray(xs, np.float64)
    fs = np.asarray(fs, np.float64)
    best = np.argsort(-fs, kind="stable")[:nb]
    bx = xs[best]
    return best, bx.mean(axis=0), bx.std(axis=0), bx[0]


def average_policy_std(xs, lens, act_dim, min_std=1e-6):
    """GaussianMLPPolicy.log_diagnostics over every step of every episode (lens [members][evals]): each member's
    state-independent std counts once per step its episodes ran."""
    ls = np.maximum(np.asarray(xs, np.float64)[:, -act_dim:], np.log(min_std))
    steps = np.asarray(lens, np.float64).reshape(len(ls), -1).sum(axis=1)
    return float(np.sum(np.mean(np.exp(ls), axis=1) * steps) / np.sum(steps))


def tabular(itr, cur_std, ustat, fs, lens):
    """The CEM keys of cem.py:144-160 (lens: every episode's length)."""
    ustat = np.asarray(ustat, np.float64)
    return dict(Iteration=itr, CurStdMean=float(np.mean(cur_std)), AverageReturn=float(np.mean(ustat)),
                StdReturn=float(np.std(ustat)), MaxReturn=float(np.max(ustat)), MinReturn=float(np.min(ustat)),
                AverageDiscountedReturn=float(np.mean(fs)), NumTrajs=len(fs),
                AvgTrajLen=float(np.mean(np.asarray(lens, np.float64))))
