"""Float64 oracle of the KL-penalty term of PPO's objective: the closed-form gradient of mean KL(old || new) over a
batch, by the manual back-propagation of oracle/policy.py.  With oracle.policy.grad_surr it gives the gradient of the
penalised objective surrogate + penalty * mean KL (penalty_lbfgs_optimizer.py:52-63 over npo.py:72-82) that
b200rl_grad_penalized computes."""
import numpy as np

from oracle import policy as P


def grad_mean_kl(flat, batch, dims, min_std=1e-6):
    """Gradient of mean_s KL(old_s || new_s) (diagonal_gaussian.py:36-56, with its +1e-8) with respect to the flat
    parameters; the log_std slot is 0 where the min_std clamp is active (TT.maximum passes the gradient to the larger
    argument)."""
    mean, log_std, acts = P.forward(flat, batch["obs"], dims, min_std, keep=True)
    B = mean.shape[0]
    var = np.exp(2.0 * log_std)
    var_old = np.exp(2.0 * np.asarray(batch["old_log_std"], dtype=np.float64)) * np.ones_like(mean)
    den = 2.0 * var + 1e-8
    dm = batch["old_mean"] - mean
    num = dm * dm + var_old - var
    dmean = (-2.0 * dm / den) / B
    dlog_std = (1.0 - 2.0 * var * (den + 2.0 * num) / den ** 2).sum(axis=0) / B
    if min_std is not None:
        ts = P.unpack(flat, dims)
        dlog_std = np.where(ts[-1] > np.log(min_std), dlog_std, 0.0)
    return P._backward(flat, dims, acts, dmean, dlog_std)


def grad_penalized(flat, batch, dims, kind, penalty, min_std=1e-6):
    return P.grad_surr(flat, batch, dims, kind, min_std) + penalty * grad_mean_kl(flat, batch, dims, min_std)


def penalized_loss(flat, batch, dims, kind, penalty, min_std=1e-6):
    """(loss + penalty * mean KL, loss, mean KL)"""
    loss = (P.surr_loss_trpo if kind == "trpo" else P.surr_loss_vpg)(flat, batch, dims, min_std)
    mkl = P.kl_stats(flat, batch, dims, min_std)[0]
    return loss + penalty * mkl, loss, mkl
