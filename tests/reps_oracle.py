"""Oracle: REPS (rllab/algos/reps.py) in float64 NumPy.

TEST INFRASTRUCTURE ONLY.  Restates:
  * the feature map and feat_diff of reps.py:207-211,227-238, in the reference's path-list form and in the lane form of
    the device batch (obs [O][T][N], flags / tstep [T][N]: the successor of (t, n) is (t + 1, n) unless (t, n) carries
    FLAG_END, then phi = 0);
  * the Bellman error, the dual and its gradient (reps.py:101-102,164-187), the policy-step weights and loss
    (reps.py:106-118), the latter through oracle/policy.py;
  * optimize_policy (reps.py:214-333) as plain scipy calls on these callables.
"""
import numpy as np
import scipy.optimize

from oracle import policy as P

FLAG_END, FLAG_MASKED = 2, 8


def features(obs, tsteps=None):
    """reps.py:207-211 on one path (tsteps = 0..L-1 unless given)."""
    o = np.clip(np.asarray(obs, dtype=np.float64), -10, 10)
    n = len(o)
    al = (np.arange(n) if tsteps is None else np.asarray(tsteps, dtype=np.float64)).reshape(-1, 1) / 100.0
    return np.concatenate([o, o ** 2, al, al ** 2, al ** 3, np.ones((n, 1))], axis=1)


def feat_diff_paths(paths):
    """reps.py:228-238: per path phi(t+1) - phi(t) with phi(L) = 0, stacked in path order."""
    out = []
    for path in paths:
        f = features(path["observations"])
        f = np.vstack([f, np.zeros(f.shape[1])])
        out.append(f[1:] - f[:-1])
    return np.vstack(out)


def feat_diff_lanes(obs, flags, tstep):
    """Lane form: [T][N][2O+4] from obs [O][T][N] float32, flags / tstep [T][N]."""
    O, T, N = obs.shape
    o = np.moveaxis(np.asarray(obs, dtype=np.float64), 0, -1)             # [T][N][O]
    f = features(o.reshape(-1, O), np.asarray(tstep, dtype=np.float64).reshape(-1)).reshape(T, N, -1)
    nxt = np.zeros_like(f)
    nxt[:-1] = f[1:]
    nxt[(np.asarray(flags) & FLAG_END) != 0] = 0.0
    return nxt - f


def delta(rew, fd, v):
    return np.asarray(rew, dtype=np.float64) + fd @ np.asarray(v, dtype=np.float64)


def dual(eta, v, rew, fd, epsilon, l2_reg_dual=0.0):
    """reps.py:174-184, as written there."""
    eta = np.float64(eta)
    with np.errstate(all="ignore"):
        dv = delta(rew, fd, v) / eta
        m = np.max(dv)
        return (eta * epsilon + eta * np.log(np.mean(np.exp(dv - m))) + eta * m
                + l2_reg_dual * (np.square(eta) + np.square(1 / eta)))


def dual_grad(eta, v, rew, fd, epsilon, l2_reg_dual=0.0):
    """Gradient of `dual` in closed form (the max shift cancels): [dg/deta, dg/dv]."""
    eta = np.float64(eta)
    with np.errstate(all="ignore"):
        d = delta(rew, fd, v)
        M = np.max(d)
        e = np.exp((d - M) / eta)
        s = np.sum(e)
        g_eta = (epsilon + np.log(s / len(d)) - np.sum(e * (d - M)) / (eta * s)
                 + l2_reg_dual * (2 * eta - 2 / eta ** 3))
        return np.concatenate([[g_eta], (e @ fd) / s])


def weights(eta, v, rew, fd):
    """exp(delta / eta - max(delta / eta)): the per-sample weights of the policy loss (reps.py:110-112)."""
    eta = np.float64(eta)
    with np.errstate(all="ignore"):
        dv = delta(rew, fd, v) / eta
        return np.exp(dv - np.max(dv))


def reg_slices(dims):
    """W0, W1, Wout and log_std in the flat layout (lasagne's regularizable defaults; see rllab_b200/algos/reps.py)."""
    out, k = [], 0
    for i, s in enumerate(dims.shapes):
        n = int(np.prod(s))
        if len(s) == 2 or i == len(dims.shapes) - 1:
            out.append(slice(k, k + n))
        k += n
    return out


def policy_loss(theta, batch, w, dims, l2_reg_loss=0.0, min_std=1e-6):
    """-mean(logli * w) + L2_reg_loss * sum_p mean(p^2) / n_reg   (reps.py:110-118)."""
    mean, log_std = P.forward(theta, batch["obs"], dims, min_std)
    loss = -np.mean(P.log_likelihood(batch["actions"], mean, log_std) * w)
    reg = reg_slices(dims)
    return loss + l2_reg_loss * sum(np.mean(np.square(theta[s])) for s in reg) / len(reg)


def policy_grad(theta, batch, w, dims, l2_reg_loss=0.0, min_std=1e-6):
    g = P.grad_surr(theta, dict(batch, adv=w), dims, "vpg", min_std)
    reg = reg_slices(dims)
    for s in reg:
        g[s] += l2_reg_loss * 2.0 * theta[s] / (theta[s].size * len(reg))
    return g


def _lbfgs(optimizer, **kw):
    if optimizer is scipy.optimize.fmin_l_bfgs_b:
        kw.pop("disp", None)
    return optimizer(**kw)


def optimize_policy(eta, v, theta, batch, rew, fd, dims, epsilon=0.5, l2_reg_dual=0.0, l2_reg_loss=0.0,
                    max_opt_itr=50, min_std=1e-6, optimizer=scipy.optimize.fmin_l_bfgs_b, dual_fns=None, loss_fns=None):
    """reps.py:240-333 on float64 callables.  batch: dict(obs, actions, old_mean, old_log_std) of the samples that rew
    and fd (feat_diff) belong to.  dual_fns / loss_fns: (f, fprime) replacing the oracle's own (f(x), fprime(x)).
    Returns dict(eta, v, theta, eta_before, LossBefore, LossAfter, DualBefore, DualAfter, MeanKL)."""
    if dual_fns is None:
        dual_fns = (lambda x: dual(x[0], x[1:], rew, fd, epsilon, l2_reg_dual),
                    lambda x: dual_grad(x[0], x[1:], rew, fd, epsilon, l2_reg_dual))
    x0 = np.hstack([eta, v])
    bounds = [(-np.inf, np.inf) for _ in x0]
    bounds[0] = (0., np.inf)
    dual_before = dual_fns[0](x0)
    x, _, _ = _lbfgs(optimizer, func=dual_fns[0], x0=x0, fprime=dual_fns[1], bounds=bounds, maxiter=max_opt_itr, disp=0)
    dual_after = dual_fns[0](x)
    eta_new, v_new = x[0], x[1:]
    if loss_fns is None:
        w = weights(eta_new, v_new, rew, fd)
        loss_fns = (lambda th: policy_loss(th, batch, w, dims, l2_reg_loss, min_std),
                    lambda th: policy_grad(th, batch, w, dims, l2_reg_loss, min_std))
    theta0 = np.array(theta, dtype=np.float64)
    loss_before = loss_fns[0](theta0)
    th, _, _ = _lbfgs(optimizer, func=loss_fns[0], x0=theta0, fprime=loss_fns[1], disp=0, maxiter=max_opt_itr)
    loss_after = loss_fns[0](th)
    mean, log_std = P.forward(th, batch["obs"], dims, min_std)
    old_ls = np.asarray(batch["old_log_std"], dtype=np.float64) * np.ones_like(batch["old_mean"])
    mean_kl = np.mean(P.kl(batch["old_mean"], old_ls, mean, log_std * np.ones_like(mean)))
    return dict(eta=eta_new, v=v_new, theta=th, eta_before=x0[0], LossBefore=loss_before, LossAfter=loss_after,
                DualBefore=dual_before, DualAfter=dual_after, MeanKL=mean_kl)
