"""float64 oracle of CategoricalMLPPolicy and gym CartPole-v0 (test infrastructure, as tests/ppo_oracle.py).

Restates rllab/policies/categorical_mlp_policy.py (tanh MLP, softmax output), rllab/distributions/categorical.py (kl,
log_likelihood, likelihood ratio, entropy; TINY = 1e-8), rllab/misc/special.py:weighted_sample_n, the NPO / VPG
surrogates over it, their gradients, and the Fisher-vector product J^T M J x at theta_old (DESIGN.md section 5), and
gym 0.7.4's CartPole-v0 dynamics.  Flat layout [W0, b0, W1, b1, Wout, bout].
"""
import numpy as np

from oracle import optim as OPT

TINY = 1e-8


class CatDims(object):
    def __init__(self, obs_dim, hidden_sizes, n):
        self.O, self.H, self.A = int(obs_dim), tuple(int(h) for h in hidden_sizes), int(n)
        sizes = (self.O,) + self.H + (self.A,)
        self.shapes = []
        for i in range(len(sizes) - 1):
            self.shapes += [(sizes[i], sizes[i + 1]), (sizes[i + 1],)]
        self.P = int(sum(int(np.prod(s)) for s in self.shapes))


def unpack(flat, dims):
    out, k = [], 0
    for s in dims.shapes:
        n = int(np.prod(s))
        out.append(np.asarray(flat[k:k + n], dtype=np.float64).reshape(s))
        k += n
    return out


def init_params(dims, rng):
    ts = []
    for s in dims.shapes:
        if len(s) == 2:
            a = np.sqrt(6.0 / (s[0] + s[1]))
            ts.append(rng.uniform(-a, a, size=s).reshape(-1))
        else:
            ts.append(np.zeros(s))
    return np.concatenate(ts)


def softmax(z):
    e = np.exp(z - np.max(z, axis=-1, keepdims=True))
    return e / np.sum(e, axis=-1, keepdims=True)


def forward(flat, obs, dims):
    """(logits (B,n), activations [x, h1, h2])"""
    ts = unpack(flat, dims)
    h = np.asarray(obs, dtype=np.float64)
    acts = [h]
    nl = len(dims.H)
    for i in range(nl):
        h = np.tanh(h @ ts[2 * i] + ts[2 * i + 1])
        acts.append(h)
    return h @ ts[2 * nl] + ts[2 * nl + 1], acts


def prob(flat, obs, dims):
    return softmax(forward(flat, obs, dims)[0])


def saturated_params(dims, gap, rng, sign=1.0):
    """theta (n = 2) whose logit gap z0 - z1 lies within gap +- 0.25 at every input (sign -1: z1 - z0): Wout scaled so
    that |h2 (Wout[:, 0] - Wout[:, 1])| <= 0.25 for any |h2| <= 1, bout = +-gap / 2; non-zero hidden biases."""
    assert dims.A == 2
    ts = unpack(init_params(dims, rng) + 0.05 * rng.randn(dims.P), dims)
    ts[-2] *= 0.25 / np.abs(ts[-2][:, 0] - ts[-2][:, 1]).sum()
    ts[-1] = sign * 0.5 * gap * np.array([1.0, -1.0])
    return np.concatenate([t.reshape(-1) for t in ts])


def weighted_sample_n(p, u):
    """special.weighted_sample_n with the uniforms given: #{k : cumsum_k(p) < u}, clipped to n - 1."""
    k = (np.cumsum(p, axis=1) < np.asarray(u).reshape(-1, 1)).sum(axis=1)
    return np.minimum(k, p.shape[1] - 1)


def kl(old_p, new_p):
    return np.sum(old_p * (np.log(old_p + TINY) - np.log(new_p + TINY)), axis=-1)


def log_likelihood(x_onehot, p):
    return np.log(np.sum(p * x_onehot, axis=-1) + TINY)


def likelihood_ratio(x_onehot, old_p, new_p):
    return (np.sum(new_p * x_onehot, axis=-1) + TINY) / (np.sum(old_p * x_onehot, axis=-1) + TINY)


def entropy(p):
    return -np.sum(p * np.log(p + TINY), axis=-1)


# batch = dict(obs (B,O), actions (B,n) one-hot, adv (B,), old_prob (B,n))
def surr_loss(flat, batch, dims, kind):
    p = prob(flat, batch["obs"], dims)
    if kind == "trpo":
        return -np.mean(likelihood_ratio(batch["actions"], batch["old_prob"], p) * batch["adv"])
    return -np.mean(log_likelihood(batch["actions"], p) * batch["adv"])


def kl_stats(flat, batch, dims):
    k = kl(batch["old_prob"], prob(flat, batch["obs"], dims))
    return np.mean(k), np.max(k)


def _backward(flat, dims, acts, dz):
    ts = unpack(flat, dims)
    nl = len(dims.H)
    grads = [None] * len(ts)
    delta = dz
    grads[2 * nl] = acts[nl].T @ delta
    grads[2 * nl + 1] = delta.sum(axis=0)
    for i in range(nl - 1, -1, -1):
        delta = (delta @ ts[2 * (i + 1)].T) * (1.0 - np.square(acts[i + 1]))
        grads[2 * i] = acts[i].T @ delta
        grads[2 * i + 1] = delta.sum(axis=0)
    return np.concatenate([g.reshape(-1) for g in grads])


# The logit-space terms below are written without differences of nearly equal numbers, so that they stay exact when
# one probability is near 1 (a confident policy).  Softmax is shift-invariant, so wherever the textbook form has
# 1 - p_a or y_k - sum_j p_j y_j, it is computed as sum_j p_j (y_k - y_j): each p_j is accurate to rounding relative to
# itself, and the terms of the sum are exact differences of the y's.  (The direct forms lose all accuracy in float64
# once the smaller probability falls below ~1e-16 of the larger, a logit gap of ~37.)
def _centered(p, y):
    """y_k - sum_j p_j y_j as sum_j p_j (y_k - y_j), (B, n)."""
    return np.einsum("bj,bkj->bk", p, y[:, :, None] - y[:, None, :])


def _kl_logit_grad(p, q):
    """d kl(q || softmax(z)) / dz_k = -r_k + p_k sum_j r_j, r = q p / (p + TINY), as sum_j (p_k r_j - r_k p_j)."""
    r = q * p / (p + TINY)
    return np.sum(p[:, :, None] * r[:, None, :] - r[:, :, None] * p[:, None, :], axis=2)


def logit_grad(p, batch, kind, penalty=0.0):
    """d (surrogate term + penalty kl) / dz per sample (B, n): -c p_k (x_k - pa) with x_k - pa = sum_j p_j (x_k - x_j)."""
    x, q, adv = batch["actions"], batch["old_prob"], batch["adv"]
    pa = np.sum(p * x, axis=-1)
    c = adv / (np.sum(q * x, axis=-1) + TINY) if kind == "trpo" else adv / (pa + TINY)
    dz = -c[:, None] * p * _centered(p, x)
    if penalty:
        dz = dz + penalty * _kl_logit_grad(p, q)
    return dz


def grad_surr(flat, batch, dims, kind, penalty=0.0):
    """Flat gradient of the surrogate + penalty * mean KL(old || new) (the objective of PPO's penalised step)."""
    z, acts = forward(flat, batch["obs"], dims)
    dz = logit_grad(softmax(z), batch, kind, penalty)
    return _backward(flat, dims, acts, dz / dz.shape[0])


def grad_kl(flat, batch, dims):
    """Flat gradient of mean KL(old || new) (FiniteDifferenceHvp's gradient, b200rl_categorical_update_f64's LOSS_KL)."""
    z, acts = forward(flat, batch["obs"], dims)
    g = _kl_logit_grad(softmax(z), batch["old_prob"])
    return _backward(flat, dims, acts, g / g.shape[0])


def _hessian_terms(p):
    pe = p + TINY
    R = np.sum(p * p / pe, axis=-1)
    s = TINY * p * p / (pe * pe)
    return R, s


def logit_hessian(p):
    """Hessian in z of kl(q || softmax(z)) at q = softmax(z), TINY kept (B, n, n):
    M = diag(R p - s) + s p^T + p s^T - (R + S) p p^T.  Its rows sum to zero (shift invariance), so the diagonal is
    minus the sum of the off-diagonal entries, which have no cancellation."""
    R, s = _hessian_terms(p)
    S = s.sum(axis=-1)
    M = s[:, :, None] * p[:, None, :] + p[:, :, None] * s[:, None, :]
    M -= (R + S)[:, None, None] * p[:, :, None] * p[:, None, :]
    n = p.shape[1]
    M[:, np.arange(n), np.arange(n)] = 0.0
    M[:, np.arange(n), np.arange(n)] = -M.sum(axis=2)
    return M


def logit_hvp(p, tz):
    """M tz per sample (B, n) as (R p_k - s_k) u_k + p_k sum_j s_j u_j, u = tz - p.tz = sum_j p_j (tz_k - tz_j)."""
    R, s = _hessian_terms(p)
    u = _centered(p, tz)
    return (R[:, None] * p - s) * u + p * np.sum(s * u, axis=-1, keepdims=True)


def fvp(flat, batch, x, dims, reg_coeff=1e-5, curvature=True):
    """Hx = grad(grad(mean KL) . x) + reg * x at theta_old (PerlmutterHvp, conjugate_gradient_optimizer.py:22-55), exact
    in float64: J^T M J x / B plus sum_j g_j (d^2 z_j)[x] / B, g = d kl / dz (O(TINY) at theta_old, DESIGN.md section 5),
    the second term as the tangent along x of the backward pass of g.  curvature=False leaves the second term out: the
    Gauss-Newton product J^T M J x / B of the float32 pass (b200rl_categorical_fvp)."""
    ts, xs = unpack(flat, dims), unpack(x, dims)
    assert len(dims.H) == 2
    W0, b0, W1, b1, Wo, bo = ts
    V0, c0, V1, c1, Vo, co = xs
    z, (X, h1, h2) = forward(flat, batch["obs"], dims)
    p = softmax(z)
    B = p.shape[0]
    d1h, d2h = 1.0 - h1 * h1, 1.0 - h2 * h2
    t1 = d1h * (X @ V0 + c0)
    t2 = d2h * (t1 @ W1 + h1 @ V1 + c1)
    tz = t2 @ Wo + h2 @ Vo + co
    dz = logit_hvp(p, tz)
    g = _kl_logit_grad(p, p) if curvature else np.zeros_like(p)
    d2g = (g @ Wo.T) * d2h
    D2 = (dz @ Wo.T) * d2h + (g @ Vo.T) * d2h - 2.0 * (g @ Wo.T) * h2 * t2
    D1 = (D2 @ W1.T + d2g @ V1.T) * d1h - 2.0 * (d2g @ W1.T) * h1 * t1
    out = [X.T @ D1, D1.sum(0), h1.T @ D2 + t1.T @ d2g, D2.sum(0), h2.T @ dz + t2.T @ g, dz.sum(0)]
    return np.concatenate([o.reshape(-1) for o in out]) / B + reg_coeff * np.asarray(x)


def trpo_step(theta, batch, dims, step_size=0.01, cg_iters=10, reg_coeff=1e-5, curvature=True):
    """One TRPO step; curvature=False solves with the Gauss-Newton product of the float32 pass (see fvp)."""
    f_loss = lambda th: surr_loss(th, batch, dims, "trpo")
    f_grad = lambda th: grad_surr(th, batch, dims, "trpo")
    f_lc = lambda th: (surr_loss(th, batch, dims, "trpo"), kl_stats(th, batch, dims)[0])
    f_Hx = lambda th, v: fvp(th, batch, v, dims, reg_coeff, curvature)
    return OPT.trpo_optimize(f_loss, f_grad, f_lc, f_Hx, theta, step_size, cg_iters)


def rollout_cartpole_v0(theta, dims, N, T, max_path_length, u, reset_raw):
    """Lane rollout of CartPole-v0 with the categorical policy (b200rl_rollout_categorical's semantics: auto-reset,
    FLAG_DONE / FLAG_END / FLAG_CUT, tstep), float64; u [T][N] action uniforms, reset_raw [T+1][4][N].  Returns the lane
    dict of oracle/sampler.py (obs [4][T][N], act one-hot [2][T][N], mean = prob [2][T][N], rew, flags, tstep)."""
    env = CartPoleV0()
    obs = np.zeros((4, T, N))
    act = np.zeros((2, T, N))
    prob = np.zeros((2, T, N))
    rew = np.zeros((T, N))
    flags = np.zeros((T, N), np.uint8)
    tstep = np.zeros((T, N), np.uint16)
    s = env.reset(reset_raw[0])
    plen = np.zeros(N, dtype=int)
    for t in range(T):
        p = softmax(forward(theta, s.T, dims)[0])
        k = weighted_sample_n(p, u[t])
        obs[:, t], prob[:, t] = s, p.T
        act[k, t, np.arange(N)] = 1.0
        s, r, done = env.step(s, k)
        rew[t], tstep[t] = r, plen
        plen += 1
        whole = done | (plen >= max_path_length)
        end = whole | (t == T - 1)
        flags[t] = (done * 1 | end * 2 | (end & ~whole) * 4).astype(np.uint8)
        s = np.where(end[None], env.reset(reset_raw[t + 1]), s)
        plen = np.where(end, 0, plen)
    return dict(obs=obs, act=act, mean=prob, rew=rew, flags=flags, tstep=tstep, log_std=np.zeros(1))


# ---------------------------------------------------------------- gym 0.7.4 CartPole-v0
class CartPoleV0(object):
    O, A, S, K = 4, 1, 4, 4
    THR = 12 * 2 * np.pi / 360

    def __init__(self, dtype=np.float64):
        self.dt = dtype

    def reset(self, raw):
        raw = np.asarray(raw, dtype=self.dt)
        return self.dt(-0.05) + self.dt(0.1) * raw

    def step(self, s, action):
        """s (4,) or (4, N); action index (or array of them); returns (s', reward, done)."""
        dt = self.dt
        x, xd, th, thd = (np.asarray(v, dtype=dt) for v in s)
        force = np.where(np.asarray(action) == 1, dt(10.0), dt(-10.0))
        g, mp, total, l, pml, tau = dt(9.8), dt(0.1), dt(1.1), dt(0.5), dt(0.05), dt(0.02)
        cs, sn = np.cos(th), np.sin(th)
        temp = (force + pml * thd * thd * sn) / total
        thacc = (g * sn - cs * temp) / (l * (dt(4.0) / dt(3.0) - mp * cs * cs / total))
        xacc = temp - pml * thacc * cs / total
        ns = np.stack([x + tau * xd, xd + tau * xacc, th + tau * thd, thd + tau * thacc])
        done = (ns[0] < -2.4) | (ns[0] > 2.4) | (ns[2] < -self.THR) | (ns[2] > self.THR)
        return ns, np.ones_like(ns[0]), done
