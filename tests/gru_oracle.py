"""float64 oracle of GaussianGRUPolicy over a lane batch (test infrastructure, as tests/categorical_oracle.py).

Restates rllab/core/network.py GRULayer.step (r, u sigmoid gates, tanh candidate, h' = (1 - u) h + u c), GRUNetwork's
linear mean head, the recurrent dist_info_sym of rllab/policies/gaussian_gru_policy.py (x_t = [obs_t, prev_action_t]),
and the NPO / VPG surrogates and mean / max KL with valids (npo.py:67-82, vpg.py:66-90) over it.  Lanes are time-major
planes [dim][T][N] with tstep; a path starts where tstep == 0: h = 0 and prev_action = 0 there, otherwise prev_action is
act[t-1] of the lane.  Gradients by backpropagation through time, the Fisher-vector product J^T M J x by a forward
tangent sweep, and a TRPO step.  Flat layout [W_xr, W_hr, b_r, W_xu, W_hu, b_u, W_xc, W_hc, b_c, W_out, b_out, log_std].
"""
import numpy as np

from oracle import envs as E
from oracle import optim as OPT

EPS = 1e-8


class GruDims(object):
    def __init__(self, obs_dim, hidden, act_dim, include_action=True):
        self.O, self.H, self.A, self.inc = int(obs_dim), int(hidden), int(act_dim), bool(include_action)
        self.I = self.O + (self.A if self.inc else 0)
        I, H, A = self.I, self.H, self.A
        self.names = ["W_xr", "W_hr", "b_r", "W_xu", "W_hu", "b_u", "W_xc", "W_hc", "b_c", "W_out", "b_out", "log_std"]
        self.shapes = [(I, H), (H, H), (H,)] * 3 + [(H, A), (A,), (A,)]
        self.P = int(sum(int(np.prod(s)) for s in self.shapes))


def unpack(flat, dims):
    out, k = {}, 0
    for name, s in zip(dims.names, dims.shapes):
        n = int(np.prod(s))
        out[name] = np.asarray(flat[k:k + n], dtype=np.float64).reshape(s)
        k += n
    return out


def pack(d, dims):
    return np.concatenate([np.asarray(d[name], dtype=np.float64).reshape(-1) for name in dims.names])


def init_params(dims, rng, init_std=1.0):
    vals = []
    for s in dims.shapes[:-1]:
        if len(s) == 2:
            a = np.sqrt(6.0 / (s[0] + s[1]))
            vals.append(rng.uniform(-a, a, size=s).reshape(-1))
        else:
            vals.append(np.zeros(s))
    vals.append(np.full((dims.A,), np.log(init_std)))
    return np.concatenate(vals)


def sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def cell(p, x, h):
    """One GRU step for rows x (n, I), h (n, H) -> (h', r, u, c, hc)."""
    r = sigmoid(x @ p["W_xr"] + h @ p["W_hr"] + p["b_r"])
    u = sigmoid(x @ p["W_xu"] + h @ p["W_hu"] + p["b_u"])
    hc = h @ p["W_hc"]
    c = np.tanh(x @ p["W_xc"] + r * hc + p["b_c"])
    return (1.0 - u) * h + u * c, r, u, c, hc


def inputs(lanes, dims, t):
    """x_t (N, I) and the path-start mask of step t."""
    start = lanes["tstep"][t] == 0
    x = lanes["obs"][:, t].T.astype(np.float64)
    if dims.inc:
        pa = np.zeros((x.shape[0], dims.A)) if t == 0 else lanes["act"][:, t - 1].T.astype(np.float64)
        pa = np.where(start[:, None], 0.0, pa)
        x = np.concatenate([x, pa], axis=1)
    return x, start


def forward(flat, lanes, dims):
    """mean [A][T][N] and the per-step cache (x, h_prev, r, u, c, hc, h_new)."""
    p = unpack(flat, dims)
    T, N = lanes["tstep"].shape
    h = np.zeros((N, dims.H))
    mean = np.zeros((dims.A, T, N))
    cache = []
    for t in range(T):
        x, start = inputs(lanes, dims, t)
        h = np.where(start[:, None], 0.0, h)
        hn, r, u, c, hc = cell(p, x, h)
        mean[:, t] = (hn @ p["W_out"] + p["b_out"]).T
        cache.append((x, h, r, u, c, hc, hn, start))
        h = hn
    return mean, cache


def valid_of(lanes):
    return lanes.get("valid", np.ones(lanes["tstep"].shape, dtype=bool))


def _terms(flat, lanes, dims, kind, penalty=0.0):
    """Per-sample (term, kl, dmu, dls) (dmu, dls [T][N][A]) and the mean (A, T, N)."""
    p = unpack(flat, dims)
    mean, cache = forward(flat, lanes, dims)
    ls, ls_old = p["log_std"], np.asarray(lanes["old_log_std"], dtype=np.float64)
    mu = np.moveaxis(mean, 0, -1)
    act = np.moveaxis(lanes["act"].astype(np.float64), 0, -1)
    om = np.moveaxis(lanes["old_mean"].astype(np.float64), 0, -1)
    var, var_old = np.exp(2 * ls), np.exp(2 * ls_old)
    var2 = 2 * var + EPS
    z = (act - mu) / np.exp(ls)
    zo = (act - om) / np.exp(ls_old)
    logp = -ls.sum() - 0.5 * np.sum(z * z, -1) - 0.5 * dims.A * np.log(2 * np.pi)
    logp_old = -ls_old.sum() - 0.5 * np.sum(zo * zo, -1) - 0.5 * dims.A * np.log(2 * np.pi)
    dm = om - mu
    num = dm * dm + var_old - var
    kl = np.sum(num / var2 + ls - ls_old, -1)
    adv = lanes["adv"].astype(np.float64)
    if kind == "trpo":
        w = np.exp(logp - logp_old) * adv
        term = -w
    elif kind == "vpg":
        w = adv
        term = -logp * adv
    else:                                     # "kl": the gradient of mean KL alone (FiniteDifferenceHvp)
        w = np.zeros_like(adv)
        term = np.zeros_like(adv)
        penalty = 1.0
    dmu = -w[..., None] * z / np.exp(ls)
    dls = -w[..., None] * (z * z - 1.0)
    if penalty:
        dmu = dmu + penalty * (-2.0 * dm / var2)
        dls = dls + penalty * (1.0 - 2.0 * var * (var2 + 2.0 * num) / (var2 * var2))
    return term, kl, dmu, dls, cache


def loss_kl(flat, lanes, dims, kind):
    """(surrogate, mean KL, max KL) over the valid samples (npo.py:67-82)."""
    term, kl, _, _, _ = _terms(flat, lanes, dims, kind)
    v = valid_of(lanes)
    return term[v].mean(), kl[v].mean(), kl[v].max()


def _bptt(flat, dims, cache, dmu, dls):
    """Flat gradient from per-sample output deltas dmu [T][N][A] (already masked and scaled) and dls [T][N][A]."""
    p = unpack(flat, dims)
    g = {k: np.zeros_like(v) for k, v in p.items()}
    N = dmu.shape[1]
    carry = np.zeros((N, dims.H))
    for t in range(len(cache) - 1, -1, -1):
        x, h, r, u, c, hc, hn, start = cache[t]
        g["W_out"] += hn.T @ dmu[t]
        g["b_out"] += dmu[t].sum(0)
        dh = carry + dmu[t] @ p["W_out"].T
        du = dh * (c - h) * u * (1 - u)
        dc = dh * u * (1 - c * c)
        dhc = dc * r
        dr = dc * hc * r * (1 - r)
        for gate, d, dwh in (("r", dr, dr), ("u", du, du), ("c", dc, dhc)):
            g["W_x" + gate] += x.T @ d
            g["W_h" + gate] += h.T @ dwh
            g["b_" + gate] += d.sum(0)
        dprev = dh * (1 - u) + dr @ p["W_hr"].T + du @ p["W_hu"].T + dhc @ p["W_hc"].T
        carry = np.where(start[:, None], 0.0, dprev)      # the path ends here going backwards
    g["log_std"] = dls.reshape(-1, dims.A).sum(0)
    return pack(g, dims)


def grad(flat, lanes, dims, kind, penalty=0.0):
    """Gradient of the surrogate (+ penalty * mean KL); kind "kl": gradient of mean KL."""
    _, _, dmu, dls, cache = _terms(flat, lanes, dims, kind, penalty)
    v = valid_of(lanes)
    n = v.sum()
    dmu = np.where(v[..., None], dmu, 0.0) / n
    dls = np.where(v[..., None], dls, 0.0) / n
    return _bptt(flat, dims, cache, dmu, dls)


def tangent_mean(flat, lanes, dims, xvec):
    """J x: the directional derivative of the mean along xvec, [T][N][A]."""
    p, v = unpack(flat, dims), unpack(xvec, dims)
    T, N = lanes["tstep"].shape
    h = np.zeros((N, dims.H))
    th = np.zeros((N, dims.H))
    out = np.zeros((T, N, dims.A))
    for t in range(T):
        x, start = inputs(lanes, dims, t)
        h = np.where(start[:, None], 0.0, h)
        th = np.where(start[:, None], 0.0, th)
        hn, r, u, c, hc = cell(p, x, h)
        tr = r * (1 - r) * (x @ v["W_xr"] + h @ v["W_hr"] + v["b_r"] + th @ p["W_hr"])
        tu = u * (1 - u) * (x @ v["W_xu"] + h @ v["W_hu"] + v["b_u"] + th @ p["W_hu"])
        thc = h @ v["W_hc"] + th @ p["W_hc"]
        tc = (1 - c * c) * (x @ v["W_xc"] + v["b_c"] + tr * hc + r * thc)
        tn = (1 - u) * th + tu * (c - h) + u * tc
        out[t] = tn @ p["W_out"] + hn @ v["W_out"] + v["b_out"]
        h, th = hn, tn
    return out


def fvp(flat, lanes, dims, xvec, reg_coeff=1e-5):
    """Hx = grad(grad(mean KL) . x) + reg x at theta_old = J^T M J x / n_valid + the log_std block (exact there: the
    KL's derivative in the mean is zero at theta_old and log_std enters linearly)."""
    p = unpack(flat, dims)
    v = valid_of(lanes)
    n = v.sum()
    s = np.exp(2 * p["log_std"])
    M_mu = 2.0 / (2.0 * s + EPS)
    M_l = 4.0 * s * (2.0 * s - EPS) / np.square(2.0 * s + EPS)
    _, cache = forward(flat, lanes, dims)
    dmu = np.where(v[..., None], tangent_mean(flat, lanes, dims, xvec) * M_mu, 0.0) / n
    out = _bptt(flat, dims, cache, dmu, np.zeros_like(dmu))
    out[-dims.A:] += M_l * unpack(xvec, dims)["log_std"]
    return out + reg_coeff * np.asarray(xvec)


def trpo_step(theta, lanes, dims, step_size=0.01, cg_iters=10, reg_coeff=1e-5):
    f_loss = lambda th: loss_kl(th, lanes, dims, "trpo")[0]
    f_grad = lambda th: grad(th, lanes, dims, "trpo")
    f_lc = lambda th: loss_kl(th, lanes, dims, "trpo")[:2]
    f_Hx = lambda th, x: fvp(th, lanes, dims, x, reg_coeff)
    return OPT.trpo_optimize(f_loss, f_grad, f_lc, f_Hx, theta, step_size, cg_iters)


def rollout_cartpole(theta, dims, N, T, max_path_length, eps, reset_raw, dtype=np.float64):
    """Lane rollout of normalize(CartpoleEnv()) with the GRU policy (b200rl_rollout_gru's semantics: auto-reset, h and
    prev_action reset at every path start, FLAG_DONE / FLAG_END / FLAG_CUT, tstep).  eps [T][A][N], reset_raw
    [T+1][4][N].  Returns the lane dict of oracle/sampler.py."""
    env = E.make("cartpole", dtype)
    p = unpack(theta, dims)
    A = dims.A
    obs = np.zeros((4, T, N))
    act = np.zeros((A, T, N))
    mean = np.zeros((A, T, N))
    rew = np.zeros((T, N))
    flags = np.zeros((T, N), np.uint8)
    tstep = np.zeros((T, N), np.uint16)
    s = env.reset(reset_raw[0])
    plen = np.zeros(N, dtype=int)
    h = np.zeros((N, dims.H))
    pa = np.zeros((N, A))
    std = np.exp(p["log_std"])
    for t in range(T):
        start = plen == 0
        h = np.where(start[:, None], 0.0, h)
        pa = np.where(start[:, None], 0.0, pa)
        o = env.obs(s).astype(np.float64)
        x = np.concatenate([o.T, pa], axis=1) if dims.inc else o.T
        h, _, _, _, _ = cell(p, x, h)
        mu = h @ p["W_out"] + p["b_out"]
        a = mu + std * np.asarray(eps[t], dtype=np.float64).T
        obs[:, t], act[:, t], mean[:, t] = o, a.T, mu.T
        s2, r, done = env.step(s, env.scale_action(a.T.astype(dtype)))
        rew[t], tstep[t] = r, plen
        plen = plen + 1
        whole = done | (plen >= max_path_length)
        end = whole | (t == T - 1)
        flags[t] = (done * 1 | end * 2 | (end & ~whole) * 4).astype(np.uint8)
        s = np.where(end[None], env.reset(reset_raw[t + 1]), s2).astype(dtype)
        plen = np.where(end, 0, plen)
        pa = a
    return dict(obs=obs, act=act, mean=mean, rew=rew, flags=flags, tstep=tstep, log_std=p["log_std"].copy())


def synthetic_lanes(dims, N, T, rng, theta, path_len=(1, 40), masked_frac=0.0):
    """Random lanes recorded at theta: paths of random lengths (restarts mid-lane), obs ~ N(0, s), actions sampled from
    the policy, advantages ~ N(0, 1); masked_frac of the paths marked invalid (whole paths, like FLAG_MASKED)."""
    tstep = np.zeros((T, N), np.uint16)
    valid = np.ones((T, N), dtype=bool)
    for n in range(N):
        t = 0
        while t < T:
            L = rng.randint(path_len[0], path_len[1] + 1)
            tstep[t:t + L, n] = np.arange(min(L, T - t))
            if rng.rand() < masked_frac:
                valid[t:t + L, n] = False
            t += L
    obs = (rng.randn(dims.O, T, N) * np.array([1.0, 1.5, 0.2, 1.5])[:dims.O, None, None]).astype(np.float32)
    lanes = dict(obs=obs, tstep=tstep, act=np.zeros((dims.A, T, N), np.float32), valid=valid)
    # actions drawn step by step at theta (prev_action feeds back into the input)
    p = unpack(theta, dims)
    h = np.zeros((N, dims.H))
    mean = np.zeros((dims.A, T, N), np.float32)
    for t in range(T):
        x, start = inputs(lanes, dims, t)
        h = np.where(start[:, None], 0.0, h)
        h, _, _, _, _ = cell(p, x, h)
        mu = h @ p["W_out"] + p["b_out"]
        lanes["act"][:, t] = (mu + np.exp(p["log_std"]) * rng.randn(N, dims.A)).T
        mean[:, t] = mu.T
    lanes["old_mean"] = mean
    lanes["old_log_std"] = p["log_std"].astype(np.float32)
    lanes["adv"] = rng.randn(T, N).astype(np.float32)
    return lanes
