"""float64 oracle of CategoricalGRUPolicy over a lane batch (test infrastructure).

The recurrence is tests/gru_oracle.py's (GRULayer.step, the path-start resets, backpropagation through time, the
forward tangent sweep) and the softmax head tests/categorical_oracle.py's (rllab/distributions/categorical.py terms with
TINY = 1e-8, the cancellation-free logit derivatives, the logit Fisher block M), both imported.  The net is
rllab/policies/categorical_gru_policy.py: x_t = [obs_t, one-hot prev_action_t] (state_include_action) or obs_t, logits
z = h' W_out + b_out, prob = softmax(z); h = 0 and prev_action = 0 where a path starts (tstep == 0), otherwise
prev_action is the one-hot act[t-1] of the lane.  Flat layout [W_xr, W_hr, b_r, W_xu, W_hu, b_u, W_xc, W_hc, b_c, W_out,
b_out].  The Fisher-vector product is the Gauss-Newton product J^T M J x (M at theta_old), which leaves out the O(TINY)
first-derivative term of the exact Hessian of mean KL (categorical_oracle.fvp's curvature=False).
"""
import numpy as np

import categorical_oracle as CO
import gru_oracle as GO
from oracle import optim as OPT

TINY = CO.TINY


class CatGruDims(GO.GruDims):
    """GruDims with A = n actions and no log_std."""

    def __init__(self, obs_dim, hidden, n, include_action=True):
        GO.GruDims.__init__(self, obs_dim, hidden, n, include_action)
        self.names, self.shapes = self.names[:-1], self.shapes[:-1]
        self.P = int(sum(int(np.prod(s)) for s in self.shapes))


def init_params(dims, rng):
    """GlorotUniform weights, zero biases."""
    vals = []
    for s in dims.shapes:
        vals.append(rng.uniform(-np.sqrt(6.0 / sum(s)), np.sqrt(6.0 / sum(s)), size=s).reshape(-1) if len(s) == 2
                    else np.zeros(s))
    return np.concatenate(vals)


def forward(flat, lanes, dims):
    """prob (T, N, n), logits (T, N, n) and gru_oracle's per-step cache."""
    z, cache = GO.forward(flat, lanes, dims)
    z = np.moveaxis(z, 0, -1)
    return CO.softmax(z), z, cache


def _flat_batch(lanes, p):
    """categorical_oracle's sample dict over all (t, lane) cells, row order t-major."""
    n = p.shape[-1]
    return dict(actions=np.moveaxis(lanes["act"].astype(np.float64), 0, -1).reshape(-1, n),
                old_prob=np.moveaxis(lanes["old_prob"].astype(np.float64), 0, -1).reshape(-1, n),
                adv=lanes["adv"].astype(np.float64).reshape(-1))


def terms(flat, lanes, dims, kind):
    """Per-sample surrogate term and KL (T, N)."""
    p, _, _ = forward(flat, lanes, dims)
    fb = _flat_batch(lanes, p)
    pf = p.reshape(-1, dims.A)
    if kind == "trpo":
        term = -CO.likelihood_ratio(fb["actions"], fb["old_prob"], pf) * fb["adv"]
    else:
        term = -CO.log_likelihood(fb["actions"], pf) * fb["adv"]
    return term.reshape(p.shape[:2]), CO.kl(fb["old_prob"], pf).reshape(p.shape[:2])


def loss_kl(flat, lanes, dims, kind):
    """(surrogate, mean KL, max KL) over the valid samples (npo.py:67-82 with valids)."""
    term, kl = terms(flat, lanes, dims, kind)
    v = GO.valid_of(lanes)
    return term[v].mean(), kl[v].mean(), kl[v].max()


def grad(flat, lanes, dims, kind, penalty=0.0):
    """Gradient of the surrogate (+ penalty * mean KL) over the valid samples; kind "kl": of mean KL alone."""
    p, _, cache = forward(flat, lanes, dims)
    fb = _flat_batch(lanes, p)
    pf = p.reshape(-1, dims.A)
    if kind == "kl":
        dz = CO._kl_logit_grad(pf, fb["old_prob"])
    else:
        dz = CO.logit_grad(pf, fb, kind, penalty)
    v = GO.valid_of(lanes)
    dz = np.where(v[..., None], dz.reshape(p.shape), 0.0) / v.sum()
    return GO._bptt(flat, dims, cache, dz, np.zeros_like(dz))


def fvp(flat, lanes, dims, xvec, reg_coeff=1e-5):
    """J^T M J x / n_valid + reg x at theta_old: J x the tangent of the logits (gru_oracle.tangent_mean), M the logit
    Fisher block at prob(theta_old) (categorical_oracle.logit_hvp)."""
    p, _, cache = forward(flat, lanes, dims)
    tz = GO.tangent_mean(flat, lanes, dims, xvec)
    m = CO.logit_hvp(p.reshape(-1, dims.A), tz.reshape(-1, dims.A)).reshape(p.shape)
    v = GO.valid_of(lanes)
    dz = np.where(v[..., None], m, 0.0) / v.sum()
    return GO._bptt(flat, dims, cache, dz, np.zeros_like(dz)) + reg_coeff * np.asarray(xvec)


def trpo_step(theta, lanes, dims, step_size=0.01, cg_iters=10, reg_coeff=1e-5):
    f_loss = lambda th: loss_kl(th, lanes, dims, "trpo")[0]
    f_grad = lambda th: grad(th, lanes, dims, "trpo")
    f_lc = lambda th: loss_kl(th, lanes, dims, "trpo")[:2]
    f_Hx = lambda th, x: fvp(th, lanes, dims, x, reg_coeff)
    return OPT.trpo_optimize(f_loss, f_grad, f_lc, f_Hx, theta, step_size, cg_iters)


def entropy_mean(lanes):
    """The sampler's Entropy statistic: mean over the valid samples of entropy(prob) of the recorded probabilities."""
    p = np.moveaxis(np.asarray(lanes["mean"], dtype=np.float64), 0, -1)
    return CO.entropy(p)[GO.valid_of(lanes)].mean()


def rollout_cartpole_v0(theta, dims, N, T, max_path_length, u, reset_raw):
    """Lane rollout of CartPole-v0 with the categorical GRU policy (b200rl_rollout_categorical_gru's semantics:
    auto-reset, h and prev_action reset at every path start, FLAG_DONE / FLAG_END / FLAG_CUT, tstep), float64; u [T][N]
    action uniforms, reset_raw [T+1][4][N].  Returns the lane dict (obs, one-hot act, mean = prob, rew, flags, tstep)."""
    env = CO.CartPoleV0()
    p = GO.unpack(theta, dims)
    n = dims.A
    obs = np.zeros((4, T, N))
    act = np.zeros((n, T, N))
    prob = np.zeros((n, T, N))
    rew = np.zeros((T, N))
    flags = np.zeros((T, N), np.uint8)
    tstep = np.zeros((T, N), np.uint16)
    s = env.reset(reset_raw[0])
    plen = np.zeros(N, dtype=int)
    h = np.zeros((N, dims.H))
    pa = np.zeros((N, n))
    for t in range(T):
        start = plen == 0
        h = np.where(start[:, None], 0.0, h)
        pa = np.where(start[:, None], 0.0, pa)
        x = np.concatenate([s.T, pa], axis=1) if dims.inc else s.T
        h = GO.cell(p, x, h)[0]
        pr = CO.softmax(h @ p["W_out"] + p["b_out"])
        k = CO.weighted_sample_n(pr, u[t])
        obs[:, t], prob[:, t] = s, pr.T
        act[k, t, np.arange(N)] = 1.0
        s, r, done = env.step(s, k)
        rew[t], tstep[t] = r, plen
        plen = plen + 1
        whole = done | (plen >= max_path_length)
        end = whole | (t == T - 1)
        flags[t] = (done * 1 | end * 2 | (end & ~whole) * 4).astype(np.uint8)
        s = np.where(end[None], env.reset(reset_raw[t + 1]), s)
        plen = np.where(end, 0, plen)
        pa = act[:, t].T
    return dict(obs=obs, act=act, mean=prob, rew=rew, flags=flags, tstep=tstep, log_std=np.zeros(1))


def synthetic_lanes(dims, N, T, rng, theta, path_len=(1, 40), masked_frac=0.0):
    """Random lanes recorded at theta: paths of random lengths (restarts mid-lane), obs ~ N(0, s), one-hot actions
    sampled from the policy step by step (prev_action feeds back), old_prob the float64 probabilities, advantages
    ~ N(0, 1); masked_frac of the paths marked invalid (whole paths, like FLAG_MASKED)."""
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
    p = GO.unpack(theta, dims)
    h = np.zeros((N, dims.H))
    prob = np.zeros((dims.A, T, N))
    for t in range(T):
        x, start = GO.inputs(lanes, dims, t)
        h = np.where(start[:, None], 0.0, h)
        h = GO.cell(p, x, h)[0]
        pr = CO.softmax(h @ p["W_out"] + p["b_out"])
        k = CO.weighted_sample_n(pr, rng.rand(N))
        lanes["act"][k, t, np.arange(N)] = 1.0
        prob[:, t] = pr.T
    lanes["old_prob"] = prob.astype(np.float32)
    lanes["adv"] = rng.randn(T, N).astype(np.float32)
    return lanes
