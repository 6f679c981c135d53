"""Oracle: lock-step lane rollout, process_samples (GAE/returns/centering/stats),
LinearFeatureBaseline.  float64 NumPy.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

Restates:
  * rllab/sampler/utils.py:6-43 (rollout: stores the PRE-step obs, the raw action, reward,
    agent_info; stops on done or max_path_length)
  * sandbox/rocky/tf/samplers/vectorized_sampler.py:54-100 +
    sandbox/rocky/tf/envs/vec_env_executor.py:14-26 (lock-step lanes, auto-reset, horizon cut)
  * rllab/sampler/parallel_sampler.py:129-155 (a trailing cut path is still a path: truncate_paths)
  * rllab/sampler/base.py:48-182 (process_samples), rllab/misc/special.py:51-59,107-111,
    rllab/algos/util.py:7-12
  * rllab/baselines/linear_feature_baseline.py:19-43

Lane trajectory layout (identical to the CUDA path; structure-of-arrays, time-major):
  obs (O,T,N)  act (A,T,N)  mean (A,T,N)  rew (T,N)  flags (T,N) uint8  tstep (T,N) uint16
  flags bit0 = env reported done at this step, bit1 = this sample is the last of its path
  (done, or path length == max_path_length, or t == T-1).  tstep = index of the sample in its path.
"""
import numpy as np

from . import policy as P

FLAG_DONE = 1
FLAG_END = 2
FLAG_CUT = 4      # with FLAG_END: the path was cut by the end of the lane buffer (neither done nor max_path_length)
FLAG_MASKED = 8   # device only: set by b200rl_process_samples(drop_cut_paths) on the samples of a dropped path


def rollout_lanes(env, theta, dims, N, T, max_path_length, eps, reset_raw, min_std=1e-6,
                  reset_states=None, policy_dtype=np.float64):
    """eps (T,A,N) N(0,1) action noise; reset_raw (T+1,K,N) raw reset noise: row 0 seeds the initial
    reset, row t+1 the auto-reset that follows a path ending at step t.  `reset_states` (T+1,S,N)
    optionally overrides env.reset(raw) (used to replay reference trajectories exactly)."""
    dt = env.dtype
    O, A = env.O, env.A
    obs = np.zeros((O, T, N), dt)
    act = np.zeros((A, T, N), dt)
    mean = np.zeros((A, T, N), dt)
    rew = np.zeros((T, N), dt)
    flags = np.zeros((T, N), np.uint8)
    tstep = np.zeros((T, N), np.uint16)
    state = env.reset(reset_raw[0]) if reset_states is None else np.array(reset_states[0], dt)
    plen = np.zeros(N, np.int64)
    log_std = None
    for t in range(T):
        o = env.obs(state)
        mu, log_std = P.forward(np.asarray(theta, policy_dtype), o.T.astype(policy_dtype), dims, min_std)
        mu = mu.T.astype(dt)                                    # (A,N)
        a = (mu + np.exp(log_std).astype(dt).reshape(A, 1) * np.asarray(eps[t], dt)).astype(dt)
        u = env.scale_action(a)
        state2, r, done = env.step(state, u)
        obs[:, t], act[:, t], mean[:, t], rew[t] = o, a, mu, r
        tstep[t] = plen
        plen = plen + 1
        whole = done | (plen >= max_path_length)
        end = whole | (t == T - 1)
        flags[t] = done.astype(np.uint8) * FLAG_DONE + end.astype(np.uint8) * FLAG_END + \
            (end & ~whole).astype(np.uint8) * FLAG_CUT
        fresh = env.reset(reset_raw[t + 1]) if reset_states is None else np.array(reset_states[t + 1], dt)
        state = np.where(end[None, :], fresh, state2).astype(dt)
        plen = np.where(end, 0, plen)
    return dict(obs=obs, act=act, mean=mean, rew=rew, flags=flags, tstep=tstep,
                log_std=np.asarray(log_std, dt))


def valid_mask(traj, drop_cut=True):
    """(T, N) bool: samples of whole paths.  A path whose last sample carries FLAG_CUT (cut by the end of the lane
    buffer) is not a whole path: with whole_paths=True the reference's samplers never return it
    (batch_polopt.py:30-34; vectorized_sampler.py drops unfinished running_paths)."""
    fl = np.asarray(traj["flags"])
    T, N = fl.shape
    valid = np.ones((T, N), dtype=bool)
    if not drop_cut:
        return valid
    dropped = np.zeros(N, dtype=bool)
    for t in range(T - 1, -1, -1):
        e = (fl[t] & FLAG_END) != 0
        dropped = np.where(e, (fl[t] & FLAG_CUT) != 0, dropped)
        valid[t] = ~dropped
    return valid


def lanes_to_paths(traj, drop_cut=False):
    """Lane trajectories -> the reference's list-of-path-dicts wire format
    (sampler/utils.py:37-43), lane-major then time order."""
    O, T, N = traj["obs"].shape
    A = traj["act"].shape[0]
    paths = []
    ends = (traj["flags"] & FLAG_END) != 0
    for n in range(N):
        start = 0
        for t in range(T):
            if ends[t, n]:
                sl = slice(start, t + 1)
                L = t + 1 - start
                if drop_cut and (traj["flags"][t, n] & FLAG_CUT):
                    start = t + 1
                    continue
                paths.append(dict(
                    observations=traj["obs"][:, sl, n].T.copy(),
                    actions=traj["act"][:, sl, n].T.copy(),
                    rewards=traj["rew"][sl, n].copy(),
                    agent_infos=dict(mean=traj["mean"][:, sl, n].T.copy(),
                                     log_std=np.tile(traj["log_std"].reshape(1, A), (L, 1))),
                    env_infos=dict(),
                    _lane=n, _t0=start,
                ))
                start = t + 1
    return paths


def lfb_features(obs_path, dtype=np.float64):
    """linear_feature_baseline.py:19-23; obs_path (L,O)."""
    o = np.clip(np.asarray(obs_path, dtype), -10, 10)
    l = o.shape[0]
    al = np.arange(l).reshape(-1, 1) / 100.0
    return np.concatenate([o, o ** 2, al, al ** 2, al ** 3, np.ones((l, 1))], axis=1)


def lfb_features_lanes(obs, tstep):
    """Same features for lane layout: obs (O,T,N), tstep (T,N) -> (d,T,N)."""
    o = np.clip(np.asarray(obs, np.float64), -10, 10)
    al = np.asarray(tstep, np.float64)[None] / 100.0
    return np.concatenate([o, o ** 2, al, al ** 2, al ** 3, np.ones_like(al)], axis=0)


def lfb_fit_normal(AtA, Aty, reg_coeff=1e-5):
    """linear_feature_baseline.py:26-37: lstsq on the regularised normal equations, reg x10 retries."""
    reg = reg_coeff
    coeffs = None
    for _ in range(5):
        coeffs = np.linalg.lstsq(AtA + reg * np.identity(AtA.shape[0]), Aty, rcond=None)[0]
        if not np.any(np.isnan(coeffs)):
            break
        reg *= 10
    return coeffs


def lfb_fit_lanes(obs, tstep, ret, reg_coeff=1e-5, valid=None):
    F = lfb_features_lanes(obs, tstep)
    d = F.shape[0]
    Fm = F.reshape(d, -1)
    y = np.asarray(ret, np.float64).reshape(-1)
    if valid is not None:
        keep = np.asarray(valid).reshape(-1)
        Fm, y = Fm[:, keep], y[keep]
    return lfb_fit_normal(Fm @ Fm.T, Fm @ y, reg_coeff)


def discount_cumsum(x, discount):
    """special.py:107-111: y[t] = x[t] + discount*y[t+1] (scipy lfilter on the reversed signal)."""
    y = np.zeros(len(x), np.float64)
    acc = 0.0
    for t in range(len(x) - 1, -1, -1):
        acc = x[t] + discount * acc
        y[t] = acc
    return y


def explained_variance_1d(ypred, y):
    """special.py:51-59"""
    vary = np.var(y)
    if np.isclose(vary, 0):
        if np.var(ypred) > 0:
            return 0
        else:
            return 1
    return 1 - np.var(y - ypred) / (vary + 1e-8)


def process_samples_lanes(traj, coeffs, discount, gae_lambda, center_adv=True, positive_adv=False, drop_cut=False,
                          base=None):
    """sampler/base.py:48-182 on the lane layout.  `coeffs` = LinearFeatureBaseline weights of the
    previous iteration (None -> zeros, linear_feature_baseline.py:41-42).  Returns dict with
    adv/ret/base (T,N) and the tabular statistics.  drop_cut: whole paths only (see valid_mask): the samples of cut
    paths get adv = 0 and are left out of the centering and of every statistic; `valid` (T,N) is returned.
    `base` (T,N), if given, is the baseline of every sample (any baseline's predict) and `coeffs` is ignored; `und`
    (T,N) is the undiscounted return-to-go."""
    rew = np.asarray(traj["rew"], np.float64)
    T, N = rew.shape
    ends = (traj["flags"] & FLAG_END) != 0
    if base is not None:
        base = np.asarray(base, np.float64)
    elif coeffs is None:
        base = np.zeros((T, N))
    else:
        F = lfb_features_lanes(traj["obs"], traj["tstep"])
        base = np.tensordot(np.asarray(coeffs, np.float64), F, axes=(0, 0))
    adv = np.zeros((T, N))
    ret = np.zeros((T, N))
    und = np.zeros((T, N))            # undiscounted return-to-go (its value at path starts = sum(rewards))
    a_next = np.zeros(N)
    r_next = np.zeros(N)
    u_next = np.zeros(N)
    b_next = np.zeros(N)
    gl = discount * gae_lambda
    for t in range(T - 1, -1, -1):
        e = ends[t]
        a_next = np.where(e, 0.0, a_next)
        r_next = np.where(e, 0.0, r_next)
        u_next = np.where(e, 0.0, u_next)
        b_next = np.where(e, 0.0, b_next)        # path_baselines = append(b, 0)   base.py:58
        delta = rew[t] + discount * b_next - base[t]
        a_next = delta + gl * a_next
        r_next = rew[t] + discount * r_next
        u_next = rew[t] + u_next
        adv[t], ret[t], und[t] = a_next, r_next, u_next
        b_next = base[t]
    valid = valid_mask(traj, drop_cut)
    starts = (np.asarray(traj["tstep"]) == 0) & valid
    ev = explained_variance_1d(base[valid], ret[valid])
    adv_mean, adv_std = np.mean(adv[valid]), np.std(adv[valid])
    adv_v = adv[valid]
    if center_adv:
        adv_v = (adv_v - np.mean(adv_v)) / (adv_v.std() + 1e-8)             # algos/util.py:7-8
    if positive_adv:
        adv_v = (adv_v - np.min(adv_v)) + 1e-8                              # algos/util.py:11-12
    adv_out = np.zeros_like(adv)
    adv_out[valid] = adv_v
    adv = np.where(valid, adv, 0.0)
    undisc = und[starts]
    ent = float(P.entropy(np.asarray(traj["log_std"], np.float64)))
    stats = dict(
        AverageDiscountedReturn=float(np.mean(ret[starts])),
        AverageReturn=float(np.mean(undisc)),
        ExplainedVariance=float(ev),
        NumTrajs=int(starts.sum()),
        Entropy=ent,
        Perplexity=float(np.exp(ent)),
        StdReturn=float(np.std(undisc)),
        MaxReturn=float(np.max(undisc)),
        MinReturn=float(np.min(undisc)),
        adv_mean=float(adv_mean), adv_std=float(adv_std),
    )
    return dict(adv=adv_out, adv_raw=adv, ret=ret, und=und, base=base, stats=stats, valid=valid)


def truncate_paths_lengths(lengths, max_samples):
    """parallel_sampler.py:129-155 on path lengths only (the integer part that
    tests/test_sampler.py:4-32 pins): drop paths from the end while doing so keeps at least
    max_samples, then cut the last one so that the total is exactly max_samples."""
    lengths = list(lengths)
    total = sum(lengths)
    while len(lengths) > 0 and total - lengths[-1] >= max_samples:
        total -= lengths.pop(-1)
    if len(lengths) > 0:
        last = lengths.pop(-1)
        truncated_len = last - (total - max_samples)
        lengths.append(min(last, truncated_len))     # v[:truncated_len] cannot grow the path
    return lengths


def batch_from_traj(traj, adv, valid=None):
    """Flatten the lane layout to the (B, .) sample-major layout the oracle losses take; `valid` (T,N) bool keeps the
    samples of whole paths only."""
    O = traj["obs"].shape[0]
    A = traj["act"].shape[0]
    keep = slice(None) if valid is None else np.asarray(valid).reshape(-1)
    return dict(
        obs=np.asarray(traj["obs"], np.float64).reshape(O, -1).T[keep],
        actions=np.asarray(traj["act"], np.float64).reshape(A, -1).T[keep],
        adv=np.asarray(adv, np.float64).reshape(-1)[keep],
        old_mean=np.asarray(traj["mean"], np.float64).reshape(A, -1).T[keep],
        old_log_std=np.asarray(traj["log_std"], np.float64).reshape(A),
    )
