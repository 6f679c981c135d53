"""Float64 NumPy oracle of the DDPG kernels (rllab_b200/csrc/ddpg.cu): the networks of DeterministicMLPPolicy and
ContinuousMLPQFunction with a manual backward pass, DDPG.do_training (ddpg.py:331-365 with lasagne.updates.adam), the
SimpleReplayPool draws (ddpg.py:54-70) from the Philox layout of include/b200rl.h, OU / Gaussian exploration, and one
step of the train() loop (ddpg.py:216-251).  The env is passed in as callables so that the GPU tests can feed the
oracle the device's own float32 transitions.  TEST INFRASTRUCTURE ONLY.

A run's state is a dict: nets [4][P] (theta, Adam m, Adam v, target; [policy | qf] each), env_state, obs, ou, path_return,
path_length, terminal (0 / 1 / 2 as b200rl_ddpg_state), itr, adam_t, pool (obs, act, rew, term, float32 as on the device),
top, bottom, size.
"""
import numpy as np

from oracle.philox import philox4x32_10

H, BATCH = 32, 32
B1, B2, EPS = 0.9, 0.999, 1e-8
STREAM_RESET, STREAM_EXPLORE, STREAM_INDEX = 1, 3, 4


class Dims(object):
    def __init__(self, O, A):
        self.O, self.A = O, A
        self.pshapes = [(O, H), (H,), (H, H), (H,), (H, A), (A,)]
        self.qshapes = [(O, H), (H,), (H + A, H), (H,), (H, 1), (1,)]
        self.PP = sum(int(np.prod(s)) for s in self.pshapes)
        self.QP = sum(int(np.prod(s)) for s in self.qshapes)
        self.P = self.PP + self.QP

    @staticmethod
    def split(flat, shapes):
        out, k = [], 0
        for s in shapes:
            n = int(np.prod(s))
            out.append(flat[k:k + n].reshape(s))
            k += n
        return out

    def weight_mask(self):
        m = []
        for s in self.pshapes + self.qshapes:
            m.append(np.full(int(np.prod(s)), len(s) == 2))
        return np.concatenate(m)


def he_uniform(rng, shape):
    """lasagne 0.2 HeUniform (gain 1): U(+-sqrt(3 / fan_in)), fan_in = rows of W."""
    a = np.sqrt(3.0 / shape[0])
    return rng.uniform(-a, a, size=shape)


def init_params(shapes, rng):
    """HeUniform hidden weights, zero hidden biases, Uniform(-3e-3, 3e-3) output W and b."""
    vals = []
    for i, s in enumerate(shapes):
        if i >= len(shapes) - 2:
            vals.append(rng.uniform(-3e-3, 3e-3, size=s).reshape(-1))
        elif len(s) == 2:
            vals.append(he_uniform(rng, s).reshape(-1))
        else:
            vals.append(np.zeros(s))
    return np.concatenate(vals)


def relu(x):
    return np.maximum(x, 0.0)


def pi_forward(d, theta_p, obs):
    W0, b0, W1, b1, W2, b2 = Dims.split(theta_p, d.pshapes)
    a1 = relu(obs @ W0 + b0)
    a2 = relu(a1 @ W1 + b1)
    return a1, a2, np.tanh(a2 @ W2 + b2)


def q_forward(d, theta_q, obs, act):
    W0, b0, W1, b1, W2, b2 = Dims.split(theta_q, d.qshapes)
    x1 = np.concatenate([relu(obs @ W0 + b0), act], axis=1)
    x2 = relu(x1 @ W1 + b1)
    return x1, x2, (x2 @ W2 + b2)[:, 0]


def q_backward(d, theta_q, obs, x1, x2, dq):
    """Gradient of sum_b dq[b] Q(obs_b, act_b) with respect to the Q parameters and to the action input."""
    W0, b0, W1, b1, W2, b2 = Dims.split(theta_q, d.qshapes)
    d2 = dq[:, None] * W2[:, 0][None, :] * (x2 > 0)
    dx1 = d2 @ W1.T
    d1 = dx1[:, :H] * (x1[:, :H] > 0)
    g = [obs.T @ d1, d1.sum(0), x1.T @ d2, d2.sum(0), (x2.T @ dq)[:, None], np.array([dq.sum()])]
    return np.concatenate([x.reshape(-1) for x in g]), dx1[:, H:]


def pi_backward(d, theta_p, obs, a1, a2, mu, dmu):
    W0, b0, W1, b1, W2, b2 = Dims.split(theta_p, d.pshapes)
    dz = dmu * (1.0 - mu * mu)
    d2 = (dz @ W2.T) * (a2 > 0)
    d1 = (d2 @ W1.T) * (a1 > 0)
    g = [obs.T @ d1, d1.sum(0), a1.T @ d2, d2.sum(0), a2.T @ dz, dz.sum(0)]
    return np.concatenate([x.reshape(-1) for x in g])


def adam(theta, m, v, g, lr, t):
    a_t = lr * np.sqrt(1.0 - B2 ** t) / (1.0 - B1 ** t)
    m = B1 * m + (1.0 - B1) * g
    v = B2 * v + (1.0 - B2) * g * g
    return theta - a_t * m / (np.sqrt(v) + EPS), m, v


def targets_y(r, term, discount, q_next):
    """ys = rewards + (1 - terminals) * discount * Q'(s', mu'(s'))  (ddpg.py:343)."""
    return r + (1.0 - term) * discount * q_next


def soft_update(target, theta, tau):
    """target * (1 - tau) + theta * tau  (ddpg.py:352-357)."""
    return target * (1.0 - tau) + theta * tau


def do_training(d, nets, batch, hp, t):
    """One DDPG.do_training.  batch: dict s, a, r, term, s2 (float64 arrays).  Returns (new nets, info) with info =
    grad [P] (with weight decay), q, y, qf_loss, policy_surr."""
    th, m, v, tg = [x.copy() for x in nets]
    PP = d.PP
    wmask = d.weight_mask()
    s, a, r, term, s2 = batch["s"], batch["a"], batch["r"], batch["term"], batch["s2"]
    _, _, a_next = pi_forward(d, tg[:PP], s2)
    _, _, q_next = q_forward(d, tg[PP:], s2, a_next)
    y = targets_y(r, term, hp["discount"], q_next)
    x1, x2, q = q_forward(d, th[PP:], s, a)
    qf_loss = np.mean((y - q) ** 2)
    gq, _ = q_backward(d, th[PP:], s, x1, x2, -2.0 * (y - q) / BATCH)
    gq = gq + hp["qf_weight_decay"] * th[PP:] * wmask[PP:]
    th[PP:], m[PP:], v[PP:] = adam(th[PP:], m[PP:], v[PP:], gq, hp["qf_learning_rate"], t)
    a1, a2, mu = pi_forward(d, th[:PP], s)
    px1, px2, pq = q_forward(d, th[PP:], s, mu)
    surr = -np.mean(pq)
    _, dmu = q_backward(d, th[PP:], s, px1, px2, np.full(BATCH, -1.0 / BATCH))
    gp = pi_backward(d, th[:PP], s, a1, a2, mu, dmu) + hp["policy_weight_decay"] * th[:PP] * wmask[:PP]
    th[:PP], m[:PP], v[:PP] = adam(th[:PP], m[:PP], v[:PP], gp, hp["policy_learning_rate"], t)
    tg = soft_update(tg, th, hp["soft_target_tau"])
    return np.stack([th, m, v, tg]), dict(grad=np.concatenate([gp, gq]), q=q, y=y, qf_loss=qf_loss,
                                          policy_surr=surr)


def words(seed, itr, run, stream, sub):
    """The four Philox words of run `run` at step itr (include/b200rl.h, DDPG section)."""
    w = philox4x32_10(np.uint64(run), np.uint64((itr & 0x0FFFFFFF) | (stream << 28)), np.uint64(sub), np.uint64(0),
                      seed, itr >> 28)
    return [int(x) for x in w]


def accept_indices(candidates, bottom, size, rows, batch=BATCH, rejected=None):
    """SimpleReplayPool.random_batch's rule on a stream of offsets r in [0, size): index = (bottom + r) % rows, rejected
    when index == size - 1 (ddpg.py:54-70).  rejected: optional list that receives the rejected indices."""
    out = []
    for r in candidates:
        index = (bottom + r) % rows
        if index == size - 1:
            if rejected is not None:
                rejected.append(index)
            continue
        out.append(index)
        if len(out) == batch:
            break
    return np.array(out)


def index_offsets(seed, itr, run, update, size):
    """The Philox candidate offsets of one update: candidate c is word c & 3 of sub (update << 16) | (c >> 2), mapped to
    [0, size) by the 64-bit multiply-high (w * size) >> 32."""
    c = 0
    while True:
        w = words(seed, itr, run, STREAM_INDEX, (update << 16) | (c >> 2))[c & 3]
        yield (w * size) >> 32
        c += 1


def draw_indices(seed, itr, run, update, bottom, size, rows, rejected=None):
    return accept_indices(index_offsets(seed, itr, run, update, size), bottom, size, rows, rejected=rejected)


def pool_add(st, rows, obs, act, rew, term):
    """SimpleReplayPool.add_sample (ddpg.py:43-52) on st's float32 pool and its top / bottom / size."""
    pool, top = st["pool"], st["top"]
    pool["obs"][top] = obs
    pool["act"][top] = act
    pool["rew"][top] = rew
    pool["term"][top] = 1 if term else 0
    st["top"] = (top + 1) % rows
    if st["size"] >= rows:
        st["bottom"] = (st["bottom"] + 1) % rows
    else:
        st["size"] += 1


def ou_step(x, mu, theta, sigma, n):
    """OUStrategy.evolve_state: x + theta (mu - x) + sigma n."""
    return x + (theta * (mu - x) + sigma * n)


def gaussian_sigma(t, max_sigma, min_sigma, decay_period):
    return max_sigma - (max_sigma - min_sigma) * min(1.0, t * 1.0 / decay_period)


def explore_normals(seed, itr, run, A):
    n = np.zeros(A)
    for c in range((A + 3) // 4):
        w = words(seed, itr, run, STREAM_EXPLORE, c)
        for p in range(2):
            u0 = (w[2 * p] + 0.5) * 2.0 ** -32
            u1 = (w[2 * p + 1] + 0.5) * 2.0 ** -32
            rad = np.sqrt(-2.0 * np.log(u0))
            for j, val in ((0, rad * np.cos(2 * np.pi * u1)), (1, rad * np.sin(2 * np.pi * u1))):
                if c * 4 + 2 * p + j < A:
                    n[c * 4 + 2 * p + j] = val
    return n


def gather(pool, idx, rows):
    return dict(s=pool["obs"][idx].astype(np.float64), a=pool["act"][idx].astype(np.float64),
                r=pool["rew"][idx].astype(np.float64), term=pool["term"][idx].astype(np.float64),
                s2=pool["obs"][(idx + 1) % rows].astype(np.float64))


def train_step(d, st, hp, seed, run, env_reset, env_step, stats=None, record=None):
    """One iteration of DDPG.train()'s loop on the run state st (modified in place).  env_reset(itr) -> (env_state, obs)
    and env_step(env_state, action float32 in [-1, 1]) -> (env_state, obs, reward, done) are the env.  stats: optional
    dict of lists (es_returns, qf_loss, policy_surr, q, y); record: optional list that receives each update's
    (indices, info, rejected indices)."""
    rows = hp["replay_pool_size"]
    if st["terminal"]:
        st["env_state"], st["obs"] = env_reset(st["itr"])
        st["ou"] = np.full(d.A, hp["ou_mu"], np.float64)
        if st["terminal"] == 1 and stats is not None:
            stats["es_returns"].append(st["path_return"])
        st["path_length"], st["path_return"], st["terminal"] = 0, 0.0, 0
    _, _, mu = pi_forward(d, st["nets"][0][:d.PP], np.asarray(st["obs"], np.float64)[None, :])
    nz = explore_normals(seed, st["itr"], run, d.A)
    if hp["es_kind"] == 0:
        st["ou"] = ou_step(st["ou"], hp["ou_mu"], hp["ou_theta"], hp["ou_sigma"], nz)
        x = mu[0] + st["ou"]
    else:
        x = mu[0] + nz * gaussian_sigma(st["itr"], hp["gs_max_sigma"], hp["gs_min_sigma"], hp["gs_decay_period"])
    act = np.clip(x, -1.0, 1.0).astype(np.float32)
    env_state, obs2, r, done = env_step(st["env_state"], act)
    st["path_length"] += 1
    st["path_return"] += float(r)
    add, term = True, bool(done)
    if not done and st["path_length"] >= hp["max_path_length"]:
        term = True
        add = bool(hp["include_horizon_terminal_transitions"])
    if add:
        pool_add(st, rows, st["obs"], act, np.float32(float(r) * hp["scale_reward"]), term)
    st["terminal"] = 1 if term else 0
    st["env_state"], st["obs"] = env_state, obs2
    if st["size"] >= hp["min_pool_size"]:
        for u in range(hp["n_updates_per_sample"]):
            rejected = []
            idx = draw_indices(seed, st["itr"], run, u, st["bottom"], st["size"], rows, rejected=rejected)
            st["adam_t"] += 1
            st["nets"], info = do_training(d, st["nets"], gather(st["pool"], idx, rows), hp, st["adam_t"])
            if stats is not None:
                for k in ("qf_loss", "policy_surr", "q", "y"):
                    stats[k].append(info[k])
            if record is not None:
                record.append((idx, info, rejected))
    st["itr"] += 1
    return st
