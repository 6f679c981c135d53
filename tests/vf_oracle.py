"""float64 NumPy restatement of GaussianMLPRegressor (rllab/regressors/gaussian_mlp_regressor.py) for the tests of the
GaussianMLPBaseline kernels: normalisation, forward, NLL, KL and the hand-written gradient, plus a whole fit driven by
the optimizers with these callables.  Sample-major arrays: xs (n, O), ys (n,).  ReLU derivative 0 at a pre-activation
<= 0 (Theano's relu gives 1/2 at exactly 0; a measure-zero difference)."""
import numpy as np

HALF_LOG_2PI = 0.5 * np.log(2 * np.pi)


def num_params(O, H=32):
    return O * H + H + H * H + H + H + 1 + 1


def unflatten(theta, O, H=32):
    """[W0 (O,H), b0, W1 (H,H), b1, Wout (H,1), bout, log_std]  (core/lasagne_powered.py flat layout)"""
    i = 0
    out = []
    for s in [(O, H), (H,), (H, H), (H,), (H, 1), (1,), (1,)]:
        n = int(np.prod(s))
        out.append(np.asarray(theta[i:i + n], dtype=np.float64).reshape(s))
        i += n
    return out


def init_params(O, rng, init_std=1.0, H=32):
    """GlorotUniform weights, zero biases, log(init_std) (core/network.py:38-39, gaussian_mlp_regressor.py:106-112)."""
    vals = []
    for s in [(O, H), (H,), (H, H), (H,), (H, 1), (1,)]:
        if len(s) == 2:
            a = np.sqrt(6.0 / (s[0] + s[1]))
            vals.append(rng.uniform(-a, a, size=s).reshape(-1))
        else:
            vals.append(np.zeros(s))
    vals.append(np.full((1,), np.log(init_std)))
    return np.concatenate(vals)


def norm_stats(xs, ys):
    """gaussian_mlp_regressor.py:197-208: x_mean, x_std + 1e-8, y_mean, y_std + 1e-8 (np.std = population std)."""
    xs = np.asarray(xs, dtype=np.float64)
    ys = np.asarray(ys, dtype=np.float64).reshape(-1)
    return np.concatenate([xs.mean(0), xs.std(0) + 1e-8, [ys.mean(), ys.std() + 1e-8]])


def normalize(xs, ys, stats, O):
    nx = (np.asarray(xs, dtype=np.float64) - stats[:O]) / stats[O:2 * O]
    ny = None if ys is None else (np.asarray(ys, dtype=np.float64).reshape(-1) - stats[2 * O]) / stats[2 * O + 1]
    return nx, ny


def forward(theta, nx, O):
    """MLP of core/network.py:36-81 with rectify hidden units, linear output: normalised mean (n,), activations."""
    W0, b0, W1, b1, Wo, bo, _ = unflatten(theta, O)
    a1 = nx @ W0 + b0
    h1 = np.maximum(a1, 0.0)
    a2 = h1 @ W1 + b1
    h2 = np.maximum(a2, 0.0)
    mu = (h2 @ Wo + bo).reshape(-1)
    return mu, (a1, h1, a2, h2)


def predict(theta, xs, stats, O):
    """f_predict (gaussian_mlp_regressor.py:168,225-231): mu(nx) * y_std + y_mean."""
    nx, _ = normalize(xs, None, stats, O)
    return forward(theta, nx, O)[0] * stats[2 * O + 1] + stats[2 * O]


def loss_terms(theta, nx, ny, O, mu_old=None, ls_old=None):
    """Per-sample NLL (diagonal_gaussian.py:58-69) and KL(old || new) (:14-34) in normalised space."""
    mu, _ = forward(theta, nx, O)
    ls = theta[-1]
    var = np.exp(2 * ls)
    nll = ls + 0.5 * (ny - mu) ** 2 / var + HALF_LOG_2PI
    if mu_old is None:
        return nll, np.zeros_like(nll)
    var_old = np.exp(2 * ls_old)
    kl = ((mu_old - mu) ** 2 + var_old - var) / (2 * var + 1e-8) + ls - ls_old
    return nll, kl


def loss_grad(theta, nx, ny, O, penalty=0.0, mu_old=None, ls_old=None, learn_std=True, weights=None):
    """(mean NLL, mean KL, max KL, gradient [P] of mean NLL + penalty * mean KL); weights: 0/1 per sample (masked
    samples) -- means over the weighted samples.  learn_std=False: the log_std slot of the gradient is 0."""
    W0, b0, W1, b1, Wo, bo, _ = unflatten(theta, O)
    n = len(ny)
    w = np.ones(n) if weights is None else np.asarray(weights, dtype=np.float64)
    cnt = w.sum()
    mu, (a1, h1, a2, h2) = forward(theta, nx, O)
    ls = theta[-1]
    var = np.exp(2 * ls)
    var2 = 2 * var + 1e-8
    r = ny - mu
    nll = ls + 0.5 * r ** 2 / var + HALF_LOG_2PI
    dmu = -r / var
    dls = 1.0 - r ** 2 / var
    kl = np.zeros(n)
    if mu_old is not None:
        var_old = np.exp(2 * ls_old)
        dm = mu_old - mu
        num = dm ** 2 + var_old - var
        kl = num / var2 + ls - ls_old
        dmu = dmu + penalty * (-2 * dm / var2)
        dls = dls + penalty * (1.0 - 2 * var * (var2 + 2 * num) / var2 ** 2)
    dmu = dmu * w / cnt
    dls = dls * w / cnt
    d2 = (dmu[:, None] * Wo[:, 0][None, :]) * (a2 > 0)
    d1 = (d2 @ W1.T) * (a1 > 0)
    g = np.concatenate([(nx.T @ d1).reshape(-1), d1.sum(0), (h1.T @ d2).reshape(-1), d2.sum(0),
                        (h2.T @ dmu[:, None]).reshape(-1), [dmu.sum()], [dls.sum() if learn_std else 0.0]])
    valid = w > 0
    max_kl = float(kl[valid].max()) if mu_old is not None and valid.any() else -1e300
    return float((nll * w).sum() / cnt), float((kl * w).sum() / cnt), max_kl, g


class _Target(object):
    def __init__(self, theta, learn_std):
        self.theta = np.array(theta, dtype=np.float64)
        self.learn_std = learn_std

    def get_param_values(self, trainable=False, **tags):
        return (self.theta[:-1] if trainable and not self.learn_std else self.theta).copy()

    def set_param_values(self, v, trainable=False, **tags):
        if trainable and not self.learn_std:
            self.theta[:-1] = v
        else:
            self.theta[:] = v


def callables(target, O, learn_std=True):
    """The optimizer callables of the regressor (f_loss, f_constraint, f_opt, f_penalized_loss, f_opt_plain) on the
    oracle, evaluated at target.theta; inputs = (nx, ny, mu_old, ls_old, weights)."""
    def ev(inp, penalty):
        nx, ny, mu_old, ls_old, w = inp
        return loss_grad(target.theta, nx, ny, O, penalty, mu_old, ls_old, learn_std, w)

    def trainable(g):
        return g if learn_std else g[:-1]

    def f_loss(*inp):
        return ev(inp, 0.0)[0]

    def f_constraint(*inp):
        return ev(inp, 0.0)[1]

    def f_opt(*args):
        *inp, penalty = args
        nll, kl, _, g = ev(inp, penalty)
        return nll + penalty * kl, trainable(g)

    def f_penalized_loss(*args):
        *inp, penalty = args
        nll, kl, _, _ = ev(inp, 0.0)
        return nll + penalty * kl, nll, kl

    def f_opt_plain(*inp):
        nll, _, _, g = ev(inp, 0.0)
        return nll, trainable(g)
    return f_loss, f_constraint, f_opt, f_penalized_loss, f_opt_plain


def fit(theta, xs, ys, O, optimizer, use_trust_region=True, step_size=0.01, learn_std=True, stats=None, weights=None):
    """GaussianMLPRegressor.fit (gaussian_mlp_regressor.py:186-223) on the oracle with one of the rllab_b200 host
    optimizers (or the reference's, which share the interface).  Returns (theta, stats, dict of the tabular values)."""
    if stats is None:
        w = np.ones(len(ys), dtype=bool) if weights is None else np.asarray(weights) > 0
        stats = norm_stats(np.asarray(xs)[w], np.asarray(ys).reshape(-1)[w])
    nx, ny = normalize(xs, ys, stats, O)
    tgt = _Target(theta, learn_std)
    f_loss, f_constraint, f_opt, f_pen, f_plain = callables(tgt, O, learn_std)
    if use_trust_region:
        mu_old = forward(tgt.theta, nx, O)[0]
        inputs = (nx, ny, mu_old, float(tgt.theta[-1]), weights)
        optimizer._target = tgt
        optimizer._max_constraint_val = step_size
        optimizer._constraint_name = "mean_kl"
        optimizer._opt_fun = dict(f_loss=f_loss, f_constraint=f_constraint, f_penalized_loss=f_pen, f_opt=f_opt)
    else:
        inputs = (nx, ny, None, None, weights)
        optimizer._target = tgt
        optimizer._opt_fun = dict(f_loss=f_loss, f_opt=f_plain)
    loss_before = optimizer.loss(inputs)
    optimizer.optimize(inputs)
    loss_after = optimizer.loss(inputs)
    info = dict(LossBefore=loss_before, LossAfter=loss_after, dLoss=loss_before - loss_after)
    if use_trust_region:
        info["MeanKL"] = optimizer.constraint_val(inputs)
    return tgt.theta.copy(), stats, info
