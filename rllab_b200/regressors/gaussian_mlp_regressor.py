"""GaussianMLPRegressor (rllab/regressors/gaussian_mlp_regressor.py:20-244) on the GPU.

The network is the reference's default: MLP(input_dim -> 32 -> 32 -> 1), ReLU hidden units, no output nonlinearity, a
state-independent log_std (ParamLayer, trainable iff learn_std).  The flat layout is the policy's with act_dim = 1:
[W0 (O,32), b0, W1 (32,32), b1, Wout (32,1), bout, log_std].  Every pass runs in the CUDA kernels of csrc/vf.cu:

  normalisation constants   b200rl_vf_norm_stats (float64 column means / population stds + 1e-8 of the valid samples)
  mean                      b200rl_vf_forward (normalised for the trust region's old means, denormalised for predict)
  loss / gradient           b200rl_vf_loss_grad (mean NLL, mean KL, gradient of NLL + penalty * KL)

The optimizer (PenaltyLbfgsOptimizer with the trust region, LbfgsOptimizer without) runs scipy's fmin_l_bfgs_b on the
host; each of its function evaluations copies theta to the device and reads back (loss, KL, gradient).  Host arrays
passed to fit / predict are uploaded as float32 and go through the same kernels: there is no CPU path.

One deviation from the reference: fit() shuffles the samples through iterate_minibatches_generic(shuffle=True) even when
they make a single batch, which changes only the order of summation and the host RNG stream.  This version sums in
lane order and leaves np.random untouched.  The trust region's old means are the normalised network output itself,
where the reference denormalises and normalises them again (identical up to float64 rounding).
"""
import numpy as np

from .. import _lib as L
from ..misc import logger
from ..optimizers.lbfgs_optimizer import LbfgsOptimizer
from ..optimizers.penalty_lbfgs_optimizer import PenaltyLbfgsOptimizer

class _Data(object):
    """Device samples of one fit: obs [O][B], y [B] float32, flags [B] (or None), the valid-sample count."""

    def __init__(self, obs, y, flags, B, fit_id):
        self.obs, self.y, self.flags, self.B, self.fit_id = obs, y, flags, int(B), fit_id


class GaussianMLPRegressor(object):
    """
    A class for performing regression by fitting a Gaussian distribution to the outputs.
    """

    def __init__(
            self,
            input_shape,
            output_dim,
            mean_network=None,
            hidden_sizes=(32, 32),
            hidden_nonlinearity=None,
            optimizer=None,
            use_trust_region=True,
            step_size=0.01,
            learn_std=True,
            init_std=1.0,
            adaptive_std=False,
            std_share_network=False,
            std_hidden_sizes=(32, 32),
            std_nonlinearity=None,
            normalize_inputs=True,
            normalize_outputs=True,
            name=None,
            batchsize=None,
            subsample_factor=1.,
    ):
        if mean_network is not None:
            raise NotImplementedError("mean_network: only the default MLP is compiled into the kernels")
        if tuple(hidden_sizes) != (32, 32):
            raise NotImplementedError("hidden_sizes=%s: only (32, 32) is compiled into the kernels" % (hidden_sizes,))
        if hidden_nonlinearity not in (None, "rectify"):
            raise NotImplementedError("hidden_nonlinearity: only rectify (None = the default) is compiled in")
        if adaptive_std:
            raise NotImplementedError("adaptive_std")
        if std_share_network:
            raise NotImplementedError("std_share_network")
        if batchsize is not None:
            raise NotImplementedError("batchsize (mini-batches): the fit runs on the full batch")
        if subsample_factor < 1:
            raise NotImplementedError("subsample_factor < 1")
        if int(output_dim) != 1:
            raise NotImplementedError("output_dim=%d: only 1 (the value function) is compiled in" % output_dim)
        if len(input_shape) != 1:
            raise NotImplementedError("input_shape must be (obs_dim,)")
        if optimizer is not None and not isinstance(optimizer, (PenaltyLbfgsOptimizer, LbfgsOptimizer)):
            raise NotImplementedError("optimizer must be a PenaltyLbfgsOptimizer or an LbfgsOptimizer")
        self._init_args = dict(input_shape=tuple(input_shape), output_dim=output_dim, hidden_sizes=tuple(hidden_sizes),
                               use_trust_region=use_trust_region, step_size=step_size, learn_std=learn_std,
                               init_std=init_std, normalize_inputs=normalize_inputs,
                               normalize_outputs=normalize_outputs, name=name)
        self.obs_dim = O = int(input_shape[0])
        self._batchsize = batchsize
        self._subsample_factor = subsample_factor
        if optimizer is None:
            optimizer = PenaltyLbfgsOptimizer() if use_trust_region else LbfgsOptimizer()
        self._optimizer = optimizer
        self._use_trust_region = use_trust_region
        self._step_size = step_size
        self._learn_std = learn_std
        self._name = name
        self._normalize_inputs = normalize_inputs
        self._normalize_outputs = normalize_outputs

        shapes = [(O, 32), (32,), (32, 32), (32,), (32, 1), (1,)]
        vals = []
        for s in shapes:        # GlorotUniform weights, zero biases (core/network.py:38-39)
            if len(s) == 2:
                a = np.sqrt(6.0 / (s[0] + s[1]))
                vals.append(np.random.uniform(-a, a, size=s).reshape(-1))
            else:
                vals.append(np.zeros(s))
        vals.append(np.full((1,), np.log(init_std)))
        self._theta = np.concatenate(vals).astype(np.float64)
        self.n_params = self._theta.size
        self._ols = self.n_params - 1
        # [x_mean (O), x_std (O), y_mean, y_std]: zeros / ones until the first fit (gaussian_mlp_regressor.py:126-145)
        self._stats_host = np.concatenate([np.zeros(O), np.ones(O), [0.0, 1.0]])
        self._dev = None
        self.n_evals = 0
        self.last_fit = None
        self._version = 0          # bumped by set_param_values: keys the cached forward-only result
        self._n_fits = 0
        self._fwd_cache = None
        self._bind_optimizer()

    # ---------------------------------------------------------------- optimizer wiring
    def _bind_optimizer(self):
        if self._use_trust_region:
            self._optimizer.update_opt(loss=self._f_loss, target=self, leq_constraint=(self._f_constraint, self._step_size),
                                       inputs=None, constraint_name="mean_kl", f_opt=self._f_opt_penalized,
                                       f_penalized_loss=self._f_penalized_loss)
        else:
            self._optimizer.update_opt(loss=self._f_loss, target=self, inputs=None, f_opt=self._f_opt)

    def _eval(self, data, penalty, grad):
        """One device pass at the current parameters: (mean NLL, mean KL, flat gradient or None), reduced over ranks.
        The forward-only result does not depend on the penalty and is kept for the current (parameters, fit): the loss
        after the fit and the constraint value (gaussian_mlp_regressor.py:219-221) then share one pass."""
        from .. import ops
        key = (self._version, data.fit_id)
        if not grad and self._fwd_cache is not None and self._fwd_cache[0] == key:
            return self._fwd_cache[1] + (None,)
        d = self._ensure_device()
        comm = d["comm"]
        fuse = comm is not None and comm.active and comm.fuse
        out = d["out"] if grad else d["tri"]
        ops.vf_loss_grad(d["theta32"], self.obs_dim, data.B, data.obs, data.y, data.flags, d["stats"],
                         d["mu_old"] if self._use_trust_region else None, d["ls_old"], penalty, self._learn_std, 1.0,
                         d["count"], d["out"][:self.n_params] if grad else None, d["tri"], fuse=fuse)
        if comm is not None and comm.active:
            comm.after_pass(out, out.numel() - 1)
        h = out.cpu().numpy()
        self.n_evals += 1
        tri = h[-3:]
        g = None
        if grad:
            g = h[:self.n_params] if self._learn_std else h[:self._ols]
            g = np.array(g, dtype=np.float64)
        if not grad:
            self._fwd_cache = (key, (float(tri[0]), float(tri[1])))
        return float(tri[0]), float(tri[1]), g

    def _f_loss(self, data):
        return self._eval(data, 0.0, False)[0]

    def _f_constraint(self, data):
        return self._eval(data, 0.0, False)[1]

    def _f_opt(self, data):
        nll, _, g = self._eval(data, 0.0, True)
        return nll, g

    def _f_opt_penalized(self, data, penalty):
        nll, kl, g = self._eval(data, float(penalty), True)
        return nll + penalty * kl, g

    def _f_penalized_loss(self, data, penalty):
        nll, kl, _ = self._eval(data, 0.0, False)
        return nll + penalty * kl, nll, kl

    # ---------------------------------------------------------------- device state
    def _ensure_device(self):
        import torch
        if self._dev is None:
            if not torch.cuda.is_available():
                raise L.B200RLError("GaussianMLPRegressor needs a CUDA device (no CPU fallback)")
            dev = torch.device("cuda", torch.cuda.current_device())
            O, P = self.obs_dim, self.n_params
            if L.vf_num_params(O) != P:
                raise L.B200RLError("regressor parameter count mismatch")
            out = torch.zeros(P + 3, dtype=torch.float64, device=dev)   # [gradient | mean NLL, mean KL, max KL]
            self._dev = dict(device=dev, theta64=torch.as_tensor(self._theta).to(dev),
                             theta32=torch.zeros(P, dtype=torch.float32, device=dev),
                             stats=torch.as_tensor(self._stats_host).to(dev),
                             acc=torch.zeros(2 * O + 3, dtype=torch.float64, device=dev),
                             new_stats=torch.zeros(2 * O + 2, dtype=torch.float64, device=dev),
                             out=out, tri=out[P:], mu_old=None, mu_old_buf=None, ls_old=0.0, count=None, comm=None)
            self._dev["theta32"].copy_(self._dev["theta64"])
        return self._dev

    @property
    def device(self):
        return self._ensure_device()["device"]

    def get_param_values(self, trainable=False, **tags):
        if trainable and not self._learn_std:
            return self._theta[:self._ols].copy()
        return self._theta.copy()

    def set_param_values(self, flattened_params, trainable=False, **tags):
        v = np.asarray(flattened_params, dtype=np.float64)
        if trainable and not self._learn_std:
            self._theta[:self._ols] = v
        else:
            self._theta[:] = v
        self._version += 1
        if self._dev is not None:
            import torch
            d = self._dev
            d["theta64"].copy_(torch.as_tensor(self._theta))
            d["theta32"].copy_(d["theta64"])

    def get_stats(self):
        """[x_mean (O), x_std (O), y_mean, y_std] as a host float64 array."""
        if self._dev is not None:
            self._stats_host = self._dev["stats"].cpu().numpy().copy()
        return self._stats_host.copy()

    # ---------------------------------------------------------------- fit
    def fit_device(self, obs, y, flags=None, comm=None):
        """fit() on device samples: obs [O][B], y [B] float32 CUDA tensors; samples with FLAG_MASKED in flags (uint8 [B],
        or None) are left out.  With a communicator every rank passes its shard and all ranks end with the same theta."""
        from .. import ops
        import torch
        d = self._ensure_device()
        d["comm"] = comm                    # this fit's communicator (None: the samples are the whole batch)
        O = self.obs_dim
        B = int(y.numel())
        self._n_fits += 1
        data = _Data(obs, y, flags, B, self._n_fits)
        active = comm is not None and comm.active
        acc = d["acc"]
        if active:
            ops.vf_norm_stats(O, B, obs, y, flags, ops.VF_STATS_SUMS, acc, d["new_stats"])
            comm.all_reduce_sum(acc[:O + 2])
            ops.vf_norm_stats(O, B, obs, y, flags, ops.VF_STATS_SQUARES, acc, d["new_stats"])
            comm.all_reduce_sum(acc[O + 2:])
            ops.vf_norm_stats(O, B, obs, y, flags, ops.VF_STATS_FINISH, acc, d["new_stats"])
        else:
            ops.vf_norm_stats(O, B, obs, y, flags, ops.VF_STATS_ALL, acc, d["new_stats"])
        d["count"] = acc[O + 1:O + 2]
        if self._normalize_inputs:          # gaussian_mlp_regressor.py:197-208
            d["stats"][:2 * O].copy_(d["new_stats"][:2 * O])
        if self._normalize_outputs:
            d["stats"][2 * O:].copy_(d["new_stats"][2 * O:])
        self._stats_host = None
        prefix = self._name + "_" if self._name else ""
        loss_before, loss_after, mean_kl, batch_count = 0., 0., 0., 0
        batch_count += 1
        if self._use_trust_region:
            # old distribution after the new constants are set (_f_pdists at :215-216): theta_old on the new nx
            if d["mu_old_buf"] is None or d["mu_old_buf"].numel() < B:
                d["mu_old_buf"] = torch.empty(B, dtype=torch.float32, device=d["device"])
            d["mu_old"] = d["mu_old_buf"][:B]
            ops.vf_forward(d["theta32"], O, B, obs, d["stats"], d["mu_old"], False)
            d["ls_old"] = float(np.float32(self._theta[self._ols]))
        self.n_evals = 0
        inputs = [data]
        loss_before += self._optimizer.loss(inputs)
        self._optimizer.optimize(inputs)
        loss_after += self._optimizer.loss(inputs)
        if self._use_trust_region:
            mean_kl += self._optimizer.constraint_val(inputs)
        self.last_fit = dict(loss_before=loss_before, loss_after=loss_after, mean_kl=mean_kl, n_evals=self.n_evals)
        logger.record_tabular(prefix + 'LossBefore', loss_before / batch_count)
        logger.record_tabular(prefix + 'LossAfter', loss_after / batch_count)
        logger.record_tabular(prefix + 'dLoss', loss_before - loss_after / batch_count)
        if self._use_trust_region:
            logger.record_tabular(prefix + 'MeanKL', mean_kl / batch_count)

    def _upload(self, xs, ys=None):
        import torch
        d = self._ensure_device()
        xs = np.asarray(xs, dtype=np.float64).reshape(-1, self.obs_dim)
        obs = torch.as_tensor(np.ascontiguousarray(xs.T), dtype=torch.float32).to(d["device"]).contiguous()
        y = None
        if ys is not None:
            y = torch.as_tensor(np.asarray(ys, dtype=np.float64).reshape(-1), dtype=torch.float32).to(d["device"])
        return obs, y, xs.shape[0]

    def fit(self, xs, ys):
        obs, y, _ = self._upload(xs, ys)
        self.fit_device(obs, y, None, None)

    # ---------------------------------------------------------------- predict
    def predict_device(self, obs, out, normalized=False):
        """out [B] float32 = the regressor mean on obs [O][B] (denormalised unless `normalized`)."""
        from .. import ops
        d = self._ensure_device()
        ops.vf_forward(d["theta32"], self.obs_dim, int(out.numel()), obs, d["stats"], out, not normalized)

    def predict(self, xs):
        """
        Return the maximum likelihood estimate of the predicted y.
        """
        import torch
        obs, _, n = self._upload(xs)
        out = torch.empty(n, dtype=torch.float32, device=obs.device)
        self.predict_device(obs, out)
        return out.cpu().numpy().astype(np.float64).reshape(-1, 1)

    def _pdists(self, xs):
        means = self.predict(xs)
        log_std = self._theta[self._ols] + np.log(self.get_stats()[-1])
        return means, np.full_like(means, log_std)

    def sample_predict(self, xs):
        """
        Sample one possible output from the prediction distribution.
        """
        means, log_stds = self._pdists(xs)
        return np.random.normal(size=means.shape) * np.exp(log_stds) + means

    def predict_log_likelihood(self, xs, ys):
        means, log_stds = self._pdists(xs)
        zs = (np.asarray(ys, dtype=np.float64).reshape(means.shape) - means) / np.exp(log_stds)
        return - np.sum(log_stds, axis=-1) - 0.5 * np.sum(np.square(zs), axis=-1) - 0.5 * means.shape[-1] * np.log(2 * np.pi)

    # ---------------------------------------------------------------- pickling
    def __getstate__(self):
        opt = dict(self._optimizer.__dict__)
        for k in ("_opt_fun", "_target"):
            opt.pop(k, None)
        return dict(init_args=self._init_args, theta=self._theta.copy(), stats=self.get_stats(),
                    optimizer_cls=type(self._optimizer), optimizer_state=opt)

    def __setstate__(self, s):
        a = s["init_args"]
        opt = s["optimizer_cls"].__new__(s["optimizer_cls"])
        opt.__dict__.update(s["optimizer_state"])
        rng_state = np.random.get_state()     # the initial weights drawn by __init__ are overwritten below: do not let
        self.__init__(optimizer=opt, **a)     # unpickling advance the host RNG
        np.random.set_state(rng_state)
        self._theta = np.array(s["theta"], dtype=np.float64)
        self._stats_host = np.array(s["stats"], dtype=np.float64)
