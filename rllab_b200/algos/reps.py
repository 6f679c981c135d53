"""REPS (rllab/algos/reps.py): relative entropy policy search with its dual and sample weights evaluated on the GPU.

Each iteration minimises the dual

    g(eta, v) = eta eps + eta log mean exp(delta / eta - max delta / eta) + eta max(delta / eta) + L2_reg_dual (eta^2 + eta^-2)

over eta >= 0 and the value-function weights v, where delta = r + feat_diff . v is the sample Bellman error with the
linear features of reps.py:207-211, then fits the policy to the weights w = exp(delta / eta - max delta / eta) by
minimising -mean(logp * w) (+ the L2 term).  Both minimisations run scipy's L-BFGS(-B) on the host, as the reference does;
every function evaluation is one pass over the lane batch on the GPU:

  dual     b200rl_reps_delta_max (M = max delta) then b200rl_reps_dual_sums ([sum e, sum e (delta - M), sum e feat_diff]
           with e = exp((delta - M) / eta)); g and its gradient are formed on the host in float64 from these sums and
           the device-resident valid-sample count.  The features of a sample and of its successor are evaluated inside
           the pass: nothing per sample is stored (the reference builds feat_diff, 2 O + 4 floats per sample, on the host).
  weights  one more b200rl_reps_dual_sums pass at the solution writes w (float32, 0 on dropped samples) into a buffer
           owned by REPS.
  policy   PolicyObjective(policy, LOSS_VPG) on a view of the batch that shares its sample buffers but reads w as the
           advantages (samples_data's advantages are untouched): the VPG surrogate -mean(logp * adv) with adv := w is the
           REPS loss.  The L2_reg_loss term and its gradient are added on the host.
  MeanKL   mean KL(old || new) of the b200rl_loss_kl pass at the final parameters.

Regularizable parameters (the L2_reg_loss term, reps.py:115-118): lasagne's Layer.add_param tags every parameter
regularizable unless told otherwise; DenseLayer adds its bias with regularizable=False; rllab's ParamLayer
(core/lasagne_layers.py:15) adds the log_std parameter with the defaults.  So for GaussianMLPPolicy they are W0, W1,
Wout and log_std (n_reg = 4), and the term is L2_reg_loss * sum_p mean(p^2) / 4; CategoricalMLPPolicy has no log_std, so
its regularizable parameters are W0, W1 and Wout (n_reg = 3).

Multi-GPU: the maximum and the sums are all-reduced through the Comm (max, then sums), and the policy passes through
PolicyObjective's reduction, so every rank hands scipy identical numbers and theta, eta and v are bit-identical across
ranks.  The initial v (a host np.random draw, as in the reference) is taken from rank 0.

Deliberate deviations from the reference:
  * Summation order: float64 sums in fixed block order on the device (deterministic), not Theano's order; the policy
    passes are float32-grade per sample (the VPG gradient kernel).
  * One device pass serves both scipy callbacks at the same point (func and fprime are cached by the bytes of x).
  * The max shift: g uses M = max delta directly for eta max(delta / eta), and the gradient uses its analytic form (the
    shift cancels); the weights are exp((delta - M) / eta).
  * eta and v survive a snapshot: init_opt draws them only once (the reference pickles the constructor call and draws
    them again when a resumed run calls init_opt).
  * scipy >= 1.18's fmin_l_bfgs_b has no `disp` argument: when the optimizer is that function it is called without it.
    Any other optimizer receives the reference's exact keyword arguments.
  * plot=True and recurrent policies raise NotImplementedError.
"""
import copy

import numpy as np
import scipy.optimize

from .. import _lib as L
from ..core.serializable import Serializable
from ..misc import logger
from ..optimizers.conjugate_gradient_optimizer import _lane_batch
from .batch_polopt import BatchPolopt
from .policy_objective import PolicyObjective


def dual_from_sums(eta, M, sums, count, epsilon, l2_reg_dual):
    """(g, [dg/deta, dg/dv]) in float64 from M = max delta and the sums of b200rl_reps_dual_sums (all ranks)."""
    eta = np.float64(eta)
    s0, s1, sphi = sums[0], sums[1], np.asarray(sums[2:], dtype=np.float64)
    with np.errstate(all="ignore"):
        lme = np.log(s0 / count)
        g = eta * epsilon + eta * lme + M + l2_reg_dual * (np.square(eta) + np.square(1 / eta))
        dg_eta = epsilon + lme - s1 / (eta * s0) + l2_reg_dual * (2 * eta - 2 / eta ** 3)
        dg_v = sphi / s0
    return float(g), np.concatenate([[dg_eta], dg_v])


def regularizable_slices(policy):
    """Flat-parameter slices of the weight matrices and, for GaussianMLPPolicy, log_std (see the module docstring)."""
    from .. import ops
    has_log_std = not ops.is_categorical(getattr(policy, "dims", None))
    out, k = [], 0
    shapes = policy.get_param_shapes()
    for i, s in enumerate(shapes):
        n = int(np.prod(s))
        if len(s) == 2 or (has_log_std and i == len(shapes) - 1):
            out.append(slice(k, k + n))
        k += n
    return out


class REPS(BatchPolopt, Serializable):
    """
    Relative Entropy Policy Search (REPS)

    References
    ----------
    [1] J. Peters, K. Mulling, and Y. Altun, "Relative Entropy Policy Search," Artif. Intell., pp. 1607-1612, 2008.
    """

    def __init__(
            self,
            epsilon=0.5,
            L2_reg_dual=0.,
            L2_reg_loss=0.,
            max_opt_itr=50,
            optimizer=scipy.optimize.fmin_l_bfgs_b,
            **kwargs):
        """
        :param epsilon: Max KL divergence between new policy and old policy.
        :param L2_reg_dual: Dual regularization
        :param L2_reg_loss: Loss regularization
        :param max_opt_itr: Maximum number of batch optimization iterations.
        :param optimizer: the minimiser of both steps, called as scipy.optimize.fmin_l_bfgs_b is.
        Other keywords go to BatchPolopt (env, policy, baseline, n_itr, batch_size, max_path_length, ...).
        """
        Serializable.quick_init(self, locals())
        super(REPS, self).__init__(**kwargs)
        self.epsilon = epsilon
        self.L2_reg_dual = L2_reg_dual
        self.L2_reg_loss = L2_reg_loss
        self.max_opt_itr = max_opt_itr
        self.optimizer = optimizer
        self.opt_info = None
        self.param_eta = None
        self.param_v = None
        self._objective = None
        self._comm = None
        self._bufs = None
        self._view_version = 0
        self.n_dual_evals = 0         # dual passes (delta_max + dual_sums) of the last optimize_policy
        self.n_policy_evals = 0       # policy gradient passes of the last optimize_policy

    def __getstate__(self):
        d = BatchPolopt.__getstate__(self)
        d.update(_bufs=None, _comm=None)
        return d

    def __setstate__(self, d):
        BatchPolopt.__setstate__(self, d)

    def init_opt(self):
        if self.policy.recurrent:
            raise NotImplementedError("recurrent policies (the `valids` branch of reps.py) are not built")
        comm = getattr(self.sampler, "comm", None)
        self._comm = comm
        if self.param_eta is None:        # a resumed snapshot keeps its dual variables
            self.param_eta = 15.
            v = np.random.rand(self.env.observation_space.flat_dim * 2 + 4)
            if comm is not None and comm.active:
                import torch
                t = torch.tensor(v if comm.rank == 0 else np.zeros_like(v), dtype=torch.float64,
                                 device=self.policy.theta64.device)
                comm.all_reduce_mixed(t, t.numel())   # one non-zero term per entry: rank 0's draw, exactly
                v = t.cpu().numpy()
            self.param_v = v
        self._objective = PolicyObjective(self.policy, L.LOSS_VPG, comm)
        self.opt_info = dict(f_kl=self._objective.kl_stats)

    # ---- device passes
    def _buffers(self, b):
        import torch
        D = 2 * b.O + 4
        bf = self._bufs
        if bf is None or bf["w"].shape != (b.T, b.N) or bf["w"].device != b.device or bf["v"].numel() != D:
            red = torch.zeros(D + 3, dtype=torch.float64, device=b.device)     # [sums (D + 2) | M]
            bf = self._bufs = dict(v=torch.zeros(D, dtype=torch.float64, device=b.device), red=red, sums=red[:D + 2],
                                   M=red[D + 2:], w=torch.zeros((b.T, b.N), dtype=torch.float32, device=b.device))
        return bf

    def _dual_pass(self, b, x, count, w_out=None):
        """(g, gradient) at x = [eta, v]: one delta_max + dual_sums pass, reduced over the ranks."""
        import torch
        from .. import ops
        bf = self._buffers(b)
        active = self._comm is not None and self._comm.active
        bf["v"].copy_(torch.from_numpy(np.ascontiguousarray(x[1:], dtype=np.float64)))
        ops.reps_delta_max(b, bf["v"], bf["M"])
        if active:
            self._comm.all_reduce_mixed(bf["M"], 0)
        ops.reps_dual_sums(b, bf["v"], float(x[0]), bf["M"], bf["sums"], w_out)
        if active:
            self._comm.all_reduce_mixed(bf["sums"], bf["sums"].numel())
        h = bf["red"].cpu().numpy()
        self.n_dual_evals += 1
        return dual_from_sums(x[0], h[-1], h[:-1], count, self.epsilon, self.L2_reg_dual)

    def _minimize(self, **kw):
        if self.optimizer is scipy.optimize.fmin_l_bfgs_b:
            kw.pop("disp", None)
        return self.optimizer(**kw)

    def optimize_policy(self, itr, samples_data):
        b = _lane_batch(samples_data)
        count = float(b.count.cpu()[0]) if b.masked else float(b.B_global)
        self.n_dual_evals = self.n_policy_evals = 0

        def cached(fn):
            memo = {}

            def both(x):
                x = np.asarray(x, dtype=np.float64)
                key = x.tobytes()
                if key not in memo:
                    memo.clear()
                    memo[key] = fn(x)
                return memo[key]
            return (lambda x: both(x)[0]), (lambda x: both(x)[1])

        #################
        # Optimize dual #
        #################
        eval_dual, eval_dual_grad = cached(lambda x: self._dual_pass(b, x, count))
        x0 = np.hstack([self.param_eta, self.param_v])
        bounds = [(-np.inf, np.inf) for _ in x0]
        bounds[0] = (0., np.inf)
        logger.log('optimizing dual')
        eta_before = x0[0]
        dual_before = eval_dual(x0)
        params_ast, _, _ = self._minimize(func=eval_dual, x0=x0, fprime=eval_dual_grad, bounds=bounds,
                                          maxiter=self.max_opt_itr, disp=0)
        # the pass at the solution also writes the policy-step weights
        bf = self._buffers(b)
        dual_after, _ = self._dual_pass(b, params_ast, count, w_out=bf["w"])
        self.param_eta = params_ast[0]
        self.param_v = params_ast[1:]

        ###################
        # Optimize policy #
        ###################
        view = copy.copy(b)                   # the sample buffers of b, with the weights as advantages
        view.adv = bf["w"]
        self._view_version += 1
        view.version = self._view_version
        policy, obj, l2 = self.policy, self._objective, self.L2_reg_loss
        reg = regularizable_slices(policy)
        current = [None]

        def set_params(x):
            key = x.tobytes()
            if current[0] != key:
                policy.set_param_values(x, trainable=True)
                current[0] = key

        def loss_pass(x):
            set_params(x)
            loss, g = obj.f_opt(view)
            self.n_policy_evals += 1
            if l2:
                for s in reg:
                    p = x[s]
                    loss += l2 * np.mean(np.square(p)) / len(reg)
                    g[s] += l2 * 2.0 * p / (p.size * len(reg))
            return loss, g

        eval_loss, eval_loss_grad = cached(loss_pass)
        cur_params = policy.get_param_values(trainable=True)
        loss_before = eval_loss(cur_params)
        logger.log('optimizing policy')
        params_ast, _, _ = self._minimize(func=eval_loss, x0=cur_params, fprime=eval_loss_grad, disp=0,
                                          maxiter=self.max_opt_itr)
        loss_after = eval_loss(params_ast)
        set_params(np.asarray(params_ast, dtype=np.float64))
        kl = obj.eval_lazy(view)              # b200rl_loss_kl at the final parameters, read back at dump time

        logger.log('eta %f -> %f' % (eta_before, self.param_eta))
        logger.record_tabular("LossBefore", loss_before)
        logger.record_tabular("LossAfter", loss_after)
        logger.record_tabular('DualBefore', dual_before)
        logger.record_tabular('DualAfter', dual_after)
        logger.record_tabular('MeanKL', lambda: kl[1])

    def get_itr_snapshot(self, itr, samples_data):
        return dict(
            itr=itr,
            policy=self.policy,
            baseline=self.baseline,
            env=self.env,
        )
