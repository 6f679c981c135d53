"""PenaltyLbfgsOptimizer (rllab/optimizers/penalty_lbfgs_optimizer.py:10-150): constrained optimization by penalised
L-BFGS with an adaptive penalty, scipy's fmin_l_bfgs_b on the host.

update_opt takes callables instead of Theano expressions (penalty is the last positional argument):
  loss                 f_loss(*inputs) -> float
  leq_constraint       (f_constraint(*inputs) -> float, max value)
  f_opt                f_opt(*inputs, penalty) -> (penalised loss, flat gradient float64)
  f_penalized_loss     f_penalized_loss(*inputs, penalty) -> (penalised loss, loss, constraint)
all evaluated at the target's current parameters.  optimize() restates :82-150 line by line, quirks included: opt_params
starts as cur_params, so the `opt_params is None` branch never fires, and f_penalized_loss is evaluated at the
parameters scipy evaluated last, which need not be the ones it returns.

tried_penalties / terminations: the penalties tried by the last optimize() and scipy's (warnflag, task, evaluations)
for each of them.
"""
import numpy as np
import scipy.optimize

from ..misc import logger


class PenaltyLbfgsOptimizer(object):
    """
    Performs constrained optimization via penalized L-BFGS. The penalty term is adaptively adjusted to make sure that
    the constraint is satisfied.
    """

    def __init__(
            self,
            max_opt_itr=20,
            initial_penalty=1.0,
            min_penalty=1e-2,
            max_penalty=1e6,
            increase_penalty_factor=2,
            decrease_penalty_factor=0.5,
            max_penalty_itr=10,
            adapt_penalty=True):
        self._max_opt_itr = max_opt_itr
        self._penalty = initial_penalty
        self._initial_penalty = initial_penalty
        self._min_penalty = min_penalty
        self._max_penalty = max_penalty
        self._increase_penalty_factor = increase_penalty_factor
        self._decrease_penalty_factor = decrease_penalty_factor
        self._max_penalty_itr = max_penalty_itr
        self._adapt_penalty = adapt_penalty

        self._opt_fun = None
        self._target = None
        self._max_constraint_val = None
        self._constraint_name = None
        self.tried_penalties = []
        self.terminations = []

    def update_opt(self, loss, target, leq_constraint, inputs=None, constraint_name="constraint", f_opt=None,
                   f_penalized_loss=None, *args, **kwargs):
        if f_opt is None or f_penalized_loss is None:
            raise TypeError("update_opt needs f_opt=callable(*inputs, penalty) -> (penalized loss, flat_grad) and "
                            "f_penalized_loss=callable(*inputs, penalty) -> (penalized loss, loss, constraint)")
        constraint_term, constraint_value = leq_constraint
        self._target = target
        self._max_constraint_val = constraint_value
        self._constraint_name = constraint_name
        self._opt_fun = dict(f_loss=loss, f_constraint=constraint_term, f_penalized_loss=f_penalized_loss, f_opt=f_opt)

    def __getstate__(self):
        # snapshots keep the carried penalty and drop the bound callables and target: the owner binds them again
        # (NPO.init_opt on resume)
        d = dict(self.__dict__)
        d.update(_opt_fun=None, _target=None)
        return d

    def loss(self, inputs):
        return self._opt_fun["f_loss"](*inputs)

    def constraint_val(self, inputs):
        return self._opt_fun["f_constraint"](*inputs)

    def optimize(self, inputs):

        inputs = tuple(inputs)

        try_penalty = np.clip(
            self._penalty, self._min_penalty, self._max_penalty)

        penalty_scale_factor = None
        f_opt = self._opt_fun["f_opt"]
        f_penalized_loss = self._opt_fun["f_penalized_loss"]

        def gen_f_opt(penalty):
            def f(flat_params):
                self._target.set_param_values(flat_params, trainable=True)
                return f_opt(*(inputs + (penalty,)))
            return f

        cur_params = self._target.get_param_values(trainable=True).astype('float64')
        opt_params = cur_params
        self.tried_penalties = []
        self.terminations = []

        for penalty_itr in range(self._max_penalty_itr):
            logger.log('trying penalty=%.3f...' % try_penalty)

            itr_opt_params, _, info = scipy.optimize.fmin_l_bfgs_b(
                func=gen_f_opt(try_penalty), x0=cur_params,
                maxiter=self._max_opt_itr
            )
            self.tried_penalties.append(float(try_penalty))
            self.terminations.append((int(info["warnflag"]), str(info["task"]), int(info["funcalls"])))

            _, try_loss, try_constraint_val = f_penalized_loss(*(inputs + (try_penalty,)))

            logger.log('penalty %f => loss %f, %s %f (%s)' %
                       (try_penalty, try_loss, self._constraint_name, try_constraint_val, info["task"]))

            # Either constraint satisfied, or we are at the last iteration already and no alternative parameter
            # satisfies the constraint
            if try_constraint_val < self._max_constraint_val or \
                    (penalty_itr == self._max_penalty_itr - 1 and opt_params is None):
                opt_params = itr_opt_params

            if not self._adapt_penalty:
                break

            # Decide scale factor on the first iteration, or if constraint violation yields numerical error
            if penalty_scale_factor is None or np.isnan(try_constraint_val):
                # Increase penalty if constraint violated, or if constraint term is NAN
                if try_constraint_val > self._max_constraint_val or np.isnan(try_constraint_val):
                    penalty_scale_factor = self._increase_penalty_factor
                else:
                    # Otherwise (i.e. constraint satisfied), shrink penalty
                    penalty_scale_factor = self._decrease_penalty_factor
                    opt_params = itr_opt_params
            else:
                if penalty_scale_factor > 1 and \
                        try_constraint_val <= self._max_constraint_val:
                    break
                elif penalty_scale_factor < 1 and \
                        try_constraint_val >= self._max_constraint_val:
                    break

            # check if the penalty was already at the bounds. Otherwise update it. Here penalty_scale_fact is never None
            if try_penalty >= self._max_penalty and penalty_scale_factor > 1:
                logger.log('_max_penalty has already been tried!')
                self._penalty = try_penalty
                break
            elif try_penalty <= self._min_penalty and penalty_scale_factor < 1:
                logger.log('_min_penalty has already been tried!')
                self._penalty = try_penalty
                break
            else:
                try_penalty *= penalty_scale_factor
                try_penalty = np.clip(try_penalty, self._min_penalty, self._max_penalty)
                self._penalty = try_penalty

        self._target.set_param_values(opt_params, trainable=True)
