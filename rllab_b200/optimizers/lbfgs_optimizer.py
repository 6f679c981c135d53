"""LbfgsOptimizer (rllab/optimizers/lbfgs_optimizer.py:8-81): unconstrained L-BFGS with scipy's fmin_l_bfgs_b on the host.

update_opt takes callables instead of Theano expressions:
  loss     f_loss(*inputs) -> float, evaluated at the target's current parameters
  f_opt    f_opt(*inputs) -> (loss, flat gradient float64), evaluated at the target's current parameters
The device regressor (rllab_b200/regressors/gaussian_mlp_regressor.py) passes callables that run one CUDA pass each and
read back the loss and the gradient; scipy works on the host copy of theta.

termination: scipy's (warnflag, task) of the last optimize(), e.g. (0, 'CONVERGENCE: ...') or (1, 'STOP: TOTAL NO. of
ITERATIONS ...'): with float32-grade losses, an early 'ABNORMAL_TERMINATION_IN_LNSRCH' shows the line search ran out
of resolution.
"""
import time

import scipy.optimize

from ..misc import logger


class LbfgsOptimizer(object):
    """Performs unconstrained optimization via L-BFGS."""

    def __init__(self, max_opt_itr=20, callback=None):
        self._max_opt_itr = max_opt_itr
        self._opt_fun = None
        self._target = None
        self._callback = callback
        self.termination = None

    def update_opt(self, loss, target, inputs=None, extra_inputs=None, gradients=None, f_opt=None, *args, **kwargs):
        """
        :param loss: callable(*inputs) -> float
        :param target: object with get_param_values / set_param_values(trainable=True)
        :param f_opt: callable(*inputs) -> (loss, flat_grad)
        """
        if f_opt is None:
            raise TypeError("update_opt needs f_opt=callable(*inputs) -> (loss, flat_grad)")
        self._target = target
        self._opt_fun = dict(f_loss=loss, f_opt=f_opt)

    def __getstate__(self):
        # snapshots drop the bound callables and target: the owner binds them again (VPG.init_opt on resume)
        d = dict(self.__dict__)
        d.update(_opt_fun=None, _target=None)
        return d

    def loss(self, inputs, extra_inputs=None):
        if extra_inputs is None:
            extra_inputs = list()
        return self._opt_fun["f_loss"](*(list(inputs) + list(extra_inputs)))

    def optimize(self, inputs, extra_inputs=None):
        f_opt = self._opt_fun["f_opt"]

        if extra_inputs is None:
            extra_inputs = list()

        def f_opt_wrapper(flat_params):
            self._target.set_param_values(flat_params, trainable=True)
            return f_opt(*inputs)

        itr = [0]
        start_time = time.time()

        if self._callback:
            def opt_callback(params):
                loss = self._opt_fun["f_loss"](*(list(inputs) + list(extra_inputs)))
                elapsed = time.time() - start_time
                self._callback(dict(
                    loss=loss,
                    params=params,
                    itr=itr[0],
                    elapsed=elapsed,
                ))
                itr[0] += 1
        else:
            opt_callback = None

        _, _, info = scipy.optimize.fmin_l_bfgs_b(
            func=f_opt_wrapper, x0=self._target.get_param_values(trainable=True),
            maxiter=self._max_opt_itr, callback=opt_callback,
        )
        self.termination = (int(info["warnflag"]), str(info["task"]), int(info["funcalls"]))
        logger.log("lbfgs: %s after %d evaluations" % (self.termination[1], self.termination[2]))
