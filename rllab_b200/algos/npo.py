"""NPO (rllab/algos/npo.py:10-132): surrogate -mean(lr*adv) under mean KL <= step_size.

The default optimizer is the reference's, PenaltyLbfgsOptimizer (npo.py:23-27): that is PPO (ppo.py).  Its function
evaluations run the gradient pass of surrogate + penalty * mean KL on the GPU (algos/policy_objective.py); scipy's
L-BFGS runs on the host.  With a ConjugateGradientOptimizer (TRPO, TNPG) every vector stays on the GPU.
"""
from .. import _lib as L
from ..misc import logger
from ..optimizers.penalty_lbfgs_optimizer import PenaltyLbfgsOptimizer
from .batch_polopt import BatchPolopt
from .policy_objective import PolicyObjective


class NPO(BatchPolopt):
    def __init__(self, optimizer=None, optimizer_args=None, step_size=0.01, truncate_local_is_ratio=None, **kwargs):
        if truncate_local_is_ratio is not None:
            raise NotImplementedError("truncate_local_is_ratio (npo.py:75-76, default off) is not built")
        if optimizer is None:
            if optimizer_args is None:
                optimizer_args = dict()
            optimizer = PenaltyLbfgsOptimizer(**optimizer_args)
        self.optimizer = optimizer
        self.step_size = step_size
        self.truncate_local_is_ratio = truncate_local_is_ratio
        self._objective = None
        super(NPO, self).__init__(**kwargs)

    def init_opt(self):
        comm = getattr(self.sampler, "comm", None)
        if isinstance(self.optimizer, PenaltyLbfgsOptimizer):
            o = self._objective = PolicyObjective(self.policy, L.LOSS_TRPO, comm)
            self.optimizer.update_opt(loss=o.f_loss, target=self.policy, leq_constraint=(o.f_constraint, self.step_size),
                                      inputs=None, constraint_name="mean_kl", f_opt=o.f_opt,
                                      f_penalized_loss=o.f_penalized_loss)
        else:
            self.optimizer.update_opt(loss=L.LOSS_TRPO, target=self.policy, leq_constraint=("mean_kl", self.step_size),
                                      inputs=None, constraint_name="mean_kl", comm=comm)
        return dict()

    def optimize_policy(self, itr, samples_data):
        # npo.py:102-123; lazily read triples (see VPG.optimize_policy): the first host wait is at the line search
        if self._objective is not None:
            before = self._objective.eval_lazy(samples_data)
            self.optimizer.optimize([samples_data])
            after = self._objective.eval_lazy(samples_data)
        else:
            before = self.optimizer.eval_lazy(samples_data)
            self.optimizer.optimize(samples_data)
            after = self.optimizer.eval_lazy(samples_data)
        logger.record_tabular('LossBefore', lambda: before[0])
        logger.record_tabular('LossAfter', lambda: after[0])
        logger.record_tabular('MeanKLBefore', lambda: before[1])
        logger.record_tabular('MeanKL', lambda: after[1])
        logger.record_tabular('dLoss', lambda: before[0] - after[0])
        return dict()

    def get_itr_snapshot(self, itr, samples_data):
        return dict(itr=itr, policy=self.policy, baseline=self.baseline, env=self.env)
