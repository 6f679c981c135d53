"""VPG (rllab/algos/vpg.py:11-138): surrogate -mean(logp*adv), one full-batch Adam step per iteration.

With an LbfgsOptimizer (ERWR, erwr.py) scipy's L-BFGS runs on the host and each of its function evaluations is one
gradient pass on the GPU (algos/policy_objective.py)."""
from .. import _lib as L
from ..misc import logger
from ..optimizers.first_order_optimizer import FirstOrderOptimizer
from ..optimizers.lbfgs_optimizer import LbfgsOptimizer
from .batch_polopt import BatchPolopt
from .policy_objective import PolicyObjective


class VPG(BatchPolopt):
    def __init__(self, env, policy, baseline, optimizer=None, optimizer_args=None, **kwargs):
        if optimizer is None:
            default_args = dict(batch_size=None, max_epochs=1)
            optimizer_args = default_args if optimizer_args is None else dict(default_args, **optimizer_args)
            optimizer = FirstOrderOptimizer(**optimizer_args)
        self.optimizer = optimizer
        self.opt_info = None
        self._objective = None
        super(VPG, self).__init__(env=env, policy=policy, baseline=baseline, **kwargs)

    def init_opt(self):
        comm = getattr(self.sampler, "comm", None)
        if isinstance(self.optimizer, LbfgsOptimizer):
            o = self._objective = PolicyObjective(self.policy, L.LOSS_VPG, comm)
            self.optimizer.update_opt(loss=o.f_loss, target=self.policy, inputs=None, f_opt=o.f_opt)
            self.opt_info = dict(f_kl=o.kl_stats)
            return
        self.optimizer.update_opt(L.LOSS_VPG, target=self.policy, inputs=None, comm=comm)
        self.opt_info = dict(f_kl=self.optimizer.kl_stats)

    def optimize_policy(self, itr, samples_data):
        logger.log("optimizing policy")
        # same quantities as vpg.py:110-130; the triples are read back lazily (resolved by logger.dump_tabular) so that
        # the gradient pass, the Adam step and the evaluation pass are all queued before the host blocks
        if self._objective is not None:
            before = self._objective.eval_lazy(samples_data)
            self.optimizer.optimize([samples_data])
            after = self._objective.eval_lazy(samples_data)
        else:
            before = self.optimizer.eval_lazy(samples_data, want_grad=True)
            self.optimizer.optimize(samples_data)
            after = self.optimizer.eval_lazy(samples_data)
        logger.record_tabular("LossBefore", lambda: before[0])
        logger.record_tabular("LossAfter", lambda: after[0])
        logger.record_tabular('MeanKL', lambda: after[1])
        logger.record_tabular('MaxKL', lambda: after[2])

    def get_itr_snapshot(self, itr, samples_data):
        return dict(itr=itr, policy=self.policy, baseline=self.baseline, env=self.env)
