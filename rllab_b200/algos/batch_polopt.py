"""BatchPolopt (rllab/algos/batch_polopt.py:37-165): same constructor, same train() loop; the default sampler is the
device LaneSampler (the reference's BatchSampler drives a CPU process pool)."""
import numpy as np

from ..misc import logger
from ..sampler.lane_sampler import LaneSampler
from .base import RLAlgorithm


class BatchPolopt(RLAlgorithm):
    def __init__(self, env, policy, baseline, scope=None, n_itr=500, start_itr=0, batch_size=5000,
                 max_path_length=500, discount=0.99, gae_lambda=1, plot=False, pause_for_plot=False, center_adv=True,
                 positive_adv=False, store_paths=False, whole_paths=True, sampler_cls=None, sampler_args=None,
                 **kwargs):
        self.env = env
        self.policy = policy
        self.baseline = baseline
        self.scope = scope
        self.n_itr = n_itr
        self.current_itr = start_itr
        self.batch_size = batch_size
        self.max_path_length = max_path_length
        self.discount = discount
        self.gae_lambda = gae_lambda
        self.plot = plot
        self.pause_for_plot = pause_for_plot
        self.center_adv = center_adv
        self.positive_adv = positive_adv
        self.store_paths = store_paths
        self.whole_paths = whole_paths
        if plot:
            raise NotImplementedError("plotting is outside the B200 hot path")
        if sampler_cls is None:
            sampler_cls = LaneSampler
        if sampler_args is None:
            sampler_args = dict()
        self._sampler_cls, self._sampler_args = sampler_cls, dict(sampler_args)
        self.sampler = sampler_cls(self, **sampler_args)

    def start_worker(self):
        self.sampler.start_worker()

    def shutdown_worker(self):
        self.sampler.shutdown_worker()

    def train(self):
        self.start_worker()
        self.init_opt()
        for itr in range(self.current_itr, self.n_itr):
            with logger.prefix('itr #%d | ' % itr):
                self.train_itr(itr)
        self.shutdown_worker()

    def train_itr(self, itr):
        """One iteration of batch_polopt.py:118-139."""
        paths = self.sampler.obtain_samples(itr)
        samples_data = self.sampler.process_samples(itr, paths)
        self.log_diagnostics(paths)
        self.optimize_policy(itr, samples_data)
        logger.log("saving snapshot...")
        params = self.get_itr_snapshot(itr, samples_data)
        self.current_itr = itr + 1
        params["algo"] = self
        if self.store_paths:
            params["paths"] = samples_data["paths"]
        logger.save_itr_params(itr, params)
        logger.log("saved")
        logger.dump_tabular(with_prefix=False)
        return samples_data

    def log_diagnostics(self, paths):
        # AveragePolicyStd (gaussian_mlp_policy.py:155-157) from the device copy of log_std: the state-independent
        # log_std makes mean(exp(log_stds)) over samples equal to mean(exp(log_std)) over action dims.
        b = getattr(paths, "lane_batch", None)
        if b is not None:
            from .. import ops
            if not b.categorical:                     # CategoricalMLPPolicy logs no diagnostics (policies/base.py)
                p_ls = ops.PendingHost(b.log_std)          # read back when the table is dumped
                logger.record_tabular('AveragePolicyStd',
                                      lambda: float(np.mean(np.exp(p_ls.get().astype(np.float64)))))
            if self.store_paths:
                self.env.log_diagnostics(paths.to_paths())
        else:
            self.env.log_diagnostics(paths)
            self.policy.log_diagnostics(paths)
            self.baseline.log_diagnostics(paths)

    def update_plot(self):
        """batch_polopt.py:163-165: only ever called when plot=True, which the constructor rejects."""
        if self.plot:
            raise NotImplementedError("plotting is outside the B200 hot path")

    def init_opt(self):
        raise NotImplementedError

    def get_itr_snapshot(self, itr, samples_data):
        raise NotImplementedError

    def optimize_policy(self, itr, samples_data):
        raise NotImplementedError

    # snapshots pickle `algo` (batch_polopt.py:126, logger.py:216-232); resuming = unpickle + train()
    # (scripts/run_experiment_lite.py:111-115): device buffers are dropped and the sampler is rebuilt.
    def __getstate__(self):
        d = dict(self.__dict__)
        d["sampler"] = None
        args = dict(d["_sampler_args"])
        args.pop("comm", None)
        d["_sampler_args"] = args
        return d

    def __setstate__(self, d):
        self.__dict__.update(d)
        self.sampler = self._sampler_cls(self, **self._sampler_args)
