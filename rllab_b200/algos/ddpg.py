"""DDPG (rllab/algos/ddpg.py): deep deterministic policy gradient with the whole train() loop on the GPU.

Each epoch is one b200rl_ddpg_train launch (rllab_b200/csrc/ddpg.cu): one CTA runs epoch_length steps of the loop --
exploration, env step, replay pool write and n_updates_per_sample do_training calls -- with the networks, Adam moments
and targets in shared memory.  The host then reads the epoch's statistics, runs `evaluate` (noise-free paths of the
current policy from b200rl_rollout_deterministic, N = ceil(eval_samples / max_path_length) lanes of max_path_length
steps, whole paths only, as the lane sampler counts samples) and dumps the tabular.  ops.DdpgRuns runs several
independent runs in one launch.

Deliberate deviations from the reference:
  * resets, exploration noise and minibatch indices come from counter-based Philox streams (layout in include/b200rl.h)
    keyed by `seed`, not from np.random in program order;
  * the replay pool stores observations, actions and scaled rewards in float32;
  * the nets run in float32 with float64 master parameters, Adam moments and targets (f64=True: all float64).
"""
import numpy as np

from .. import _lib as L
from ..misc import logger
from ..spaces import Box
from .base import RLAlgorithm


class DDPG(RLAlgorithm):
    def __init__(self, env, policy, qf, es, batch_size=32, n_epochs=200, epoch_length=1000, min_pool_size=10000,
                 replay_pool_size=1000000, discount=0.99, max_path_length=250, qf_weight_decay=0.,
                 qf_update_method='adam', qf_learning_rate=1e-3, policy_weight_decay=0, policy_update_method='adam',
                 policy_learning_rate=1e-4, eval_samples=10000, soft_target=True, soft_target_tau=0.001,
                 n_updates_per_sample=1, scale_reward=1.0, include_horizon_terminal_transitions=False, plot=False,
                 pause_for_plot=False, seed=None, f64=False, comm=None):
        """Arguments as in the reference.  Extra keywords: seed (Philox key; default drawn from np.random), f64 (the
        float64 parity mode of the kernels), comm (rllab_b200.parallel.Comm; DDPG runs on one GPU)."""
        if plot:
            raise NotImplementedError("DDPG: plot=True is not built")
        if qf_update_method != 'adam' or policy_update_method != 'adam':
            raise NotImplementedError("DDPG: only the 'adam' update method is built")
        if batch_size != L.DDPG_BATCH:
            raise NotImplementedError("DDPG: the kernels are compiled for batch_size=%d" % L.DDPG_BATCH)
        if min_pool_size <= batch_size:
            raise ValueError("DDPG: min_pool_size must exceed batch_size (the reference asserts pool size > batch_size "
                             "at its first minibatch)")
        if comm is not None and getattr(comm, "active", False):
            raise NotImplementedError("DDPG runs on one GPU (an active multi-rank Comm is not supported)")
        if not hasattr(env, "wrapped_env") or not hasattr(env, "env_kind"):
            raise TypeError("DDPG drives normalize(<rllab_b200 env>) (the NormalizedEnv action map, clip to [-1, 1] and "
                            "rescale to the env's bounds, is fused into the kernel)")
        if env.env_kind not in L.ENV_KINDS.values() or \
                not isinstance(env.action_space, Box) or \
                env.env_kind in (L.ENV_SWIMMER, L.ENV_HOPPER, L.ENV_HALF_CHEETAH):
            raise NotImplementedError("DDPG runs the classic-control Box envs (normalize(<rllab_b200 env>)) only")
        if not hasattr(es, "ES_KIND"):
            raise NotImplementedError("DDPG: the exploration strategy must be OUStrategy or GaussianStrategy")
        self.env, self.policy, self.qf, self.es = env, policy, qf, es
        self.batch_size, self.n_epochs, self.epoch_length = batch_size, n_epochs, epoch_length
        self.min_pool_size, self.replay_pool_size, self.discount = min_pool_size, replay_pool_size, discount
        self.max_path_length = max_path_length
        self.qf_weight_decay, self.qf_learning_rate = qf_weight_decay, qf_learning_rate
        self.policy_weight_decay, self.policy_learning_rate = policy_weight_decay, policy_learning_rate
        self.eval_samples, self.soft_target_tau = eval_samples, soft_target_tau
        self.n_updates_per_sample, self.scale_reward = n_updates_per_sample, scale_reward
        self.include_horizon_terminal_transitions = include_horizon_terminal_transitions
        self.plot, self.pause_for_plot = plot, pause_for_plot
        self.seed, self.f64 = seed, f64
        self.qf_loss_averages, self.policy_surr_averages = [], []
        self.q_averages, self.y_averages = [], []   # per-epoch sums here: [sum, sum |.|, count] rows
        self.es_path_returns = []
        self.opt_info = None
        self.runs = None

    def hparams(self):
        from .. import ops
        es = self.es
        return ops.ddpg_hparams(
            n_updates_per_sample=self.n_updates_per_sample, max_path_length=self.max_path_length,
            min_pool_size=self.min_pool_size, replay_pool_size=self.replay_pool_size,
            include_horizon_terminal_transitions=int(bool(self.include_horizon_terminal_transitions)),
            es_kind=es.ES_KIND, discount=self.discount, scale_reward=self.scale_reward,
            soft_target_tau=self.soft_target_tau, qf_weight_decay=self.qf_weight_decay,
            qf_learning_rate=self.qf_learning_rate, policy_weight_decay=self.policy_weight_decay,
            policy_learning_rate=self.policy_learning_rate, ou_mu=getattr(es, "mu", 0.0),
            ou_theta=getattr(es, "theta", 0.0), ou_sigma=getattr(es, "sigma", 0.0),
            gs_max_sigma=getattr(es, "_max_sigma", 0.0), gs_min_sigma=getattr(es, "_min_sigma", 0.0),
            gs_decay_period=getattr(es, "_decay_period", 1.0))

    def init_opt(self):
        import copy
        import torch
        from .. import ops
        if not torch.cuda.is_available():
            raise L.B200RLError("DDPG needs a CUDA device (no CPU fallback)")
        if self.seed is None:
            self.seed = int(np.random.randint(0, 2 ** 31 - 1))
        pp, qp = self.policy.get_param_values(), self.qf.get_param_values()
        th = np.concatenate([pp, qp])
        nets = np.stack([th, np.zeros_like(th), np.zeros_like(th), th])
        self.runs = ops.DdpgRuns(self.env.env_kind, self.policy.obs_dim, self.policy.action_dim, 1, self.hparams(),
                                 nets[None], self.seed, torch.device("cuda", torch.cuda.current_device()),
                                 f64=self.f64, es_cap=self.epoch_length + 1)
        self.opt_info = dict(target_policy=copy.deepcopy(self.policy), target_qf=copy.deepcopy(self.qf))

    def _sync_params(self):
        nets = self.runs.nets[0].cpu().numpy()
        PP = self.policy.n_params
        self.policy.set_param_values(nets[0, :PP])
        self.qf.set_param_values(nets[0, PP:])
        self.opt_info["target_policy"].set_param_values(nets[3, :PP])
        self.opt_info["target_qf"].set_param_values(nets[3, PP:])

    def train(self):
        self.init_opt()
        for epoch in range(self.n_epochs):
            with logger.prefix('epoch #%d | ' % epoch):
                logger.log("Training started")
                self.runs.train(self.epoch_length)
                stats, es = self.runs.take_stats()
                s = stats[0]
                n = int(s[0])
                if n > 0:
                    self.qf_loss_averages.append((s[1], n))
                    self.policy_surr_averages.append((s[2], n))
                    self.q_averages.append((s[3], s[4], n * self.batch_size))
                    self.y_averages.append((s[5], s[6], s[7], n * self.batch_size))
                self.es_path_returns.extend(es[0].tolist())
                self._sync_params()
                logger.log("Training finished")
                if self.runs.host_state()[0].size >= self.min_pool_size:
                    self.evaluate(epoch)
                    params = self.get_epoch_snapshot(epoch)
                    logger.save_itr_params(epoch, params)
                logger.dump_tabular(with_prefix=False)
        self.env.terminate()
        self.policy.terminate()

    def sample_eval_paths(self):
        import torch
        from .. import ops
        from ..sampler.lane_sampler import lanes_to_paths
        T = int(self.max_path_length)
        N = max(1, -(-int(self.eval_samples) // T))
        dev = self.runs.device
        b = ops.LaneBatch(self.policy.obs_dim, self.policy.action_dim, N, T, dev)
        params = torch.as_tensor(self.policy.get_param_values(), dtype=torch.float32, device=dev)
        self._eval_itr = getattr(self, "_eval_itr", 0) + 1
        ops.rollout_deterministic(self.env.env_kind, params, b, T, seed=self.seed, it=0x40000000 + self._eval_itr)
        b.mean.copy_(b.act)      # the deterministic policy's mean is its action; it has no log_std
        b.log_std.zero_()
        paths = lanes_to_paths(b, whole_paths=True)
        for p in paths:
            p["agent_infos"] = dict()
        return paths

    def evaluate(self, epoch, pool=None):
        logger.log("Collecting samples for evaluation")
        paths = self.sample_eval_paths()
        disc = [np.sum(p["rewards"] * self.discount ** np.arange(len(p["rewards"]))) for p in paths]
        returns = [np.sum(p["rewards"]) for p in paths]
        qsum = sum(x[0] for x in self.q_averages)
        qabs = sum(x[1] for x in self.q_averages)
        nq = sum(x[2] for x in self.q_averages)
        ysum = sum(x[0] for x in self.y_averages)
        yabs = sum(x[1] for x in self.y_averages)
        qydiff = sum(x[2] for x in self.y_averages)
        nupd = sum(x[1] for x in self.qf_loss_averages)
        average_action = np.mean(np.square(np.concatenate([p["actions"] for p in paths])))
        logger.record_tabular('Epoch', epoch)
        logger.record_tabular('AverageReturn', np.mean(returns))
        logger.record_tabular('StdReturn', np.std(returns))
        logger.record_tabular('MaxReturn', np.max(returns))
        logger.record_tabular('MinReturn', np.min(returns))
        if len(self.es_path_returns) > 0:
            logger.record_tabular('AverageEsReturn', np.mean(self.es_path_returns))
            logger.record_tabular('StdEsReturn', np.std(self.es_path_returns))
            logger.record_tabular('MaxEsReturn', np.max(self.es_path_returns))
            logger.record_tabular('MinEsReturn', np.min(self.es_path_returns))
        logger.record_tabular('AverageDiscountedReturn', np.mean(disc))
        logger.record_tabular('AverageQLoss', sum(x[0] for x in self.qf_loss_averages) / nupd if nupd else np.nan)
        logger.record_tabular('AveragePolicySurr',
                              sum(x[0] for x in self.policy_surr_averages) / nupd if nupd else np.nan)
        logger.record_tabular('AverageQ', qsum / nq if nq else np.nan)
        logger.record_tabular('AverageAbsQ', qabs / nq if nq else np.nan)
        logger.record_tabular('AverageY', ysum / nq if nq else np.nan)
        logger.record_tabular('AverageAbsY', yabs / nq if nq else np.nan)
        logger.record_tabular('AverageAbsQYDiff', qydiff / nq if nq else np.nan)
        logger.record_tabular('AverageAction', average_action)
        logger.record_tabular('PolicyRegParamNorm', np.linalg.norm(self.policy.get_param_values(regularizable=True)))
        logger.record_tabular('QFunRegParamNorm', np.linalg.norm(self.qf.get_param_values(regularizable=True)))
        self.env.log_diagnostics(paths)
        self.policy.log_diagnostics(paths)
        self.qf_loss_averages, self.policy_surr_averages = [], []
        self.q_averages, self.y_averages = [], []
        self.es_path_returns = []
        self.last_eval_returns = returns

    def get_epoch_snapshot(self, epoch):
        return dict(env=self.env, epoch=epoch, qf=self.qf, policy=self.policy,
                    target_qf=self.opt_info["target_qf"], target_policy=self.opt_info["target_policy"], es=self.es)
