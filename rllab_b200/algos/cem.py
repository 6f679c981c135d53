"""CEM (rllab/algos/cem.py): cross-entropy policy search with the whole population rolled out on the GPU.

An iteration samples parameter rows theta_m ~ N(cur_mean, sample_std^2), runs n_evals episodes of every member's own
policy (b200rl_population_rollout: one warp per member), and refits cur_mean / cur_std to the best best_frac of the
members.  Everything of an iteration stays on the device: the rows, the episodes, the top-k selection
(b200rl_population_topk), the regenerated elite rows and their mean / std (b200rl_rows_mean_std).  The host reads back
the per-member statistics the table needs (and, with batch_size, the episode lengths that decide the population size);
cur_mean / cur_std are copied to the host only for the snapshot.

Multi-GPU: the members are sharded contiguously over the ranks (Comm.shard); fitness, returns and lengths are gathered
through the Comm; every rank then selects the same elites and regenerates their rows locally (a row is a pure function of
(seed, itr, member, cur_mean, cur_std)), so no parameter row crosses GPUs and cur_mean / cur_std / the policy are
bit-identical on every rank.  That requires one Philox key on all ranks: train() agrees it over the ranks (the largest
of the ranks' keys) before the first iteration, whether it was given or drawn.

Deliberate deviations from the reference:
  * theta_m, the action noise and the reset noise come from the counter-based Philox streams (2, 0 and 1) keyed by one
    seed drawn from np.random when train() starts, not from np.random in program order (the lane sampler's policy).
  * Ties in fitness go to the lower member index (numpy's default argsort is not stable).
  * plot=True raises.
"""
import numpy as np

from .. import _lib as L
from ..core.serializable import Serializable
from ..envs.base import Env
from ..misc import logger
from .base import RLAlgorithm


class CEM(RLAlgorithm, Serializable):
    def __init__(
            self,
            env,
            policy,
            n_itr=500,
            max_path_length=500,
            discount=0.99,
            init_std=1.,
            n_samples=100,
            batch_size=None,
            best_frac=0.05,
            extra_std=1.,
            extra_decay_time=100,
            plot=False,
            n_evals=1,
            **kwargs
    ):
        """Arguments as in the reference (rllab/algos/cem.py), in this project's terms:

        env, policy        normalize(<rllab_b200 env>) and a GaussianMLPPolicy; cur_mean starts at the policy's parameters.
        n_itr              iterations to run.
        max_path_length    cap on every episode; an episode also ends when the env reports done.
        discount           discount of the per-episode return G that the fitness is built from.
        init_std           cur_std of iteration 0 (a scalar, broadcast to every parameter).
        n_samples          members per iteration; with batch_size it only sets the number of elites.
        batch_size         None: exactly n_samples members.  Otherwise the population is the shortest prefix of members
                           whose LAST episode's lengths add up to batch_size.
        best_frac          elites = max(1, int(n_samples * best_frac)) best members (at most the population).
        extra_std          std added in quadrature to cur_std, decaying linearly to 0 ...
        extra_decay_time   ... over this many iterations.
        plot               must be False: plotting is not supported.
        n_evals            episodes per member; fitness = mean(G) - stderr(G) over them.
        Extra keywords: seed (Philox key; default drawn from np.random in train() and agreed over the ranks),
        comm (rllab_b200.parallel.Comm; default the process-wide one).
        """
        Serializable.quick_init(self, locals())
        if plot:
            raise NotImplementedError("plotting is outside the B200 hot path")
        from .. import ops
        if ops.is_categorical(getattr(policy, "dims", None)) or ops.is_gru(getattr(policy, "dims", None)):
            raise NotImplementedError("CEM's population rollout is built for GaussianMLPPolicy only")
        self.env = env
        self.policy = policy
        self.batch_size = batch_size
        self.plot = plot
        self.extra_decay_time = extra_decay_time
        self.extra_std = extra_std
        self.best_frac = best_frac
        self.n_samples = n_samples
        self.init_std = init_std
        self.discount = discount
        self.max_path_length = max_path_length
        self.n_itr = n_itr
        self.n_evals = n_evals
        self.seed = kwargs.get("seed")
        self.comm = kwargs.get("comm")
        self.cur_mean = None          # float64 device tensors [P] after train()
        self.cur_std = None
        self.last = None              # host view of the last iteration's population (tests, diagnostics)

    # ---- one population: rows, rollout, and the per-member values every rank needs
    def _evaluate(self, itr, start, count, extra_var):
        """Members start .. start+count-1 (global indices), sharded over the ranks.  Returns the device array [count][W],
        gathered over the ranks: f, undiscounted-return statistic, mean action std, the n_evals episode lengths, then
        the first and the last observation of every episode if the env's diagnostics need them."""
        import torch
        from .. import ops
        pol, E = self.policy, int(self.n_evals)
        n_loc, off = self.comm.shard(count)
        m0 = start + off
        res = ops.PopulationResult(n_loc, E, pol.obs_dim, self._dev, keep_obs=self._want_obs)
        if n_loc > 0:
            rows = torch.empty((n_loc, pol.n_params), dtype=torch.float64, device=self._dev)
            ops.population_sample(self.cur_mean, self.cur_std, extra_var, self.seed, itr, rows, member0=m0)
            ops.population_rollout(self.env_kind, rows, pol.h1, pol.h2, pol.min_std, E, int(self.max_path_length),
                                   float(self.discount), self.seed, itr, m0 * E, res)
        cols = [res.member, res.len.double()]
        if self._want_obs:
            cols += [res.obs_first.reshape(n_loc, E * pol.obs_dim).double(),
                     res.obs_last.reshape(n_loc, E * pol.obs_dim).double()]
        loc = torch.cat(cols, dim=1)
        if self.comm.active:
            glob = torch.zeros((count, loc.shape[1]), dtype=torch.float64, device=self._dev)
            glob[off:off + n_loc] = loc
            self.comm.all_reduce_sum(glob.view(-1))    # every entry has one non-zero term: the sum is exact
        else:
            glob = loc
        return glob

    def _population(self, itr, extra_var):
        """The population of iteration itr: n_samples members, or (batch_size) the shortest prefix of members whose last
        episodes' lengths add up to batch_size (cem.py:51 counts the last path of each member), evaluated in waves."""
        import torch
        if self.batch_size is None:
            glob = self._evaluate(itr, 0, int(self.n_samples), extra_var)
            return glob, glob.cpu().numpy()
        E = int(self.n_evals)
        wave = max(1, -(-int(self.batch_size) // int(self.max_path_length)))
        parts, hosts, start, total = [], [], 0, 0
        while True:
            glob = self._evaluate(itr, start, wave, extra_var)
            host = glob.cpu().numpy()
            csum = total + np.cumsum(host[:, 3 + E - 1])
            hit = np.nonzero(csum >= self.batch_size)[0]
            if len(hit):
                n = int(hit[0]) + 1
                parts.append(glob[:n])
                hosts.append(host[:n])
                break
            parts.append(glob)
            hosts.append(host)
            total = float(csum[-1])
            start += wave
            wave *= 2
        return torch.cat(parts, dim=0), np.concatenate(hosts, axis=0)

    def train(self):
        import torch
        from .. import ops
        from ..parallel import default_comm
        env, pol = self.env, self.policy
        if not hasattr(env, "wrapped_env") or not hasattr(env, "env_kind"):
            raise TypeError("CEM drives normalize(<rllab_b200 env>) (the NormalizedEnv action map is fused into the "
                            "kernels)")
        if not torch.cuda.is_available():
            raise L.B200RLError("CEM needs a CUDA device (no CPU fallback)")
        if self.comm is None:
            self.comm = default_comm()
        self.env_kind = env.env_kind
        self._dev = pol.theta64.device
        if self.seed is None:
            self.seed = int(np.random.randint(0, 2 ** 31 - 1))
        if self.comm.active:
            # every rank regenerates the elite rows of members other ranks evaluated, so all ranks must hold the same
            # Philox key: take the largest of the ranks' keys (exact in float64: keys are < 2^32)
            key = torch.tensor([float(int(self.seed) & 0xFFFFFFFF)], dtype=torch.float64, device=self._dev)
            self.comm.all_reduce_mixed(key, 0)
            self.seed = int(key.item())
        self._want_obs = type(env.wrapped_env).log_diagnostics is not Env.log_diagnostics
        P, O, E = pol.n_params, pol.obs_dim, int(self.n_evals)
        self.cur_mean = pol.theta64.clone()
        self.cur_std = torch.full((P,), float(self.init_std), dtype=torch.float64, device=self._dev)
        n_best = max(1, int(self.n_samples * self.best_frac))
        for itr in range(self.n_itr):
            with logger.prefix('itr #%d | ' % itr):
                extra_var_mult = max(1.0 - itr / self.extra_decay_time, 0)
                extra_var = float(np.square(self.extra_std) * extra_var_mult)
                glob, host = self._population(itr, extra_var)
                M = host.shape[0]
                k = min(n_best, M)
                f = glob[:, 0].contiguous()
                idx = torch.empty(k, dtype=torch.int64, device=self._dev)
                ops.population_topk(f, k, idx)
                best = torch.empty((k, P), dtype=torch.float64, device=self._dev)
                ops.population_sample(self.cur_mean, self.cur_std, extra_var, self.seed, itr, best, members=idx)
                new_mean = torch.empty(P, dtype=torch.float64, device=self._dev)
                new_std = torch.empty(P, dtype=torch.float64, device=self._dev)
                ops.rows_mean_std(best, new_mean, new_std)
                self.cur_mean, self.cur_std = new_mean, new_std
                std_mean = torch.empty(1, dtype=torch.float64, device=self._dev)
                ops.rows_mean_std(new_std.view(P, 1), std_mean, torch.empty_like(std_mean))
                pol.set_param_values_device(best[0])
                lens = host[:, 3:3 + E]
                ustat = host[:, 1]
                self.last = dict(M=M, k=k, f=host[:, 0].copy(), ustat=ustat.copy(), mstd=host[:, 2].copy(),
                                 lens=lens.copy(), idx=idx)
                logger.record_tabular('Iteration', itr)
                logger.record_tabular('CurStdMean', float(std_mean.item()))
                logger.record_tabular('AverageReturn', np.mean(ustat))
                logger.record_tabular('StdReturn', np.std(ustat))
                logger.record_tabular('MaxReturn', np.max(ustat))
                logger.record_tabular('MinReturn', np.min(ustat))
                logger.record_tabular('AverageDiscountedReturn', np.mean(host[:, 0]))
                logger.record_tabular('NumTrajs', M)
                logger.record_tabular('AvgTrajLen', np.mean(lens))
                if self._want_obs:
                    first = host[:, 3 + E:3 + E + E * O].reshape(M * E, O)
                    last = host[:, 3 + E + E * O:].reshape(M * E, O)
                    env.log_diagnostics([dict(observations=np.stack([a, b])) for a, b in zip(first, last)])
                # GaussianMLPPolicy.log_diagnostics over every step of every episode: each member's (state-independent)
                # std weighs with the number of steps its episodes ran
                logger.record_tabular('AveragePolicyStd', float(np.sum(host[:, 2] * lens.sum(axis=1)) / lens.sum()))
                if logger.snapshot_enabled():
                    logger.save_itr_params(itr, dict(itr=itr, policy=pol, env=env,
                                                     cur_mean=self.cur_mean.cpu().numpy(),
                                                     cur_std=self.cur_std.cpu().numpy()))
                logger.dump_tabular(with_prefix=False)
