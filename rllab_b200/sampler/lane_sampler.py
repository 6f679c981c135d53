"""LaneSampler: the GPU replacement of BatchSampler + BaseSampler.process_samples
(rllab/algos/batch_polopt.py:9-34, rllab/sampler/base.py:40-182), plugged in through the reference's own
`sampler_cls=` hook (batch_polopt.py:61-62,101-105).

obtain_samples(itr)   one fused CUDA rollout of N lanes x T steps (b200rl_rollout); returns a LanePaths handle --
                      the trajectories stay in HBM; `.to_paths()` materialises the reference's list-of-path-dicts
                      wire format (sampler/utils.py:37-43) on demand.
process_samples(...)  baseline predict + GAE + returns + statistics (b200rl_process_samples), centering
                      (b200rl_center_advantages), then -- after the advantages, as base.py:163-167 -- the baseline
                      fit (b200rl_lfb_gram + b200rl_lfb_solve); records the same tabular keys (base.py:170-180).

Batch geometry: T = max_path_length steps per lane, N = ceil(batch_size / T) lanes in total, sharded contiguously over
ranks.  Every lane runs exactly T steps with auto-reset on `done`.  The path a lane is in when its buffer ends is cut
short by the sampler, not by the env; what happens to it follows the reference's `whole_paths` switch
(batch_polopt.py:30-34):
  whole_paths=True  (default)  only whole paths are returned, as BatchSampler does (and as the vectorized sampler does
                    when it drops its unfinished running_paths, sandbox/rocky/tf/samplers/vectorized_sampler.py): the cut
                    path is dropped -- FLAG_MASKED on its samples, no contribution to advantages, baseline fit, losses,
                    NumTrajs or the return statistics.  The first path of every lane always completes (T =
                    max_path_length), so no lane is empty.
  whole_paths=False the cut path is kept as a truncated path, which is what truncate_paths does to the last path of
                    the batch (parallel_sampler.py:129-155); every (t, lane) cell is then a valid sample.
"""
import numpy as np

from .. import _lib as L
from ..misc import logger
from .base import Sampler


class LanePaths(object):
    """Handle on the device trajectories of one iteration (duck-types the reference's `paths` list lazily)."""

    def __init__(self, batch, whole_paths=True):
        self.lane_batch = batch
        self.whole_paths = whole_paths
        self._paths = None

    def to_paths(self):
        if self._paths is None:
            self._paths = lanes_to_paths(self.lane_batch, self.whole_paths)
        return self._paths

    def __len__(self):
        return len(self.to_paths())

    def __iter__(self):
        return iter(self.to_paths())

    def __getitem__(self, i):
        return self.to_paths()[i]


def lanes_to_paths(batch, whole_paths=True):
    """Device lanes -> list of path dicts {observations (L,O), actions (L,A), rewards (L,), agent_infos{mean,log_std},
    env_infos{}} (+ advantages / returns when process_samples has run), lane-major then time order.  whole_paths: leave
    out the paths cut by the end of the lane buffer (FLAG_CUT on their last sample).  A categorical batch has one-hot
    actions (L,n) and agent_infos{prob}; a recurrent batch whose policy reads the previous action also carries
    agent_infos["prev_action"] (zeros at the first step, then the path's previous raw action)."""
    t = batch.to_numpy()
    O, T, N = t["obs"].shape
    A = t["act"].shape[0]
    adv = batch.adv.cpu().numpy() if batch.processed else None
    ret = batch.ret.cpu().numpy() if batch.processed else None
    ends = (t["flags"] & L.FLAG_END) != 0
    paths = []
    ls = t["log_std"].astype(np.float64).reshape(1, A)
    for n in range(N):
        start = 0
        for e in np.nonzero(ends[:, n])[0]:
            sl = slice(start, e + 1)
            if whole_paths and (t["flags"][e, n] & L.FLAG_CUT):
                start = e + 1
                continue
            p = dict(
                observations=t["obs"][:, sl, n].T.astype(np.float64),
                actions=t["act"][:, sl, n].T.astype(np.float64),
                rewards=t["rew"][sl, n].astype(np.float64),
                agent_infos=(dict(prob=t["mean"][:, sl, n].T.astype(np.float64)) if batch.categorical else
                             dict(mean=t["mean"][:, sl, n].T.astype(np.float64), log_std=np.tile(ls, (e + 1 - start, 1)))),
                env_infos=dict(),
            )
            if getattr(batch, "prev_action_info", False):
                a = p["actions"]
                p["agent_infos"]["prev_action"] = np.concatenate([np.zeros((1, A)), a[:-1]], axis=0)
            if adv is not None:
                p["advantages"] = adv[sl, n].astype(np.float64)
                p["returns"] = ret[sl, n].astype(np.float64)
            paths.append(p)
            start = e + 1
    return paths


def recurrent_samples_entry(paths, key):
    """Entry `key` of the reference's recurrent samples_data (sampler/base.py:105-161) from path dicts whose advantages
    are already centred: every per-sample array zero-padded to (n_paths, max_path_len, ...) in path order, "valids" 1 on
    the samples of each path, agent_infos padded key by key, env_infos empty."""
    if key == "paths":
        return paths
    T = max(len(p["rewards"]) for p in paths)

    def pad(x):
        x = np.asarray(x)
        out = np.zeros((T,) + x.shape[1:])
        out[:len(x)] = x
        return out
    if key == "valids":
        return np.asarray([pad(np.ones(len(p["rewards"]))) for p in paths])
    if key == "agent_infos":
        return {k: np.asarray([pad(p["agent_infos"][k]) for p in paths]) for k in paths[0]["agent_infos"]}
    if key == "env_infos":
        return dict()
    return np.asarray([pad(p[key]) for p in paths])


class SamplesData(dict):
    """samples_data of rllab/sampler/base.py:95-104.  The device batch is under "lane_batch"; the reference's host
    arrays ("observations", "actions", "rewards", "returns", "advantages", "agent_infos", "env_infos", "paths") are
    materialised in the reference layout ((B, dim) float64, sample order t-major then lane) on first access.  For a
    recurrent policy the layout is the reference's recurrent one (base.py:105-161): every array padded with zeros to
    (n_paths, max_path_len, ...) in path order, plus "valids" (1 on the samples of each path)."""
    _LAZY = ("observations", "actions", "rewards", "returns", "advantages", "agent_infos", "env_infos", "paths",
             "valids")

    def __init__(self, batch, paths):
        dict.__init__(self, lane_batch=batch)
        self.lane_batch = batch
        self._paths = paths

    def _recurrent(self, key):
        return recurrent_samples_entry(self._paths.to_paths(), key)

    def __missing__(self, key):
        if key not in self._LAZY:
            raise KeyError(key)
        b = self.lane_batch
        if getattr(b, "recurrent", False):
            v = self[key] = self._recurrent(key)
            return v
        if key == "valids":
            raise KeyError(key)
        import torch
        from .. import ops

        def rows(src, dim):
            dst = torch.empty((b.B, dim), dtype=torch.float64, device=b.device)
            ops.planes_to_rows_f64(src, dim, b.B, dst)
            out = dst.cpu().numpy()
            return out[b.valid_mask().reshape(-1)] if b.masked else out      # dropped paths are not samples
        if key == "observations":
            v = rows(b.obs, b.O)
        elif key == "actions":
            v = rows(b.act, b.A)
        elif key in ("rewards", "returns", "advantages"):
            v = rows(dict(rewards=b.rew, returns=b.ret, advantages=b.adv)[key], 1).reshape(-1)
        elif key == "agent_infos" and b.categorical:
            v = dict(prob=rows(b.mean, b.A))
        elif key == "agent_infos":
            v_mean = rows(b.mean, b.A)
            v = dict(mean=v_mean,
                     log_std=np.tile(b.log_std.double().cpu().numpy().reshape(1, -1), (len(v_mean), 1)))
        elif key == "env_infos":
            v = dict()
        else:
            v = self._paths.to_paths()
        self[key] = v
        return v

    def __contains__(self, key):
        if key == "valids":
            return bool(getattr(self.lane_batch, "recurrent", False))
        return dict.__contains__(self, key) or key in self._LAZY


class LaneSampler(Sampler):
    def __init__(self, algo, n_envs=None, seed=None, comm=None):
        """
        :param algo: the BatchPolopt instance (supplies env, policy, baseline, batch_size, max_path_length, ...)
        :param n_envs: total number of lanes over all GPUs (default ceil(batch_size / max_path_length))
        :param seed: Philox key (default: drawn once from np.random so that ext.set_seed-style seeding carries over)
        """
        self.algo = algo
        self.n_envs = n_envs
        self.seed = seed
        self.comm = comm
        self.batch = None
        self._stats = None
        self._pending = None

    def start_worker(self):
        import torch
        from .. import ops
        algo = self.algo
        if self.comm is None:
            from ..parallel import default_comm
            self.comm = default_comm()
        if not torch.cuda.is_available():
            raise L.B200RLError("LaneSampler needs a CUDA device (no CPU fallback)")
        dev = torch.device("cuda", torch.cuda.current_device())
        env = algo.env
        if not hasattr(env, "wrapped_env") or not hasattr(env, "env_kind"):
            raise TypeError("LaneSampler drives normalize(<rllab_b200 env>) (every reference example wraps its env in "
                            "normalize(); the NormalizedEnv action map is fused into the kernels)")
        self.env_kind = env.env_kind
        T = int(algo.max_path_length)
        n_total = int(self.n_envs) if self.n_envs else -(-int(algo.batch_size) // T)
        n_local, lane0 = self.comm.shard(n_total)
        if n_local <= 0:
            raise ValueError("fewer lanes (%d) than ranks (%d)" % (n_total, self.comm.world_size))
        pol = algo.policy
        self.batch = ops.LaneBatch(pol.obs_dim, pol.action_dim, n_local, T, dev)
        self.batch.categorical = ops.is_categorical(pol.dims)
        self.batch.recurrent = ops.is_gru(pol.dims)
        self.batch.prev_action_info = self.batch.recurrent and bool(pol.state_include_action)
        if self.batch.categorical != (ops.env_num_actions(self.env_kind) > 0):
            raise TypeError("the policy's action distribution does not match the env's action space")
        self.batch.B_global = n_total * T
        self.batch.processed = False
        self.lane0 = lane0
        self.n_total = n_total
        logger.log("LaneSampler: %d lanes x %d steps = %d samples per iteration (batch_size %d rounded up to whole lanes); "
                   "whole_paths=%s" % (n_total, T, n_total * T, int(algo.batch_size), bool(getattr(algo, "whole_paths", True))))
        if self.seed is None:
            self.seed = int(np.random.randint(0, 2 ** 31 - 1))
        self._sums_host = None

    def shutdown_worker(self):
        self.batch = None

    def obtain_samples(self, itr):
        from .. import ops
        algo, b, pol = self.algo, self.batch, self.algo.policy
        if b.recurrent:
            ops.gru_rollout(pol.dims, pol.theta32, b, int(algo.max_path_length), self.env_kind, None, None,
                            int(self.seed) & 0xFFFFFFFF, int(itr) & 0xFFFFFFFF, self.lane0)
        else:
            ops.rollout(self.env_kind, pol.theta32, pol.h1, pol.h2, pol.min_std, b, int(algo.max_path_length), None, None,
                        int(self.seed) & 0xFFFFFFFF, int(itr) & 0xFFFFFFFF, self.lane0)
        b.version += 1
        b.processed = False
        b.masked = False
        return LanePaths(b, bool(getattr(algo, "whole_paths", True)))

    def process_samples(self, itr, paths):
        from .. import ops
        algo = self.algo
        b = paths.lane_batch
        # a baseline with its own device predictor (GaussianMLPBaseline) writes batch.base itself; the previous fit's
        # weights predict, the fit on this batch's returns follows the advantages (base.py:163-167)
        own_predict = hasattr(algo.baseline, "predict_lanes")
        if own_predict:
            algo.baseline.predict_lanes(b)
            ops.process_samples_base(b, algo.discount, algo.gae_lambda,
                                     drop_cut_paths=bool(getattr(algo, "whole_paths", True)))
        else:
            w = algo.baseline.device_weights(b.O, b.device)
            ops.process_samples(b, w, algo.discount, algo.gae_lambda,
                                drop_cut_paths=bool(getattr(algo, "whole_paths", True)))
        # the baseline's normal equations only need the returns: reduce them right away so that ONE collective carries
        # the advantage sums, the normal equations and the maxima (the fit itself still follows the advantages, as in
        # base.py:163-167 -- the order has no numerical effect)
        lanes_fit = hasattr(algo.baseline, "gram_lanes")
        if lanes_fit:
            algo.baseline.gram_lanes(b)
        self.comm.all_reduce_mixed(b.red, b.n_red_sum)
        if algo.center_adv or algo.positive_adv:
            ops.center_advantages(b, algo.center_adv, algo.positive_adv)
        b.version += 1
        b.processed = True
        samples_data = SamplesData(b, paths)

        logger.log("fitting baseline...")
        if lanes_fit:
            algo.baseline.solve_lanes(b)
        elif own_predict:
            algo.baseline.fit_lanes(b, self.comm)
        else:
            algo.baseline.fit(paths.to_paths())
        logger.log("fitted")

        # statistics: queued pinned-memory readbacks, resolved when the logger dumps the table (or `stats` is read), so
        # the host does not stall the GPU between process_samples and the policy update
        if b.categorical:
            # Entropy = mean over the valid samples of the state-dependent entropy(prob) (base.py:93)
            ent = self._ent_buf(b)
            ops.categorical_entropy(b, ent)
            self.comm.all_reduce_mixed(ent, 2)
            p_ent = ops.PendingHost(ent)
        else:
            p_ent = ops.PendingHost(b.log_std)
        self._pending = (itr, ops.PendingHost(b.sums), ops.PendingHost(b.maxs), p_ent, b.categorical)
        self._stats = None
        for k in ("Iteration", "AverageDiscountedReturn", "AverageReturn", "ExplainedVariance", "NumTrajs", "Entropy",
                  "Perplexity", "StdReturn", "MaxReturn", "MinReturn"):
            logger.record_tabular(k, lambda k=k: self.stats[k])
        return samples_data

    def _ent_buf(self, b):
        import torch
        buf = getattr(self, "_ent", None)
        if buf is None or buf.device != b.device:
            buf = self._ent = torch.zeros(2, dtype=torch.float64, device=b.device)
        return buf

    @property
    def stats(self):
        """The tabular statistics of the last process_samples (base.py:170-180), resolved on first use."""
        if self._stats is None:
            if self._pending is None:
                return {}
            self._stats = self._resolve_stats(*self._pending)
        return self._stats

    @staticmethod
    def _resolve_stats(itr, p_sums, p_maxs, p_ent, categorical=False):
        """p_ent: the categorical (entropy sum, sample count) when `categorical`, else the device log_std."""
        s, m = p_sums.get(), p_maxs.get()
        n_paths = s[3]
        avg_ret = s[5] / n_paths
        vary = s[8] / s[2] - (s[7] / s[2]) ** 2
        varpred = s[10] / s[2] - (s[9] / s[2]) ** 2
        varres = s[12] / s[2] - (s[11] / s[2]) ** 2
        if np.isclose(vary, 0):                        # special.explained_variance_1d, special.py:51-59
            ev = 0 if varpred > 0 else 1
        else:
            ev = 1 - varres / (vary + 1e-8)
        e = p_ent.get()
        if categorical:
            ent = float(e[0] / e[1])
        else:
            ent = float(np.sum(e.astype(np.float64) + np.log(np.sqrt(2 * np.pi * np.e))))
        return dict(
            Iteration=itr, AverageDiscountedReturn=s[4] / n_paths, AverageReturn=avg_ret, ExplainedVariance=ev,
            NumTrajs=int(round(n_paths)), Entropy=ent, Perplexity=np.exp(ent),
            StdReturn=np.sqrt(max(s[6] / n_paths - avg_ret ** 2, 0.0)), MaxReturn=m[0], MinReturn=-m[1])
