"""Device operations of the hot path as thin, typed wrappers over the C ABI (rllab_b200/_lib.py).

Tensors are torch CUDA tensors used purely as array containers (no autograd anywhere); every wrapper validates
dtype/shape/contiguity, passes raw pointers + the current CUDA stream, and raises on failure.
Layouts are documented in include/b200rl.h.
"""
import ctypes

import numpy as np
import torch

from . import _lib as L

F32, F64, U8, U16 = torch.float32, torch.float64, torch.uint8, torch.uint16


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _chk(t, dtype, name, numel=None):
    if t is None:
        return
    if not t.is_cuda or t.dtype != dtype or not t.is_contiguous():
        raise ValueError("%s must be a contiguous CUDA tensor of dtype %s (got %s, cuda=%s)" %
                         (name, dtype, t.dtype, t.is_cuda))
    if numel is not None and t.numel() != numel:
        raise ValueError("%s must have %d elements, has %d" % (name, numel, t.numel()))


_ws_cache = {}


def workspace(device):
    """float64 reduction workspace (b200rl_ws_doubles entries), one per device, allocated once."""
    key = torch.device(device).index
    ws = _ws_cache.get(key)
    if ws is None:
        n = int(L.load().b200rl_ws_doubles())
        ws = torch.empty(n, dtype=F64, device=device)
        _ws_cache[key] = ws
    return ws


class LaneBatch(object):
    """Device trajectory buffers of one rollout: N lanes x T steps (layout of include/b200rl.h)."""

    def __init__(self, O, A, N, T, device):
        self.O, self.A, self.N, self.T = O, A, N, T
        self.device = device
        self.obs = torch.empty((O, T, N), dtype=F32, device=device)
        self.act = torch.empty((A, T, N), dtype=F32, device=device)
        self.mean = torch.empty((A, T, N), dtype=F32, device=device)
        self.rew = torch.empty((T, N), dtype=F32, device=device)
        self.flags = torch.empty((T, N), dtype=U8, device=device)
        self.tstep = torch.empty((T, N), dtype=U16, device=device)
        self.log_std = torch.empty((A,), dtype=F32, device=device)
        self.adv = torch.empty((T, N), dtype=F32, device=device)
        self.ret = torch.empty((T, N), dtype=F32, device=device)
        self.base = torch.empty((T, N), dtype=F32, device=device)
        # reduction block of process_samples + the baseline fit, contiguous so that ONE collective carries all of it:
        # [sums (PS_NSUM) | LinearFeatureBaseline normal equations (d+1)(d+2)/2 | maxs (PS_NMAX)]
        d1 = 2 * O + 5
        self.n_gram = d1 * (d1 + 1) // 2
        self.red = torch.zeros((L.PS_NSUM + self.n_gram + L.PS_NMAX,), dtype=F64, device=device)
        self.sums = self.red[:L.PS_NSUM]
        self.gram = self.red[L.PS_NSUM:L.PS_NSUM + self.n_gram]
        self.maxs = self.red[L.PS_NSUM + self.n_gram:]
        self.n_red_sum = L.PS_NSUM + self.n_gram      # leading entries that are sums (the rest are maxima)
        self.count = self.sums[2:3]   # device-resident number of valid samples over all ranks (after the all-reduce)
        self.version = 0              # bumped by the sampler whenever the contents change
        self.processed = False        # adv/ret/base valid (process_samples has run on this rollout)
        self.B_global = N * T         # samples over all ranks (the sampler overwrites it under torchrun)
        self.masked = False           # process_samples dropped cut paths: passes read FLAG_MASKED and the device count
        self.categorical = False      # act holds one-hot actions and mean the probabilities of a categorical policy

    @property
    def B(self):
        return self.N * self.T

    def hcache(self, h1, h2):
        """[h1+h2][T][N] float32 activation cache for the CG solve (allocated on first use; 256 B/sample at 32,32)."""
        hc = getattr(self, "_hcache", None)
        if hc is None or hc.shape[0] != h1 + h2:
            hc = torch.empty((h1 + h2, self.T, self.N), dtype=F32, device=self.device)
            self._hcache = hc
        return hc

    def valid_mask(self):
        """(T, N) bool host array: samples that are not part of a dropped (cut) path."""
        if not self.masked:
            return np.ones((self.T, self.N), dtype=bool)
        return (self.flags.cpu().numpy() & L.FLAG_MASKED) == 0

    def to_numpy(self):
        """Host copy in the oracle's dict layout (tests / path materialisation)."""
        return dict(obs=self.obs.cpu().numpy(), act=self.act.cpu().numpy(), mean=self.mean.cpu().numpy(),
                    rew=self.rew.cpu().numpy(), flags=self.flags.cpu().numpy(),
                    tstep=self.tstep.cpu().view(torch.int16).numpy().view(np.uint16),
                    log_std=self.log_std.cpu().numpy())


class CategoricalDims(tuple):
    """(O, h1, h2, n) of a CategoricalMLPPolicy.  A policy hands its `dims` to the update passes below; this type is what
    makes them run the categorical kernels (b200rl_categorical_*), with batch.mean holding the old probabilities and
    batch.act the one-hot actions.  A plain tuple (O, h1, h2, A) selects the Gaussian kernels."""

    def __new__(cls, O, h1, h2, n):
        return tuple.__new__(cls, (int(O), int(h1), int(h2), int(n)))

    def __getnewargs__(self):
        return tuple(self)


def is_categorical(dims):
    return isinstance(dims, CategoricalDims)


_n_actions = {}


def env_num_actions(kind):
    """Discrete actions of an env kind (0: Box), cached per kind."""
    n = _n_actions.get(kind)
    if n is None:
        n = _n_actions[kind] = L.env_num_actions(kind)
    return n


def fill_noise(out, rows, row0, K, N, lane0, kind, seed, it, stream_id):
    _chk(out, F32, "out", rows * K * N)
    L.call("b200rl_fill_noise", L.ptr(out), rows, row0, K, N, lane0, kind, seed, it, stream_id, _stream())


def env_reset(kind, N, state, obs_out, reset_raw=None, seed=0, it=0, row=0, lane0=0):
    _chk(state, F32, "state"), _chk(obs_out, F32, "obs_out"), _chk(reset_raw, F32, "reset_raw")
    L.call("b200rl_env_reset", kind, N, L.ptr(state), L.ptr(obs_out), L.ptr(reset_raw), seed, it, row, lane0, _stream())


def env_step(kind, N, state, actions, obs_out, rew_out, done_out, normalized=True):
    _chk(state, F32, "state"), _chk(actions, F32, "actions"), _chk(obs_out, F32, "obs_out")
    _chk(rew_out, F32, "rew_out", N), _chk(done_out, U8, "done_out", N)
    L.call("b200rl_env_step", kind, N, int(bool(normalized)), L.ptr(state), L.ptr(actions), L.ptr(obs_out), L.ptr(rew_out), L.ptr(done_out),
           _stream())


def policy_get_actions(params32, O, h1, h2, A, min_std, obs, n, eps, seed, it, row, lane0, act_out, mean_out, log_std_out):
    _chk(params32, F32, "params32"), _chk(obs, F32, "obs", O * n), _chk(eps, F32, "eps")
    _chk(act_out, F32, "act_out", A * n), _chk(mean_out, F32, "mean_out", A * n), _chk(log_std_out, F32, "log_std_out", A)
    L.call("b200rl_policy_get_actions", L.ptr(params32), O, h1, h2, A, float(min_std or 0.0), L.ptr(obs), n, L.ptr(eps),
           seed, it, row, lane0, L.ptr(act_out), L.ptr(mean_out), L.ptr(log_std_out), _stream())


def rollout(kind, params32, h1, h2, min_std, batch, max_path_length, eps=None, reset_raw=None, seed=0, it=0, lane0=0):
    """Fused rollout.  A discrete-action env kind runs the categorical rollout: `eps` is then the injected uniform u
    [T][N] of the action draw, batch.act receives one-hot actions and batch.mean the probabilities."""
    b = batch
    _chk(params32, F32, "params32"), _chk(eps, F32, "eps"), _chk(reset_raw, F32, "reset_raw")
    if env_num_actions(kind) > 0:
        _chk(eps, F32, "u", b.T * b.N)
        L.call("b200rl_rollout_categorical", kind, L.ptr(params32), h1, h2, b.N, b.T, max_path_length, L.ptr(eps),
               L.ptr(reset_raw), seed, it, lane0, L.ptr(b.obs), L.ptr(b.act), L.ptr(b.mean), L.ptr(b.rew),
               L.ptr(b.flags), L.ptr(b.tstep), _stream())
        return
    L.call("b200rl_rollout", kind, L.ptr(params32), h1, h2, float(min_std or 0.0), b.N, b.T, max_path_length,
           L.ptr(eps), L.ptr(reset_raw), seed, it, lane0, L.ptr(b.obs), L.ptr(b.act), L.ptr(b.mean), L.ptr(b.rew),
           L.ptr(b.flags), L.ptr(b.tstep), L.ptr(b.log_std), _stream())


def categorical_get_actions(params32, dims, obs, n, u, seed, it, row, lane0, act_out, prob_out):
    """act_out [n] int32 = weighted_sample(prob, u), prob_out [n_actions][n] (b200rl_categorical_get_actions)."""
    O, h1, h2, A = dims
    _chk(params32, F32, "params32"), _chk(obs, F32, "obs", O * n), _chk(u, F32, "u", n)
    _chk(act_out, torch.int32, "act_out", n), _chk(prob_out, F32, "prob_out", A * n)
    L.call("b200rl_categorical_get_actions", L.ptr(params32), O, h1, h2, A, L.ptr(obs), n, L.ptr(u), seed, it, row,
           lane0, L.ptr(act_out), L.ptr(prob_out), _stream())


def categorical_entropy(batch, out):
    """out [2] float64 = (sum of the entropy of batch.mean's probabilities, number of samples) over the valid samples."""
    b = batch
    _chk(out, F64, "out", 2)
    L.call("b200rl_categorical_entropy", b.A, b.B, L.ptr(b.mean), L.ptr(b.flags) if b.masked else None, L.ptr(out),
           L.ptr(workspace(b.device)), _stream())


def process_samples(batch, w, discount, gae_lambda, drop_cut_paths=False):
    b = batch
    _chk(w, F64, "w", 2 * b.O + 4)
    L.call("b200rl_process_samples", b.O, b.N, b.T, L.ptr(b.obs), L.ptr(b.rew), L.ptr(b.flags), L.ptr(b.tstep),
           L.ptr(w), float(discount), float(gae_lambda), int(bool(drop_cut_paths)), L.ptr(b.adv), L.ptr(b.ret),
           L.ptr(b.base), L.ptr(b.sums), L.ptr(b.maxs), L.ptr(workspace(b.device)), _stream())
    b.masked = bool(drop_cut_paths)


def process_samples_base(batch, discount, gae_lambda, drop_cut_paths=False):
    """process_samples with the baseline already in batch.base (GaussianMLPBaseline.predict_lanes)."""
    b = batch
    L.call("b200rl_process_samples_base", b.O, b.N, b.T, L.ptr(b.obs), L.ptr(b.rew), L.ptr(b.flags), L.ptr(b.tstep),
           L.ptr(b.base), float(discount), float(gae_lambda), int(bool(drop_cut_paths)), L.ptr(b.adv), L.ptr(b.ret),
           L.ptr(b.sums), L.ptr(b.maxs), L.ptr(workspace(b.device)), _stream())
    b.masked = bool(drop_cut_paths)


VF_STATS_SUMS, VF_STATS_SQUARES, VF_STATS_FINISH, VF_STATS_ALL = 0, 1, 2, 3


def vf_norm_stats(O, B, obs, y, flags, stage, acc, stats_out):
    """Regressor normalisation constants (b200rl_vf_norm_stats): acc [2O+3], stats_out [2O+2] float64."""
    _chk(obs, F32, "obs", O * B), _chk(y, F32, "y", B), _chk(flags, U8, "flags", B)
    _chk(acc, F64, "acc", 2 * O + 3), _chk(stats_out, F64, "stats_out", 2 * O + 2)
    L.call("b200rl_vf_norm_stats", O, B, L.ptr(obs), L.ptr(y), L.ptr(flags), int(stage), L.ptr(acc), L.ptr(stats_out),
           L.ptr(workspace(obs.device)), _stream())


def vf_forward(params32, O, B, obs, stats, out, denormalize):
    _chk(params32, F32, "params32", L.vf_num_params(O)), _chk(obs, F32, "obs", O * B)
    _chk(stats, F64, "stats", 2 * O + 2), _chk(out, F32, "out", B)
    L.call("b200rl_vf_forward", L.ptr(params32), O, 32, 32, B, L.ptr(obs), L.ptr(stats), int(bool(denormalize)),
           L.ptr(out), _stream())


def vf_loss_grad(params32, O, B, obs, y, flags, stats, mu_old, old_log_std, penalty, learn_std, scale, count, g_out,
                 loss_out, fuse=False):
    """loss_out[3] = (mean NLL, mean KL, max KL); g_out [P] (or None) = gradient of mean NLL + penalty * mean KL."""
    P = L.vf_num_params(O)
    _chk(params32, F32, "params32", P), _chk(obs, F32, "obs", O * B), _chk(y, F32, "y", B)
    _chk(flags, U8, "flags", B), _chk(stats, F64, "stats", 2 * O + 2), _chk(mu_old, F32, "mu_old", B)
    _chk(count, F64, "count", 1), _chk(g_out, F64, "g_out", P), _chk(loss_out, F64, "loss_out", 3)
    with _Fused(fuse):
        L.call("b200rl_vf_loss_grad", L.ptr(params32), O, 32, 32, B, L.ptr(obs), L.ptr(y), L.ptr(flags), L.ptr(stats),
               L.ptr(mu_old), float(old_log_std), float(penalty), int(bool(learn_std)), float(scale), L.ptr(count),
               L.ptr(g_out), L.ptr(loss_out), L.ptr(workspace(obs.device)), _stream())


def _mask(batch):
    """(flags pointer, scale, count pointer) of an update pass over `batch`: with dropped paths the kernels skip
    FLAG_MASKED samples and divide by the device-resident valid-sample count; otherwise by B_global on the host."""
    if batch.masked:
        return L.ptr(batch.flags), 1.0, L.ptr(batch.count)
    return None, 1.0 / batch.B_global, None


def center_advantages(batch, center, positive):
    b = batch
    L.call("b200rl_center_advantages", L.ptr(b.adv), b.B, L.ptr(b.flags) if b.masked else None, L.ptr(b.sums),
           L.ptr(b.maxs), int(center), int(positive), _stream())


def lfb_gram(batch, gram_out):
    b = batch
    d1 = 2 * b.O + 5
    _chk(gram_out, F64, "gram_out", d1 * (d1 + 1) // 2)
    L.call("b200rl_lfb_gram", b.O, b.B, L.ptr(b.obs), L.ptr(b.tstep), L.ptr(b.ret),
           L.ptr(b.flags) if b.masked else None, L.ptr(gram_out), L.ptr(workspace(b.device)), _stream())


def lfb_solve(obs_dim, gram, reg_coeff, w_out, info_out):
    _chk(gram, F64, "gram"), _chk(w_out, F64, "w_out", 2 * obs_dim + 4), _chk(info_out, F64, "info_out", 3)
    L.call("b200rl_lfb_solve", obs_dim, L.ptr(gram), float(reg_coeff), L.ptr(w_out), L.ptr(info_out), _stream())


class _Fused(object):
    """`with _Fused(fuse):` -- the update pass launched inside reduces its outputs over the ranks of the bound peer-memory
    communicator in its own finalize kernel (csrc/peer.cuh).  The switch is per call, not per process: a process may drive
    a sharded job and a single-rank job side by side (bench.py's shard check does)."""

    def __init__(self, fuse):
        self.fuse = bool(fuse)

    def __enter__(self):
        if self.fuse:
            L.call("b200rl_peer_fuse_updates", 1)

    def __exit__(self, *exc):
        if self.fuse:
            L.call("b200rl_peer_fuse_updates", 0)
        return False


def peer_allreduce_mixed(t, n_sum):
    """In place over the bound peer-memory communicator: t[:n_sum] summed, t[n_sum:] maximised over ranks (rank order)."""
    _chk(t, F64, "t")
    L.call("b200rl_peer_allreduce_mixed", L.ptr(t), t.numel(), int(n_sum), _stream())


def loss_kl(loss_kind, params32, dims, min_std, batch, out, fuse=False):
    """out[3] = (surrogate loss, mean KL, max KL) of this rank's samples, already divided by the global sample count
    (fuse=True: of all ranks' samples)."""
    O, h1, h2, A = dims
    b = batch
    fl, scale, cnt = _mask(b)
    _chk(params32, F32, "params32"), _chk(out, F64, "out", 3)
    if is_categorical(dims):
        with _Fused(fuse):
            L.call("b200rl_categorical_loss_kl", loss_kind, L.ptr(params32), O, h1, h2, A, b.B, L.ptr(b.obs),
                   L.ptr(b.act), L.ptr(b.adv), L.ptr(b.mean), fl, scale, cnt, L.ptr(out), L.ptr(workspace(b.device)),
                   _stream())
        return
    with _Fused(fuse):
        L.call("b200rl_loss_kl", loss_kind, L.ptr(params32), O, h1, h2, A, float(min_std or 0.0), b.B, L.ptr(b.obs),
               L.ptr(b.act), L.ptr(b.adv), L.ptr(b.mean), L.ptr(b.log_std), fl, scale, cnt, L.ptr(out),
               L.ptr(workspace(b.device)), _stream())


def grad(loss_kind, params32, dims, min_std, batch, g_out, loss_out=None, h_cache=None, fuse=False):
    O, h1, h2, A = dims
    b = batch
    fl, scale, cnt = _mask(b)
    _chk(params32, F32, "params32"), _chk(g_out, F64, "g_out")
    if is_categorical(dims):
        _categorical_grad(loss_kind, 0.0, params32, dims, b, g_out, loss_out, h_cache, fuse)
        return
    with _Fused(fuse):
        L.call("b200rl_grad", loss_kind, L.ptr(params32), O, h1, h2, A, float(min_std or 0.0), b.B, L.ptr(b.obs),
               L.ptr(b.act), L.ptr(b.adv), L.ptr(b.mean), L.ptr(b.log_std), fl, scale, cnt, L.ptr(g_out), L.ptr(loss_out),
               L.ptr(h_cache), L.ptr(workspace(b.device)), _stream())


def grad_penalized(loss_kind, penalty, params32, dims, min_std, batch, g_out, loss_out=None, fuse=False):
    """g_out = gradient of surrogate + penalty * mean KL(old || new); loss_out[3] = the unpenalised (loss, mean KL,
    max KL) of the same pass (b200rl_grad_penalized)."""
    O, h1, h2, A = dims
    b = batch
    fl, scale, cnt = _mask(b)
    _chk(params32, F32, "params32"), _chk(g_out, F64, "g_out")
    if is_categorical(dims):
        _categorical_grad(loss_kind, penalty, params32, dims, b, g_out, loss_out, None, fuse)
        return
    with _Fused(fuse):
        L.call("b200rl_grad_penalized", loss_kind, float(penalty), L.ptr(params32), O, h1, h2, A, float(min_std or 0.0),
               b.B, L.ptr(b.obs), L.ptr(b.act), L.ptr(b.adv), L.ptr(b.mean), L.ptr(b.log_std), fl, scale, cnt,
               L.ptr(g_out), L.ptr(loss_out), L.ptr(workspace(b.device)), _stream())


def _categorical_grad(loss_kind, penalty, params32, dims, batch, g_out, loss_out, h_cache, fuse):
    O, h1, h2, A = dims
    b = batch
    fl, scale, cnt = _mask(b)
    with _Fused(fuse):
        L.call("b200rl_categorical_grad", loss_kind, float(penalty), L.ptr(params32), O, h1, h2, A, b.B, L.ptr(b.obs),
               L.ptr(b.act), L.ptr(b.adv), L.ptr(b.mean), fl, scale, cnt, L.ptr(g_out), L.ptr(loss_out),
               L.ptr(h_cache), L.ptr(workspace(b.device)), _stream())


def fvp(params32, dims, min_std, batch, x, reg_coeff, diag_scale, Hx_out, h_cache=None, tile_list=None, count=None,
        fuse=False):
    """tile_list (int32 device tensor) + count (float64 device scalar: valid samples in those tiles over all ranks):
    the sub-sampled product of subsample_factor < 1."""
    O, h1, h2, A = dims
    b = batch
    fl, scale, cnt = _mask(b)
    if tile_list is not None:
        scale, cnt = 1.0, L.ptr(count)
    _chk(params32, F32, "params32"), _chk(x, F64, "x"), _chk(Hx_out, F64, "Hx_out", x.numel())
    if is_categorical(dims):
        with _Fused(fuse):
            L.call("b200rl_categorical_fvp", L.ptr(params32), O, h1, h2, A, b.B, L.ptr(b.obs), fl, L.ptr(x), scale, cnt,
                   float(reg_coeff), float(diag_scale), L.ptr(Hx_out), L.ptr(h_cache), L.ptr(tile_list),
                   0 if tile_list is None else int(tile_list.numel()), L.ptr(workspace(b.device)), _stream())
        return
    with _Fused(fuse):
        L.call("b200rl_fvp", L.ptr(params32), O, h1, h2, A, float(min_std or 0.0), b.B, L.ptr(b.obs), fl, L.ptr(x), scale,
               cnt, float(reg_coeff), float(diag_scale), L.ptr(Hx_out), L.ptr(h_cache), L.ptr(tile_list),
               0 if tile_list is None else int(tile_list.numel()), L.ptr(workspace(b.device)), _stream())


def count_valid(batch, tile_list, out):
    b = batch
    L.call("b200rl_count_valid", b.B, L.ptr(b.flags) if b.masked else None, L.ptr(tile_list),
           0 if tile_list is None else int(tile_list.numel()), L.ptr(out), L.ptr(workspace(b.device)), _stream())


def update_f64(mode, loss_kind, params64, dims, min_std, batch, x, reg_coeff, diag_scale, vec_out, loss_out, fuse=False):
    """float64 parity-mode pass: mode 0 loss/KL, 1 gradient (+loss), 2 Fisher-vector product."""
    O, h1, h2, A = dims
    b = batch
    fl, scale, cnt = _mask(b)
    _chk(params64, F64, "params64"), _chk(x, F64, "x"), _chk(vec_out, F64, "vec_out"), _chk(loss_out, F64, "loss_out", 3)
    if is_categorical(dims):
        with _Fused(fuse):
            L.call("b200rl_categorical_update_f64", mode, loss_kind, L.ptr(params64), O, h1, h2, A, b.B, L.ptr(b.obs),
                   L.ptr(b.act), L.ptr(b.adv), L.ptr(b.mean), fl, L.ptr(x), scale, cnt, float(reg_coeff),
                   float(diag_scale), L.ptr(vec_out), L.ptr(loss_out), L.ptr(workspace(b.device)), _stream())
        return
    with _Fused(fuse):
        L.call("b200rl_update_f64", mode, loss_kind, L.ptr(params64), O, h1, h2, A, float(min_std or 0.0), b.B, L.ptr(b.obs),
               L.ptr(b.act), L.ptr(b.adv), L.ptr(b.mean), L.ptr(b.log_std), fl, L.ptr(x), scale, cnt, float(reg_coeff),
               float(diag_scale), L.ptr(vec_out), L.ptr(loss_out), L.ptr(workspace(b.device)), _stream())


def cg_init(g, x, r, p, st, p_f32=False):
    L.call("b200rl_cg_init", g.numel(), L.ptr(g), L.ptr(x), L.ptr(r), L.ptr(p), L.ptr(st), int(bool(p_f32)), _stream())


def cg_step(z, x, r, p, st, tol=1e-10, p_f32=False):
    L.call("b200rl_cg_step", z.numel(), L.ptr(z), L.ptr(x), L.ptr(r), L.ptr(p), L.ptr(st), float(tol), int(bool(p_f32)),
           _stream())


def trpo_step_size(x, Hx, delta, step_out, info_out):
    L.call("b200rl_trpo_step_size", x.numel(), L.ptr(x), L.ptr(Hx), float(delta), L.ptr(step_out), L.ptr(info_out),
           _stream())


def axpy_params(prev, step, ratio, out64, out32):
    L.call("b200rl_axpy_params", prev.numel(), L.ptr(prev), L.ptr(step), float(ratio), L.ptr(out64), L.ptr(out32),
           _stream())


def adam_step(theta64, theta32, g, m, v, t, lr=1e-3, b1=0.9, b2=0.999, eps=1e-8):
    L.call("b200rl_adam_step", theta64.numel(), L.ptr(theta64), L.ptr(theta32), L.ptr(g), L.ptr(m), L.ptr(v), int(t),
           float(lr), float(b1), float(b2), float(eps), _stream())


def f64_to_f32(src, dst):
    L.call("b200rl_f64_to_f32", src.numel(), L.ptr(src), L.ptr(dst), _stream())


def reduce_ranks(gathered, world, n, n_sum, out):
    _chk(gathered, F64, "gathered", world * n), _chk(out, F64, "out", n)
    L.call("b200rl_reduce_ranks", L.ptr(gathered), int(world), int(n), int(n_sum), L.ptr(out), _stream())


def planes_to_rows_f64(src, dim, B, dst):
    _chk(src, F32, "src", dim * B), _chk(dst, F64, "dst", dim * B)
    L.call("b200rl_planes_to_rows_f64", dim, B, L.ptr(src), L.ptr(dst), _stream())


I64, I32 = torch.int64, torch.int32


def population_sample(cur_mean, cur_std, extra_var, seed, it, theta_out, members=None, member0=0):
    """theta_out [n][P] float64: CEM parameter rows of members `members` (int64 device tensor) or member0 .. member0+n-1."""
    P = cur_mean.numel()
    _chk(cur_mean, F64, "cur_mean"), _chk(cur_std, F64, "cur_std", P), _chk(members, I64, "members")
    n = theta_out.shape[0]
    _chk(theta_out, F64, "theta_out", n * P)
    if members is not None and members.numel() != n:
        raise ValueError("members must have one entry per row of theta_out")
    L.call("b200rl_population_sample", P, L.ptr(cur_mean), L.ptr(cur_std), float(extra_var), int(seed) & 0xFFFFFFFF,
           int(it) & 0xFFFFFFFF, L.ptr(members), int(member0), n, L.ptr(theta_out), _stream())


class PopulationResult(object):
    """Device outputs of one population rollout of M members x E evals (b200rl_population_rollout)."""

    def __init__(self, M, E, O, device, keep_obs=True):
        self.M, self.E, self.O = M, E, O
        self.ret = torch.empty((M, E), dtype=F64, device=device)
        self.undisc = torch.empty((M, E), dtype=F64, device=device)
        self.len = torch.empty((M, E), dtype=I32, device=device)
        self.obs_first = torch.empty((M, E, O), dtype=F32, device=device) if keep_obs else None
        self.obs_last = torch.empty((M, E, O), dtype=F32, device=device) if keep_obs else None
        self.member = torch.empty((M, 3), dtype=F64, device=device)


def population_rollout(kind, theta, h1, h2, min_std, n_evals, max_path_length, discount, seed, it, lane0, out):
    """out: PopulationResult with out.M == theta.shape[0]; lane0 = global lane of member 0, eval 0."""
    M = theta.shape[0]
    _chk(theta, F64, "theta")
    if out.M != M or out.E != n_evals:
        raise ValueError("result buffers are %d x %d, the call is %d x %d" % (out.M, out.E, M, n_evals))
    info = L.env_info(kind)                                  # raises on an unknown env kind
    if out.O != info["obs_dim"]:
        raise ValueError("result buffers hold %d-dim observations, the env has %d" % (out.O, info["obs_dim"]))
    if h1 == h2 and h1 in (32, 64):                          # other shapes are rejected by the library itself
        P = L.policy_num_params(info["obs_dim"], h1, h2, info["act_dim"])
        if theta.dim() != 2 or theta.shape[1] != P:
            raise ValueError("theta must be [M][%d] for this env and net, got %s" % (P, tuple(theta.shape)))
    L.call("b200rl_population_rollout", kind, h1, h2, float(min_std or 0.0), L.ptr(theta), M, n_evals,
           int(max_path_length), float(discount), int(seed) & 0xFFFFFFFF, int(it) & 0xFFFFFFFF, int(lane0),
           L.ptr(out.ret), L.ptr(out.undisc), L.ptr(out.len), L.ptr(out.obs_first), L.ptr(out.obs_last),
           L.ptr(out.member), L.ptr(workspace(theta.device)), _stream())


def population_topk(f, k, idx_out):
    """idx_out [k] int64: indices of the k largest of f (float64), descending, ties to the lower index."""
    _chk(f, F64, "f"), _chk(idx_out, I64, "idx_out", k)
    L.call("b200rl_population_topk", L.ptr(f), f.numel(), int(k), L.ptr(idx_out), L.ptr(workspace(f.device)),
           _stream())


def rows_mean_std(rows, mean_out, std_out):
    """Column mean / population std of rows [k][P] float64 in row order."""
    k, P = rows.shape
    _chk(rows, F64, "rows"), _chk(mean_out, F64, "mean_out", P), _chk(std_out, F64, "std_out", P)
    L.call("b200rl_rows_mean_std", P, k, L.ptr(rows), L.ptr(mean_out), L.ptr(std_out), _stream())


def reps_delta_max(batch, v, out_max):
    """out_max[1] = max over this GPU's valid samples of the REPS Bellman error r + feat_diff . v (b200rl_reps_delta_max)."""
    b = batch
    _chk(v, F64, "v", 2 * b.O + 4), _chk(out_max, F64, "out_max", 1)
    L.call("b200rl_reps_delta_max", b.O, b.N, b.T, L.ptr(b.obs), L.ptr(b.rew), L.ptr(b.flags), L.ptr(b.tstep),
           int(bool(b.masked)), L.ptr(v), L.ptr(out_max), L.ptr(workspace(b.device)), _stream())


def reps_dual_sums(batch, v, eta, M, out, w_out=None):
    """out [2O+6] = [sum e, sum e (delta - M), sum e feat_diff] with e = exp((delta - M) / eta) over this GPU's valid
    samples; w_out ([T][N] float32 or None) = e, 0 on masked samples (b200rl_reps_dual_sums).  M: float64 device [1]."""
    b = batch
    _chk(v, F64, "v", 2 * b.O + 4), _chk(M, F64, "M", 1), _chk(out, F64, "out", 2 * b.O + 6)
    _chk(w_out, F32, "w_out", b.B)
    L.call("b200rl_reps_dual_sums", b.O, b.N, b.T, L.ptr(b.obs), L.ptr(b.rew), L.ptr(b.flags), L.ptr(b.tstep),
           int(bool(b.masked)), L.ptr(v), float(eta), L.ptr(M), L.ptr(out), L.ptr(w_out), L.ptr(workspace(b.device)),
           _stream())


class PendingHost(object):
    """Asynchronous device->host readback of a small tensor: the copy into pinned host memory is queued on the current
    stream together with an event; `get()` waits for that event only (not for later work on the stream) and returns a
    numpy copy.  Lets an iteration queue all of its kernels before the host blocks once, at logging time.  Pinned
    staging buffers are pooled (page-locking is far too slow to do per call)."""
    _pool = {}
    bytes_total = 0          # device->host bytes queued so far (bench.py reports the per-step figure)

    def __init__(self, src):
        import torch
        PendingHost.bytes_total += src.numel() * src.element_size()
        self._key = (tuple(src.shape), src.dtype)
        free = PendingHost._pool.setdefault(self._key, [])
        self._host = free.pop() if free else torch.empty(src.shape, dtype=src.dtype).pin_memory()
        self._host.copy_(src, non_blocking=True)
        self._event = torch.cuda.Event()
        self._event.record()
        self._val = None

    def get(self):
        if self._val is None:
            self._event.synchronize()
            self._val = self._host.numpy().copy()
            PendingHost._pool[self._key].append(self._host)
            self._host = None
        return self._val

    def __del__(self):
        # never read: hand the staging buffer back (a later copy into it is ordered behind this one on the stream)
        host = getattr(self, "_host", None)
        if host is not None:
            try:
                PendingHost._pool[self._key].append(host)
            except Exception:
                pass


class LazyTriple(object):
    """(loss, mean KL, max KL) of one pass, read back lazily: indexing blocks on the readback event."""

    def __init__(self, src):
        self._p = PendingHost(src)
        self._v = None

    def values(self):
        if self._v is None:
            self._v = tuple(float(x) for x in self._p.get())
        return self._v

    def __getitem__(self, i):
        return self.values()[i]

    def __iter__(self):
        return iter(self.values())
