"""ConjugateGradientOptimizer, device-resident (API of rllab/optimizers/conjugate_gradient_optimizer.py:118-296).

update_opt / loss / constraint_val / optimize keep the reference's names and meaning; instead of symbolic Theano
expressions, `loss` names the surrogate kind compiled into the CUDA kernels (b200rl_loss_kl / b200rl_grad /
b200rl_fvp) and `inputs` is the device sample batch.  `optimize` follows :229-296 line by line: loss_before, flat
gradient, krylov.cg with Hessian(KL)-vector products (+reg_coeff*x), initial step size sqrt(2*delta/(x.Hx+1e-8)),
backtracking over backtrack_ratio**k with the accept test `loss < loss_before and kl <= delta`, and the final
reject-and-restore test (note >= there).  All P-vectors stay on the GPU; the host reads two scalars per
line-search trial.

Hessian-vector products (hvp_approach=):
  None / PerlmutterHvp()      exact product of the Hessian of mean KL = Gauss-Newton / Fisher product (:22-55).
                              The float32 b200rl_fvp kernels (precision="f32", tensor cores) or the float64 parity kernels
                              (precision="f64").  NOTE: the reference's product is float64; on ill-conditioned Fisher systems
                              the float32 product costs the 10-iteration CG solve about three iterations of depth, which
                              shows in the learning speed of Swimmer (DESIGN.md section 5) -- raise cg_iters or use
                              precision="f64" where that matters more than speed.
  FiniteDifferenceHvp(...)    (:58-115) two gradient passes of mean KL at theta +- eps x; eps = base_eps / |theta| ~ 1e-9
                              is below float32 resolution, so this approach always runs the float64 kernels
subsample_factor < 1 (:235-245): the products use a random subset of the batch, drawn with np.random.choice like the
reference but at the granularity of the kernels' 128-sample tiles.

Multi-GPU: every reduction vector is made global by ONE collective (Comm.all_reduce_mixed) before use -- the flat
gradient travels together with the (loss, mean KL | max KL) triple of the same pass.
"""
import numpy as np

from .. import _lib as L
from ..misc import logger


class PerlmutterHvp(object):
    """Marker for the exact Hessian-vector product (conjugate_gradient_optimizer.py:22-55); the default."""

    def __init__(self, num_slices=1):
        self._num_slices = num_slices


class FiniteDifferenceHvp(object):
    """conjugate_gradient_optimizer.py:58-115 (same constructor)."""

    def __init__(self, base_eps=1e-8, symmetric=True, grad_clip=None, num_slices=1):
        self.base_eps = base_eps
        self.symmetric = symmetric
        self.grad_clip = grad_clip
        self._num_slices = num_slices


class ConjugateGradientOptimizer(object):
    def __init__(self, cg_iters=10, reg_coeff=1e-5, subsample_factor=1., backtrack_ratio=0.8, max_backtracks=15,
                 accept_violation=False, hvp_approach=None, num_slices=1, residual_tol=1e-10,
                 use_activation_cache=True, precision="f32", cg_direction_f32=False):
        if not (0.0 < subsample_factor <= 1.0):
            raise ValueError("subsample_factor must be in (0, 1]")
        if hvp_approach is not None and not isinstance(hvp_approach, (PerlmutterHvp, FiniteDifferenceHvp)):
            raise TypeError("hvp_approach must be PerlmutterHvp() or FiniteDifferenceHvp()")
        if precision not in ("f32", "f64"):
            raise ValueError("precision must be 'f32' (fast path) or 'f64' (parity mode)")
        self._cg_iters = cg_iters
        self._reg_coeff = reg_coeff
        self._subsample_factor = subsample_factor
        self._backtrack_ratio = backtrack_ratio
        self._max_backtracks = max_backtracks
        self._accept_violation = accept_violation
        self._residual_tol = residual_tol
        self._hvp = hvp_approach
        self._fd = isinstance(hvp_approach, FiniteDifferenceHvp)
        self._target = None
        self._max_constraint_val = None
        self._constraint_name = None
        self._loss_kind = L.LOSS_TRPO
        self._comm = None
        self._bufs = None
        self._cache = None     # (policy version, batch id) -> (loss, mean_kl, max_kl)
        self._g_key = None     # key for which the `g` buffer holds the flat gradient
        self._hc_key = None    # key for which the batch's activation cache is valid
        self._f64 = precision == "f64"
        self._use_hcache = use_activation_cache and not self._f64
        self._p_f32 = bool(cg_direction_f32) and not self._f64
        self.last_info = {}

    def __getstate__(self):
        return _drop_device_state(self.__dict__, ("_bufs", "_cache", "_g_key", "_hc_key", "_comm"))

    def update_opt(self, loss, target, leq_constraint, inputs=None, extra_inputs=None, constraint_name="constraint",
                   comm=None, *args, **kwargs):
        constraint_term, constraint_value = leq_constraint
        self._loss_kind = loss
        self._target = target
        self._max_constraint_val = constraint_value
        self._constraint_name = constraint_name
        self._comm = comm

    # ---- helpers
    def _buffers(self, P, dev):
        import torch
        if self._bufs is None or self._bufs["g"].numel() != P or self._bufs["g"].device != dev:
            z = lambda n=P: torch.zeros(n, dtype=torch.float64, device=dev)
            gl = z(P + 3)                       # [flat gradient | loss, sum KL | max KL]: one collective for all of it
            self._bufs = dict(gl=gl, g=gl[:P], gout=gl[P:], x=z(), r=z(), p=z(), z=z(), Hx=z(), step=z(), prev=z(),
                              st=z(4), info=z(2), out=z(3), tmp=z(), tmp2=z(), cnt=z(1),
                              scratch32=torch.zeros(P, dtype=torch.float32, device=dev))
        return self._bufs

    def _world(self):
        return self._comm.world_size if (self._comm is not None and self._comm.active) else 1

    def _reduce(self, t, n_sum=None):
        if self._world() > 1:
            self._comm.all_reduce_mixed(t, t.numel() if n_sum is None else n_sum)

    def _fuse(self):
        """Update passes reduce over ranks inside their own finalize kernel (peer-memory transport, csrc/peer.cuh)."""
        return self._world() > 1 and self._comm.fuse

    def _after_pass(self, t, n_sum=None):
        """Make the output of an update pass launched with fuse=self._fuse() global (no-op when it was fused)."""
        if self._world() > 1:
            self._comm.after_pass(t, t.numel() if n_sum is None else n_sum)

    def _eval(self, batch, want_grad=False):
        """surrogate loss, mean KL, max KL at the target's current parameters (one pass over the batch).
        want_grad: run the gradient pass instead, which yields the same triple for free and leaves the flat
        gradient in the `g` buffer (f_loss + f_grad of cg_opt.py:248,253 fused into one pass)."""
        from .. import ops
        pol = self._target
        key = (pol.version, id(batch), batch.version)
        if self._cache is not None and self._cache[0] == key:
            return self._cache[1]
        b = self._buffers(pol.n_params, batch.device)
        P = pol.n_params
        if want_grad:
            if self._f64:
                ops.update_f64(1, self._loss_kind, pol.theta64, pol.dims, pol.min_std, batch, None, 0.0, 0.0, b["g"],
                               b["gout"], fuse=self._fuse())
            else:
                hc = batch.hcache(pol.h1, pol.h2) if self._use_hcache else None
                ops.grad(self._loss_kind, pol.theta32, pol.dims, pol.min_std, batch, b["g"], b["gout"], hc,
                         fuse=self._fuse())
                self._hc_key = key if hc is not None else None
            self._after_pass(b["gl"], P + 2)
            self._g_key = key
            src = b["gout"]
        else:
            if self._f64:
                ops.update_f64(0, self._loss_kind, pol.theta64, pol.dims, pol.min_std, batch, None, 0.0, 0.0, None,
                               b["out"], fuse=self._fuse())
            else:
                ops.loss_kl(self._loss_kind, pol.theta32, pol.dims, pol.min_std, batch, b["out"], fuse=self._fuse())
            self._after_pass(b["out"], 2)
            src = b["out"]
        vals = ops.LazyTriple(src)            # pinned-memory readback queued behind the pass; blocks when indexed
        self._cache = (key, vals)
        return vals

    def eval_lazy(self, inputs, want_grad=True):
        """The (loss, mean_kl, max_kl) triple as a lazily read ops.LazyTriple (see FirstOrderOptimizer.eval_lazy)."""
        return self._eval(_lane_batch(inputs), want_grad=want_grad)

    def loss(self, inputs, extra_inputs=None):
        return self._eval(_lane_batch(inputs), want_grad=True)[0]

    def constraint_val(self, inputs, extra_inputs=None):
        return self._eval(_lane_batch(inputs), want_grad=True)[1]

    def _draw_subsample(self, batch, b):
        """np.random.choice of int(n_tiles * factor) tiles of 128 samples (conjugate_gradient_optimizer.py:235-245 at tile
        granularity; every rank draws its own subset of its own lanes) and the number of valid samples in it."""
        import torch
        from .. import ops
        n_tiles = -(-batch.B // 128)
        k = max(1, int(n_tiles * self._subsample_factor))
        inds = np.sort(np.random.choice(n_tiles, k, replace=False)).astype(np.int32)
        tiles = torch.as_tensor(inds).to(batch.device)
        ops.count_valid(batch, tiles, b["cnt"])
        self._reduce(b["cnt"])
        self.last_subsample = inds
        return tiles

    def _make_Hx(self, batch, b, hcache, tiles):
        from .. import ops
        pol = self._target
        world = self._world()
        if self._fd:
            # FiniteDifferenceHvp.f_Hx_plain (:77-97): gradients of mean KL at theta +- eps x, float64 kernels
            hv = self._hvp
            theta = pol.theta64
            eps = float(np.float32(hv.base_eps / (float(theta.norm().item()) + 1e-8)))

            def grad_kl(sign, vec, out):
                ops.axpy_params(theta, vec, -sign * eps, b["tmp2"], b["scratch32"])      # theta + sign * eps * x
                ops.update_f64(1, L.LOSS_KL, b["tmp2"], pol.dims, pol.min_std, batch, None, 0.0, 0.0, out, None,
                               fuse=self._fuse())

            def Hx(vec, out):
                grad_kl(+1.0, vec, out)
                if hv.symmetric:
                    grad_kl(-1.0, vec, b["tmp"])
                    out.sub_(b["tmp"]).div_(2.0 * eps)
                else:
                    grad_kl(0.0, vec, b["tmp"])
                    out.sub_(b["tmp"]).div_(eps)
                self._after_pass(out)               # both gradients were made global by their own passes when fused
                out.add_(vec, alpha=self._reg_coeff)
            return Hx

        def Hx(vec, out):
            if self._f64:
                ops.update_f64(2, self._loss_kind, pol.theta64, pol.dims, pol.min_std, batch, vec, self._reg_coeff,
                               1.0 / world, out, None, fuse=self._fuse())
            else:
                ops.fvp(pol.theta32, pol.dims, pol.min_std, batch, vec, self._reg_coeff, 1.0 / world, out, hcache,
                        tiles, b["cnt"] if tiles is not None else None, fuse=self._fuse())
            self._after_pass(out)
        return Hx

    def optimize(self, inputs, extra_inputs=None, subsample_grouped_inputs=None):
        from .. import ops
        batch = _lane_batch(inputs)
        pol = self._target
        P = pol.n_params
        b = self._buffers(P, batch.device)

        tiles = None
        if self._subsample_factor < 1:
            if self._f64 or self._fd:
                raise NotImplementedError("subsample_factor < 1 is built for the float32 Fisher-vector kernels")
            if ops.is_gru(pol.dims):
                raise NotImplementedError("subsample_factor < 1 is not built for a recurrent policy (the reference "
                                          "sub-samples whole paths, not 128-sample tiles)")
            tiles = self._draw_subsample(batch, b)

        logger.log("computing loss before")
        before = self._eval(batch, want_grad=True)      # read back at the line search, after the CG solve is queued
        logger.log("performing update")
        logger.log("computing descent direction")
        key0 = (pol.version, id(batch), batch.version)
        assert self._g_key == key0
        hcache = batch.hcache(pol.h1, pol.h2) if (self._use_hcache and self._hc_key == key0) else None
        Hx = self._make_Hx(batch, b, hcache, tiles)

        ops.cg_init(b["g"], b["x"], b["r"], b["p"], b["st"], self._p_f32)
        for _ in range(self._cg_iters):
            Hx(b["p"], b["z"])
            ops.cg_step(b["z"], b["x"], b["r"], b["p"], b["st"], self._residual_tol, self._p_f32)
        Hx(b["x"], b["Hx"])
        ops.trpo_step_size(b["x"], b["Hx"], self._max_constraint_val, b["step"], b["info"])
        logger.log("descent direction computed")

        ops.axpy_params(pol.theta64, b["step"], 0.0, b["prev"], b["scratch32"])          # prev = theta
        loss_before = before[0]
        n_iter = 0
        loss = constraint_val = np.nan
        for n_iter, ratio in enumerate(self._backtrack_ratio ** np.arange(self._max_backtracks)):
            ops.axpy_params(b["prev"], b["step"], ratio, pol.theta64, pol.theta32)
            pol.bump_version()
            loss, constraint_val, _ = self._eval(batch)
            if loss < loss_before and constraint_val <= self._max_constraint_val:
                break
        rejected = False
        if (np.isnan(loss) or np.isnan(constraint_val) or loss >= loss_before or
                constraint_val >= self._max_constraint_val) and not self._accept_violation:
            logger.log("Line search condition violated. Rejecting the step!")
            if np.isnan(loss):
                logger.log("Violated because loss is NaN")
            if np.isnan(constraint_val):
                logger.log("Violated because constraint %s is NaN" % self._constraint_name)
            if loss >= loss_before:
                logger.log("Violated because loss not improving")
            if constraint_val >= self._max_constraint_val:
                logger.log("Violated because constraint %s is violated" % self._constraint_name)
            ops.axpy_params(b["prev"], b["step"], 0.0, pol.theta64, pol.theta32)
            pol.bump_version()
            rejected = True
        logger.log("backtrack iters: %d" % n_iter)
        logger.log("computing loss after")
        logger.log("optimization finished")
        self.last_info = dict(loss_before=loss_before, loss=loss, constraint_val=constraint_val, n_iter=n_iter,
                              rejected=rejected)


def _drop_device_state(obj_dict, keys):
    d = dict(obj_dict)
    for k in keys:
        d[k] = None
    return d


def _lane_batch(inputs):
    if hasattr(inputs, "lane_batch"):
        return inputs.lane_batch
    if isinstance(inputs, dict) and "lane_batch" in inputs:
        return inputs["lane_batch"]
    if hasattr(inputs, "obs") and hasattr(inputs, "B_global"):
        return inputs
    raise TypeError("the B200 optimizers take the device sample batch (samples_data or its lane_batch) as `inputs`; "
                    "host arrays would need a host->device copy of the whole batch every call")
