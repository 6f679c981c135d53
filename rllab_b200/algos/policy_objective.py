"""The policy objective of the L-BFGS policy updates (PPO = NPO + PenaltyLbfgsOptimizer, ERWR = VPG + LbfgsOptimizer):
the callables the host optimizers take, each running one device pass over the sample batch at the policy's current
parameters.

  f_loss(batch), f_constraint(batch)   surrogate loss / mean KL(old || new) of the loss pass (b200rl_loss_kl)
  f_opt(batch, penalty=0)              (loss + penalty * mean KL, flat gradient of it) as float64, from one
                                       b200rl_grad_penalized pass (b200rl_grad when the penalty is 0); the pass also
                                       yields the unpenalised (loss, mean KL, max KL) triple
  f_penalized_loss(batch, penalty)     (loss + penalty * mean KL, loss, mean KL) from the triple of the last f_opt pass
                                       at the same (parameters, batch) -- the point scipy evaluated last, which is the
                                       one the reference evaluates (penalty_lbfgs_optimizer.py:114) -- else a loss pass

Replaces the compiled f_opt / f_penalized_loss of rllab/optimizers/penalty_lbfgs_optimizer.py:42-78 over the NPO
surrogate (npo.py:72-98) and f_opt of lbfgs_optimizer.py:20-45 over the VPG surrogate (vpg.py:88-99).  The penalised
value is formed on the host in float64; NaN / inf propagate unchanged (the penalty adaptation keys on NaN).

Multi-GPU: the [gradient | loss, sum KL | max KL] vector of each pass is reduced over the ranks (fused into the pass on
the peer-memory transport, else by one collective after it), so every rank hands scipy identical numbers and theta stays
bit-identical across ranks.
"""
import numpy as np

from ..optimizers.conjugate_gradient_optimizer import _lane_batch


class PolicyObjective(object):
    def __init__(self, policy, loss_kind, comm=None):
        self._policy = policy
        self._loss_kind = loss_kind
        self._comm = comm
        self._bufs = None
        self._loss_cache = None      # (key, LazyTriple) of the last loss pass
        self._grad_triple = None     # (key, (loss, mean KL, max KL)) of the last gradient pass
        self.n_evals = 0             # gradient passes (L-BFGS function evaluations) so far

    def __getstate__(self):
        d = dict(self.__dict__)
        d.update(_bufs=None, _loss_cache=None, _grad_triple=None, _comm=None)
        return d

    def _active(self):
        return self._comm is not None and self._comm.active

    def _buffers(self, dev):
        import torch
        P = self._policy.n_params
        if self._bufs is None or self._bufs["gl"].device != dev:
            gl = torch.zeros(P + 3, dtype=torch.float64, device=dev)   # [gradient | loss, sum KL | max KL]
            self._bufs = dict(gl=gl, g=gl[:P], tri=gl[P:], out=torch.zeros(3, dtype=torch.float64, device=dev))
        return self._bufs

    def _key(self, batch):
        return (self._policy.version, id(batch), batch.version)

    def eval_lazy(self, inputs):
        """(loss, mean KL, max KL) of the loss pass at the current parameters, read back lazily (ops.LazyTriple)."""
        from .. import ops
        batch = _lane_batch(inputs)
        key = self._key(batch)
        if self._loss_cache is not None and self._loss_cache[0] == key:
            return self._loss_cache[1]
        pol = self._policy
        b = self._buffers(batch.device)
        fuse = self._active() and self._comm.fuse
        ops.loss_kl(self._loss_kind, pol.theta32, pol.dims, pol.min_std, batch, b["out"], fuse=fuse)
        if self._active():
            self._comm.after_pass(b["out"], 2)
        vals = ops.LazyTriple(b["out"])
        self._loss_cache = (key, vals)
        return vals

    def f_loss(self, batch):
        return self.eval_lazy(batch)[0]

    def f_constraint(self, batch):
        return self.eval_lazy(batch)[1]

    def kl_stats(self, batch):
        """(mean KL, max KL): f_kl of vpg.py:100-103, from the same pass as the loss."""
        v = self.eval_lazy(batch)
        return v[1], v[2]

    def f_opt(self, batch, penalty=0.0):
        from .. import ops
        batch = _lane_batch(batch)
        pol = self._policy
        P = pol.n_params
        b = self._buffers(batch.device)
        fuse = self._active() and self._comm.fuse
        if penalty == 0:
            ops.grad(self._loss_kind, pol.theta32, pol.dims, pol.min_std, batch, b["g"], b["tri"], fuse=fuse)
        else:
            ops.grad_penalized(self._loss_kind, penalty, pol.theta32, pol.dims, pol.min_std, batch, b["g"], b["tri"],
                               fuse=fuse)
        if self._active():
            self._comm.after_pass(b["gl"], P + 2)
        h = b["gl"].cpu().numpy()
        self.n_evals += 1
        loss, mean_kl, max_kl = (float(x) for x in h[P:])
        self._grad_triple = (self._key(batch), (loss, mean_kl, max_kl))
        return loss + penalty * mean_kl, np.array(h[:P], dtype=np.float64)

    def f_penalized_loss(self, batch, penalty):
        batch = _lane_batch(batch)
        if self._grad_triple is not None and self._grad_triple[0] == self._key(batch):
            loss, mean_kl, _ = self._grad_triple[1]
        else:
            loss, mean_kl, _ = self.eval_lazy(batch)
        return loss + penalty * mean_kl, loss, mean_kl
