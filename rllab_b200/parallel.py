"""Multi-GPU plumbing: one process per GPU (torchrun), lanes sharded by rank, all-reduce of the small float64 reduction
vectors (gradient, FVP, loss/KL scalars, advantage statistics, baseline normal equations) over NVLink/NVSwitch.

torch.distributed (NCCL) is the rendezvous and the fallback transport.  The data path on a multi-GPU box is the library's own
peer-memory exchange (csrc/peer.cuh): every rank maps every other rank's exchange window (CUDA IPC), and one kernel per
reduction pushes the vector through NVLink into all windows and folds the `world` copies in rank order -- fused into the
finalize kernel of the policy-update passes (gradient, Fisher-vector product, loss/KL), stand-alone for the statistics
and the baseline normal equations.  No NCCL call remains on the iteration's critical path.

The reference has no counterpart (its update is single-process; SURVEY.md 2b): this is row (e) of the scope table.  With
world_size == 1 every method is a no-op (no communicator is created)."""
import ctypes
import os

PEER_SLOT_DOUBLES = 8192          # >= P + 3 of the largest compiled-in policy (5 702) and every statistics vector


class Comm(object):
    def __init__(self, backend=None):
        import torch
        import torch.distributed as dist
        self.dist = dist
        self.world_size = int(os.environ.get("WORLD_SIZE", "1"))
        self.rank = int(os.environ.get("RANK", "0"))
        self.local_rank = int(os.environ.get("LOCAL_RANK", "0"))
        self.active = self.world_size > 1
        self._gather_bufs = {}
        self.n_collectives = 0            # NCCL / gloo collectives issued
        self.n_peer_exchanges = 0         # peer-memory exchanges (stand-alone kernels + fused into update passes)
        self._owns_group = False
        self.peer = False                 # peer-memory transport bound (CUDA + every rank on one NVLink domain)
        self._windows = None
        if self.active and not dist.is_initialized():
            self._owns_group = True
            if backend is None:
                backend = "nccl" if torch.cuda.is_available() else "gloo"
            kw = {}
            if backend == "nccl":
                torch.cuda.set_device(self.local_rank)
                kw["device_id"] = torch.device("cuda", self.local_rank)
            dist.init_process_group(backend=backend, **kw)
        if self.active and torch.cuda.is_available() and dist.get_backend() == "nccl" \
                and os.environ.get("B200RL_PEER", "1") != "0":
            self._bind_peer_windows()

    # ---- peer-memory transport
    def _bind_peer_windows(self):
        """Create this rank's exchange window, swap IPC handles through the process group, map the peers' windows and
        bind the communicator in the library.  Any failure (no peer access between the GPUs, IPC disabled in the
        container) leaves the NCCL transport in place -- agreed on by all ranks, so nobody waits on a window."""
        import torch
        from . import _lib as L
        from .misc import logger
        L.load()
        w, r = self.world_size, self.rank
        own, handle, opened, err = ctypes.c_void_p(), (ctypes.c_ubyte * 64)(), {}, None
        try:
            L.call("b200rl_peer_window_create", w, PEER_SLOT_DOUBLES, ctypes.byref(own), handle)
        except RuntimeError as exc:
            err = str(exc)
        handles = [None] * w
        self.dist.all_gather_object(handles, None if err else bytes(handle))
        if err is None and all(h is not None for h in handles):
            try:
                for q, h in enumerate(handles):
                    if q != r:
                        ptr = ctypes.c_void_p()
                        L.call("b200rl_peer_window_open", (ctypes.c_ubyte * 64).from_buffer_copy(h), ctypes.byref(ptr))
                        opened[q] = ptr
            except RuntimeError as exc:
                err = str(exc)
        else:
            err = err or "a peer could not create its window"
        oks = [None] * w
        self.dist.all_gather_object(oks, err is None)
        if all(oks):
            table = (ctypes.c_void_p * w)(*[own if q == r else opened[q] for q in range(w)])
            L.call("b200rl_peer_bind", table, r, w, PEER_SLOT_DOUBLES)
            self._windows = (own, opened)
            self.peer = True
        else:
            for ptr in opened.values():
                L.call("b200rl_peer_window_close", ptr)
            if own.value:
                L.call("b200rl_peer_window_destroy", own)
            if r == 0:
                logger.log("peer-memory transport unavailable (%s): NCCL all-gather path" % (err or "a peer failed"))
        torch.cuda.synchronize()
        self.dist.barrier()

    def peer_timeouts(self):
        """Collectives of this rank that gave up waiting for a peer (synchronising read; 0 without the peer transport)."""
        if not self.peer:
            return 0
        from . import _lib as L
        n = ctypes.c_uint(0)
        L.call("b200rl_peer_timeouts", ctypes.byref(n))
        return int(n.value)

    @property
    def fuse(self):
        """True when the update passes should reduce over ranks inside their own finalize kernel."""
        return self.active and self.peer

    def after_pass(self, t, n_sum):
        """Make the output of an update pass global: nothing to do when the pass was launched with fuse=True (the
        exchange happened inside its finalize kernel), one mixed all-reduce otherwise."""
        if self.fuse:
            self.n_peer_exchanges += 1
            return t
        return self.all_reduce_mixed(t, n_sum)

    def all_reduce_sum(self, t):
        if self.active:
            if self.peer and t.is_cuda:
                return self.all_reduce_mixed(t, t.numel())
            self.dist.all_reduce(t, op=self.dist.ReduceOp.SUM)
            self.n_collectives += 1
        return t

    def all_reduce_max(self, t):
        if self.active:
            self.dist.all_reduce(t, op=self.dist.ReduceOp.MAX)
        return t

    def all_reduce_mixed(self, t, n_sum):
        """In place: t[:n_sum] summed over ranks, t[n_sum:] maximised over ranks, with ONE collective: an all-gather of
        the whole vector followed by a local fixed-order reduction (b200rl_reduce_ranks).  Every reduction vector of an
        iteration is a few KB, so the cost of a collective is its launch latency, not its bytes: gathering world x n
        doubles instead of reducing n costs nothing extra, halves the number of collectives for vectors that carry sums
        and maxima (statistics; loss / KL triples), and makes the summation order rank order by construction -- every
        rank computes bit-identical results whatever algorithm NCCL picks."""
        if not self.active:
            return t
        import torch
        n = t.numel()
        if self.peer and t.is_cuda and t.dtype == torch.float64 and t.is_contiguous() and n <= PEER_SLOT_DOUBLES:
            from . import ops
            ops.peer_allreduce_mixed(t, n_sum)
            self.n_peer_exchanges += 1
            return t
        key = (n, t.device, t.dtype)
        buf = self._gather_bufs.get(key)
        if buf is None:
            buf = torch.empty(self.world_size * n, dtype=t.dtype, device=t.device)
            self._gather_bufs[key] = buf
        self.dist.all_gather_into_tensor(buf, t)
        self.n_collectives += 1
        if t.is_cuda:
            from . import ops
            ops.reduce_ranks(buf, self.world_size, n, n_sum, t)
        else:                    # CPU tensors only occur in the gloo tests of this plumbing (no kernels involved)
            g = buf.view(self.world_size, n)
            t[:n_sum] = g[:, :n_sum].sum(0)
            if n_sum < n:
                t[n_sum:] = g[:, n_sum:].max(0).values
        return t

    def barrier(self):
        if self.active:
            self.dist.barrier()

    def close(self):
        """Unbind the peer windows and tear the process group down (NCCL warns at exit otherwise); the group only if
        this object created it."""
        if self.peer:
            import torch
            from . import _lib as L
            torch.cuda.synchronize()
            self.dist.barrier()                      # nobody still pushes into a window that is about to go away
            n_timeouts = self.peer_timeouts()
            L.call("b200rl_peer_bind", None, 0, 0, 0)
            own, opened = self._windows
            for ptr in opened.values():
                L.call("b200rl_peer_window_close", ptr)
            L.call("b200rl_peer_window_destroy", own)
            self.peer, self._windows = False, None
        else:
            n_timeouts = 0
        if self.active and self._owns_group and self.dist.is_initialized():
            self.dist.destroy_process_group()
            self._owns_group = False
        if n_timeouts:
            raise RuntimeError("%d peer-memory collective(s) of rank %d timed out waiting for a peer; their results were "
                               "NaN" % (n_timeouts, self.rank))

    def shard(self, n_total):
        """Contiguous lane block of this rank: lane i -> GPU floor(i*G/N) (SURVEY 8e)."""
        per = n_total // self.world_size
        rem = n_total % self.world_size
        n = per + (1 if self.rank < rem else 0)
        lane0 = self.rank * per + min(self.rank, rem)
        return n, lane0


_default = None


def default_comm():
    global _default
    if _default is None:
        _default = Comm()
    return _default
