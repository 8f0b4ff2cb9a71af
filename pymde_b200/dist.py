"""Edge-sharded multi-GPU solve (SURVEY section 8e): one process per GPU, edges split across ranks,
X replicated, and ONE all-reduce of [gradient | loss] per evaluation over NVLink.

E and grad E are sums over edges (pymde/average_distortion.py:51,77-78), so each rank runs the
same fused kernel on its shard with the GLOBAL edge count as divisor; after the all-reduce
every rank holds bit-identical gradient and loss, the device-resident L-BFGS state is
replicated and (thanks to fixed-order reductions) takes identical decisions on every rank.

Two transports for the solver's all-reduce:
  * peer memory (default): the library's own kernels sum the ranks' partial buffers over
    NVLink (cudaIpc-mapped, flag handshake, rank-ordered sums) inside the same CUDA graph as the
    rest of the step.  `torch.distributed` is used ONCE, to exchange the 64-byte IPC handles.
  * host hook (`make_allreduce`): an NCCL all-reduce enqueued from Python between two kernels --
    the transport used when no exchange function is given (ranks without cudaIpc peer access).
Evaluations outside the solver (`MDE.average_distortion`, gradients through autograd) are
all-reduced with `torch.distributed` so that a sharded MDE behaves like the global problem."""
import os

import torch
import torch.distributed as dist

from . import _lib


def shard_range(p, rank, world):
    """Contiguous edge range [lo, hi) of `rank` (balanced to within one edge)."""
    base, rem = divmod(int(p), int(world))
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


class _Wrap(object):
    def __init__(self, ptr, count):
        self.__cuda_array_interface__ = {"shape": (int(count),), "typestr": "<f4", "data": (int(ptr), False),
                                         "version": 3}


def make_allreduce(device, group=None):
    """ctypes-callable (user, buf, count, stream) -> int doing an in-place NCCL sum on torch's
    current stream (the solver enqueues on that same stream)."""
    cache = {}

    def cb(user, buf, count, stream):
        try:
            key = (buf, count)
            t = cache.get(key)
            if t is None:
                with torch.cuda.device(device):
                    t = torch.as_tensor(_Wrap(buf, count), device=device)
                cache[key] = t
            dist.all_reduce(t, op=dist.ReduceOp.SUM, group=group)
            return 0
        except Exception:  # never let an exception cross the C boundary
            import traceback
            traceback.print_exc()
            return _lib.MDE_E_INVALID

    return cb


def pack_handles(chunks):
    """[bytes (64 each), ...] in rank order -> one bytes object (what mde_solver_comm_connect reads)."""
    for c in chunks:
        if len(c) != _lib.IPC_HANDLE_BYTES:
            raise ValueError("an IPC handle is %d bytes, got %d" % (_lib.IPC_HANDLE_BYTES, len(c)))
    return b"".join(chunks)


def make_exchange(device=None, group=None):
    """exchange(my_handle: bytes) -> bytes of all ranks' handles in rank order (an all-gather of 64 bytes).
    Works on any backend: NCCL gathers a CUDA uint8 tensor, gloo a CPU one."""

    def exchange(mine):
        world = dist.get_world_size(group)
        backend = dist.get_backend(group)
        dev = torch.device(device) if (device is not None and backend == "nccl") else torch.device("cpu")
        t = torch.tensor(list(mine), dtype=torch.uint8, device=dev)
        out = [torch.empty_like(t) for _ in range(world)]
        dist.all_gather(out, t, group=group)
        return pack_handles([bytes(o.cpu().tolist()) for o in out])

    return exchange


def allreduce_evaluation(loss, grad, group=None):
    """Sum a shard's (loss sum, gradient) across ranks in place (evaluations outside the solver)."""
    if grad is not None:
        dist.all_reduce(grad, op=dist.ReduceOp.SUM, group=group)
    dist.all_reduce(loss, op=dist.ReduceOp.SUM, group=group)


def attach(mde, rank, world_size, p_total, device, group=None, transport=None):
    """Mark `mde` (built over this rank's edge shard) as one shard of a `p_total`-edge problem."""
    if world_size <= 1:
        return mde
    transport = transport or os.environ.get("PYMDE_B200_ALLREDUCE", "peer")
    d = {"rank": int(rank), "world_size": int(world_size), "p_total": int(p_total), "group": group}
    if transport == "peer":
        d["exchange"] = make_exchange(device, group)
    else:
        d["allreduce"] = make_allreduce(torch.device(device), group)
    mde.__dict__["_dist"] = d
    return mde


def shard_mde(mde_cls, n_items, embedding_dim, edges, make_function, constraint, device, rank=None,
              world_size=None, group=None, transport=None):
    """Build this rank's MDE over its edge shard.

    edges: full (p,2) int64 tensor (host or device); make_function(lo, hi) -> distortion function
    for edges[lo:hi].  The returned MDE is global: `average_distortion` (value and gradient) and
    `embed()` act on the whole edge set; `distances()/distortions()` return this rank's shard."""
    rank = dist.get_rank(group) if rank is None else rank
    world_size = dist.get_world_size(group) if world_size is None else world_size
    p = int(edges.shape[0])
    lo, hi = shard_range(p, rank, world_size)
    mde = mde_cls(n_items, embedding_dim, edges[lo:hi].to(device), make_function(lo, hi), constraint, device=device)
    return attach(mde, rank, world_size, p, device, group, transport)
