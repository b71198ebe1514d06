"""Reference-compatible helpers on top of the communicators.

``reduce_mean(tensor, nprocs)`` is the function every multi-process reference script defines
(/root/reference/distributed.py:105-109): clone -> all_reduce(SUM) -> divide.  Here scalars (<= 8 floats) take the
low-latency peer-memory path (one kernel, flag travels with the payload); larger tensors use the fused all-reduce;
without a fused communicator it falls back to ``torch.distributed``.  ``nprocs`` is accepted for signature parity but
the divisor is the real world size (SURVEY Q7).
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.distributed as dist

_default_comm = None


def set_default_communicator(comm) -> None:
    global _default_comm
    _default_comm = comm


def default_communicator():
    """The communicator synchronised BatchNorm layers bind to: the one registered for this process (this package's DDP
    and apex DDP register theirs when the model has synchronised layers), else ``hvd.init()``'s, else None."""
    if _default_comm is not None:
        return _default_comm
    from ..parallel import hvd
    return hvd.communicator() if hvd.is_initialized() else None


def register_for_sync_batchnorm(module, comm) -> None:
    """Register ``comm`` for the synchronised BatchNorm layers of ``module`` (if it has any and none is registered yet)."""
    from ..models.resnet import SyncBNAct
    if _default_comm is None and any(isinstance(m, SyncBNAct) for m in module.modules()):
        set_default_communicator(comm)


def reduce_mean(tensor: torch.Tensor, nprocs: Optional[int] = None, comm=None) -> torch.Tensor:
    rt = tensor.detach().clone()
    comm = comm or _default_comm
    if comm is not None and comm.world > 1:
        if getattr(comm, "backend", "") == "fused" and rt.is_cuda:
            if rt.dtype == torch.float32 and rt.numel() <= 8:
                comm.reduce_scalars_(rt.reshape(-1) if rt.dim() == 0 else rt, average=True)
            else:
                comm.all_reduce_([rt], average=True)
        else:
            comm.reduce_scalars_(rt, average=True)
        return rt
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(rt, op=dist.ReduceOp.SUM)
        rt /= dist.get_world_size()
    return rt


def barrier(comm=None) -> None:
    comm = comm or _default_comm
    if comm is not None:
        comm.barrier()
    elif dist.is_available() and dist.is_initialized():
        dist.barrier()
