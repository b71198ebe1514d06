"""The ``sync=`` argument of the fused BatchNorm ops: what a synchronised BatchNorm needs to reach the other ranks.

With a handle, the fused ops (``bn_act``, ``conv1x1_bn_act``, ``bn_relu_maxpool``, ``stem_conv_bn_relu_maxpool``) combine
their per-channel sums across the data-parallel ranks (``csrc/sync_bn.cu``) and normalise with the statistics of the
global batch, as ``torch.nn.SyncBatchNorm`` does.  ``sync=None`` (or a world of 1) is the unsynchronised op.

* Fused communicator: the handle owns an exchange area of the symmetric arena (same offset on every rank), its own
  signal channel and a device call counter, so the exchange replays inside CUDA graphs.
* Any other communicator (``--comm nccl|gloo``): the CPU emulation of the kernels sums the statistics with the
  communicator's ``all_reduce_``, and layers the fused kernels cannot take run ``torch.nn.SyncBatchNorm``'s autograd
  function over the process group.
"""
from __future__ import annotations

import torch


def sync_work_len(c: int) -> int:
    """floats of a synchronised work slice: [local 2C sums | global 2C sums | global row count (int64)] (csrc/host.h)."""
    return 4 * c + 4


def work_len(c: int, sync) -> int:
    """floats one direction (forward or backward) of a fused BatchNorm layer takes from the step workspace."""
    return sync_work_len(c) if sync is not None else 2 * c


def effective(sync, training: bool):
    """``sync`` when the layer has something to synchronise (training-mode statistics, more than one rank), else None."""
    return None if sync is None or not training or sync.world == 1 else sync


def kernel_arg(sync, kernels):
    """The ``sync`` argument of an entry point of the kernel module ``kernels`` (``SyncContext.kernel_arg``; None: unsynchronised)."""
    return None if sync is None else sync.kernel_arg(kernels)


class SyncContext:
    """One per communicator; every synchronised layer of the process shares it (the exchanges run in layer order on
    the compute stream, the same order on every rank)."""

    def __init__(self, comm, native=None, calls=None):
        self.comm = comm
        self.world = comm.world
        self.native = native         # _C.SyncBN on the fused communicator, else None
        self.calls = calls           # keeps the device call counters alive

    @classmethod
    def for_communicator(cls, comm) -> "SyncContext":
        ctx = getattr(comm, "_sync_bn_ctx", None)
        if ctx is None:
            native = calls = None
            if getattr(comm, "backend", "") == "fused":
                C = comm._C
                xoff = comm.alloc(C.SYNC_BN_AREA_BYTES)
                channel = comm.new_channel()
                if comm.world > 1:     # the protocol needs the area at one offset on every rank: a mismatch is an error, not a hang
                    got = comm._gather_obj((xoff, channel))
                    if any(g != got[0] for g in got):
                        raise RuntimeError("synchronised BatchNorm: exchange area / channel differ across ranks %s; bind the "
                                           "layers at the same point of the program on every rank" % (got,))
                calls = torch.zeros(C.MAX_BLOCKS, dtype=torch.int32, device=comm.device)
                native = comm.arena.sync_bn(channel, xoff, calls.data_ptr())
            ctx = cls(comm, native, calls)
            comm._sync_bn_ctx = ctx
        return ctx

    def kernel_arg(self, kernels):
        """What the kernel module takes as ``sync``: the native handle, or this context for the PyTorch emulation."""
        if getattr(kernels, "is_emulation", False):
            return self
        if self.native is None:
            raise RuntimeError("synchronised BatchNorm on CUDA tensors needs the fused communicator (--comm fused); with "
                               "--comm %s the layers run torch.nn.SyncBatchNorm" % getattr(self.comm, "backend", "?"))
        return self.native

    def all_reduce_sum_(self, t: torch.Tensor) -> torch.Tensor:
        self.comm.all_reduce_([t], average=False, wire="fp32")
        return t
