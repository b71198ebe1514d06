"""``apex.parallel.DistributedDataParallel(model)`` equivalent (/root/reference/apex_distributed.py:217).

apex's wrapper takes no ``device_ids``, learns its buckets (``message_size`` elements, default 1e7) from gradient
arrival and all-reduces flat buffers on a side stream.  Here it is a thin front over the same
:class:`~pytorch_distributed_b200.parallel.ddp.GradientEngine` as our DDP: fixed reverse-order buckets of
``message_size`` elements, the fused peer-memory kernel, fp16/bf16 wire chosen from the amp state, and - when amp's
dynamic loss scaling is on - the non-finite test folded into the all-reduce so all ranks skip the same steps.
"""
from __future__ import annotations

from contextlib import contextmanager

import torch
import torch.nn as nn

from ...parallel import amp as _amp
from ...parallel.comm import make_communicator
from ...parallel.ddp import GradientEngine, _float_buffers, sync_module_states
from ...utils.dist_ops import register_for_sync_batchnorm
from ...models.resnet import SyncBNAct, convert_sync_batchnorm
from .LARC import LARC  # noqa: F401  (apex.parallel.LARC; the submodule stays importable as apex.parallel.LARC)

_WIRE = {torch.float16: "fp16", torch.bfloat16: "bf16", torch.float32: "fp32"}


class DistributedDataParallel(nn.Module):
    """apex.parallel.DistributedDataParallel arguments and what they do here:

    ``message_size``              bucket size in ELEMENTS (apex default 1e7), fixed reverse-order buckets
    ``delay_allreduce``           True: nothing is launched from the hooks, every bucket goes out at the end of backward
    ``gradient_average``          divide by the world size (default) or leave the sum
    ``gradient_predivide_factor`` apex divides by f before and multiplies by f/world after the all-reduce to keep an fp16 sum in
                                  range; the fused kernel pre-scales in the pack pass and accumulates in fp32 (in the switch),
                                  so only the net factor matters: 1/world with averaging, 1/f without
    ``allreduce_always_fp32``     fp32 wire format
    ``retain_allreduce_buffers``  ``self.allreduce_buffers`` = the per-bucket flat slices of the symmetric gradient arena
    ``num_allreduce_streams`` > 1, ``allreduce_communicators``, ``allreduce_trigger_params``, ``shared_param`` are rejected:
    there is one communication stream and one (symmetric-memory) communicator by design.

    Extensions (apex has neither): ``no_sync()``, torch DDP's context for backwards that only accumulate, and
    ``fp32_grad_accumulation``, which keeps that running sum in fp32 outside ``p.grad`` (see ``GradientEngine``).
    """

    def __init__(self, module: nn.Module, message_size: int = 10000000, delay_allreduce: bool = False, shared_param=None,
                 allreduce_trigger_params=None, retain_allreduce_buffers: bool = False, allreduce_always_fp32: bool = False,
                 num_allreduce_streams: int = 1, allreduce_communicators=None, gradient_average: bool = True,
                 gradient_predivide_factor: float = 1.0, comm="auto", wire_dtype=None, process_group=None,
                 fp32_grad_accumulation: bool = False):
        super().__init__()
        if shared_param is not None:
            raise ValueError("shared_param is no longer supported as an option (apex removed it as well); use delay_allreduce=True")
        if allreduce_trigger_params is not None:
            raise NotImplementedError("allreduce_trigger_params: buckets are fixed by message_size here, custom triggers are not supported")
        if num_allreduce_streams != 1:
            raise NotImplementedError("num_allreduce_streams=%r: the fused data plane uses exactly one communication stream" %
                                      (num_allreduce_streams,))
        if allreduce_communicators is not None:
            raise NotImplementedError("allreduce_communicators: the symmetric-memory communicator is created internally")
        self.module = module
        params = [p for p in module.parameters() if p.requires_grad]
        device = params[0].device
        if isinstance(comm, str):
            comm = make_communicator(comm, group=process_group, device=device)
        self.comm = comm
        register_for_sync_batchnorm(module, comm)
        scaler = _amp.current_scaler()
        if wire_dtype is None:
            if allreduce_always_fp32 or device.type != "cuda":
                wire_dtype = "fp32"
            elif scaler is not None:
                wire_dtype = _WIRE[_amp._amp_state.half_dtype]
            else:
                wire_dtype = "bf16"
        check_inf = scaler is not None and scaler.dynamic and getattr(comm, "backend", "") == "fused"
        if check_inf:
            scaler.rebind_found_inf(comm.found_inf)
        sync_module_states(module, comm, root=0)
        esz = 2 if wire_dtype != "fp32" else 4
        world = comm.world
        scale = (1.0 / world) if gradient_average else (1.0 / float(gradient_predivide_factor))
        self.engine = GradientEngine(params, comm, wire_dtype=wire_dtype, bucket_cap_mb=message_size * esz / float(1 << 20),
                                     first_bucket_mb=message_size * esz / float(1 << 20), check_inf=check_inf,
                                     average=gradient_average, delay_allreduce=delay_allreduce, scale=scale, tail_bucket_mb=None,
                                     fp32_grad_accumulation=fp32_grad_accumulation)
        self.delay_allreduce = delay_allreduce
        self.gradient_average = gradient_average
        self.gradient_predivide_factor = gradient_predivide_factor
        self.retain_allreduce_buffers = retain_allreduce_buffers
        self._buffers_f = _float_buffers(module)

    @property
    def allreduce_buffers(self):
        """Flat per-bucket views of the reduced gradients (apex ``retain_allreduce_buffers``); fused data plane only."""
        eng = self.engine
        if not self.retain_allreduce_buffers or not eng.fused:
            return []
        flat = eng.grad_arena()
        return [flat[b.elem_off:b.elem_off + b.region_elems] for b in eng.buckets]

    def forward(self, *inputs, **kwargs):
        return self.module(*inputs, **kwargs)

    @contextmanager
    def no_sync(self):
        """Backwards inside this context reduce nothing across ranks (torch DDP's ``no_sync``; an extension here)."""
        old = self.engine.enabled
        self.engine.enabled = False
        try:
            yield
        finally:
            self.engine.enabled = old


class Reducer:
    """apex.parallel.Reducer: manual ``reduce()`` of a module's gradients (average across ranks)."""

    def __init__(self, module_or_grads_list, comm="auto"):
        if isinstance(module_or_grads_list, nn.Module):
            self.module = module_or_grads_list
            params = list(self.module.parameters())
        else:
            self.module = None
            params = list(module_or_grads_list)
        self.params = params
        self.comm = make_communicator(comm, device=params[0].device) if isinstance(comm, str) else comm
        if self.module is not None:
            sync_module_states(self.module, self.comm, root=0)

    def reduce(self):
        grads = [p.grad for p in self.params if p.grad is not None]
        self.comm.all_reduce_(grads, average=True)


def flatten(tensors):
    """apex_C.flatten: one contiguous 1-D tensor holding the given dense tensors back to back."""
    return torch.cat([t.contiguous().view(-1) for t in tensors]) if len(tensors) else torch.empty(0)


def unflatten(flat, tensors):
    """apex_C.unflatten: views of ``flat`` shaped like ``tensors``."""
    out, off = [], 0
    for t in tensors:
        n = t.numel()
        out.append(flat.narrow(0, off, n).view_as(t))
        off += n
    return out


class SyncBatchNorm(SyncBNAct):
    """apex.parallel.SyncBatchNorm: apex's signature over the synchronised fused BatchNorm.  ``fuse_relu`` applies the
    ReLU inside the layer (``forward(x, z)`` adds ``z`` first, as apex's); ``channel_last`` is accepted for parity: the fused
    kernels take channels_last activations whatever it says, other layouts run torch's synchronised BatchNorm."""

    def __init__(self, num_features, eps=1e-5, momentum=0.1, affine=True, track_running_stats=True, process_group=None,
                 channel_last=False, fuse_relu=False):
        super().__init__(num_features, eps=eps, momentum=momentum, affine=affine, track_running_stats=track_running_stats,
                         process_group=process_group, relu=bool(fuse_relu))
        self.channel_last = channel_last

    def forward(self, input, z=None):  # type: ignore[override]
        return super().forward(input, z)


def convert_syncbn_model(module: nn.Module, process_group=None, channel_last: bool = False) -> nn.Module:
    """apex.parallel.convert_syncbn_model: every BatchNorm layer of ``module`` becomes a synchronised one (``SyncBatchNorm``,
    sharing its Parameters and buffers).  ``channel_last`` is accepted for signature parity: the fused kernels take
    channels_last activations whatever it says, other layouts run torch's synchronised BatchNorm."""
    return convert_sync_batchnorm(module, process_group)
