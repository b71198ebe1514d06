"""``bn_relu_maxpool``: the ResNet stem tail (BatchNorm -> ReLU -> MaxPool 3x3/2/1) as one autograd op.

CUDA + channels_last -> ``csrc/bn_act.cu`` (stem_* kernels): the 112x112 normalised activation and its gradient never
reach HBM; otherwise the plain PyTorch composition (also the oracle of ``tests/test_gpu_kernels.py``).
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from .bn_act import bn_act_reference, sync_batch_norm_unfused, workspace
from .sync_bn import work_len


def bn_relu_maxpool_reference(x, weight, bias, running_mean, running_var, training=True, momentum=0.1, eps=1e-5):
    y = bn_act_reference(x, weight, bias, running_mean, running_var, None, True, training, momentum, eps)
    return F.max_pool2d(y, kernel_size=3, stride=2, padding=1)


class _StemFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, running_mean, running_var, nbt, training, momentum, eps, need_grad, sync=None):
        from .. import _ext
        C = _ext.lib()
        nc = x.size(1)
        ws = workspace(x.device)
        wl = work_len(nc, sync)
        if training:
            work, gen = ws.take(2 * wl)
        else:
            work, gen = torch.empty(0, dtype=torch.float32, device=x.device), -1
        _ext.note_launch(3 if training else 1)
        y, saved, code = C.stem_forward(x, weight, bias, running_mean, running_var, nbt, training, momentum, eps, need_grad,
                                        work[:wl] if training else work, None if sync is None else sync.native)
        ctx.work = work[wl:] if training else None
        ctx.gen, ctx.ws, ctx.sync = gen, ws, sync
        if need_grad:
            if not training:
                raise RuntimeError("fused stem: backward through eval-mode batch norm is not supported")
            ctx.save_for_backward(x, code, weight, saved)
        return y

    @staticmethod
    def backward(ctx, dy):
        from .. import _ext
        C = _ext.lib()
        x, code, weight, saved = ctx.saved_tensors
        work = ctx.work
        sync = ctx.sync
        if work is None or (ctx.gen != -1 and ctx.gen != ctx.ws.generation):
            work = torch.zeros(work_len(x.size(1), sync), dtype=torch.float32, device=x.device)
        _ext.note_launch(3)
        dx, dw, db = C.stem_backward(dy, x, code, weight, saved, work, None if sync is None else sync.native)
        return dx, dw, db, None, None, None, None, None, None, None, None


def can_fuse_stem(x, weight, running_mean) -> bool:
    c = x.size(1) if x.dim() == 4 else 0
    return (x.is_cuda and x.dim() == 4 and c % 8 == 0 and c >= 8 and 256 % (c // 8) == 0 and weight is not None
            and running_mean is not None and x.dtype in (torch.float32, torch.bfloat16, torch.float16)
            and x.is_contiguous(memory_format=torch.channels_last) and x.size(2) >= 2 and x.size(3) >= 2)


def bn_relu_maxpool(x, weight, bias, running_mean, running_var, training=True, momentum=0.1, eps=1e-5, fused=None,
                    num_batches_tracked=None, sync=None):
    """maxpool(relu(bn(x))); ``sync`` (a ``SyncContext``, see ``ops/sync_bn.py``) synchronises the training statistics."""
    if sync is not None and (not training or sync.world == 1):
        sync = None
    ok = can_fuse_stem(x, weight, running_mean)
    need_grad = torch.is_grad_enabled() and (x.requires_grad or (weight is not None and weight.requires_grad))
    if need_grad and not training:
        ok = False
    use = ok if fused is None else (fused and ok)
    if sync is not None and not (use and sync.native is not None):
        y = sync_batch_norm_unfused(x, weight, bias, running_mean, running_var, momentum, eps, num_batches_tracked, sync)
        return F.max_pool2d(F.relu(y), kernel_size=3, stride=2, padding=1)
    if not use:
        if training and num_batches_tracked is not None:
            num_batches_tracked.add_(1)
        if weight is not None and x.is_cuda and weight.dtype != torch.float32 and x.dtype != weight.dtype:
            weight, bias = weight.to(x.dtype), bias.to(x.dtype)
        if not x.is_cuda and x.dtype != torch.float32:
            return bn_relu_maxpool_reference(x.float(), weight.float(), bias.float(), running_mean, running_var, training, momentum,
                                             eps).to(x.dtype)
        return bn_relu_maxpool_reference(x, weight, bias, running_mean, running_var, training, momentum, eps)
    return _StemFn.apply(x, weight, bias, running_mean, running_var, num_batches_tracked, training, float(momentum), float(eps), need_grad,
                         sync)
