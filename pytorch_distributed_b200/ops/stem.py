"""``bn_relu_maxpool``: the ResNet stem tail (BatchNorm -> ReLU -> MaxPool 3x3/2/1) as one autograd op.

CUDA + channels_last -> ``csrc/bn_act.cu`` (stem_* kernels): the 112x112 normalised activation and its gradient never
reach HBM; otherwise the plain PyTorch composition (also the oracle of ``tests/test_gpu_kernels.py``).
"""
from __future__ import annotations

import torch
import torch.nn.functional as F
from torch.autograd.function import once_differentiable

from .bn_act import batch_norm_unfused, bn_act_reference, workspace
from .sync_bn import effective, kernel_arg


def bn_relu_maxpool_reference(x, weight, bias, running_mean, running_var, training=True, momentum=0.1, eps=1e-5):
    y = bn_act_reference(x, weight, bias, running_mean, running_var, None, True, training, momentum, eps)
    return F.max_pool2d(y, kernel_size=3, stride=2, padding=1)


class _StemFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, running_mean, running_var, nbt, training, momentum, eps, need_grad, sync=None, pre=None):
        from .. import _ext
        C = _ext.lib()
        stats_ready = pre is not None          # the layer's slices: sums already reduced by the producing GEMM (stem_conv.py)
        lw = pre if stats_ready else (workspace(x.device).layer(x.size(1), sync) if training else None)
        _ext.note_launch(1 if (stats_ready or not training) else 3)
        fwd = C.stem_forward_pre if stats_ready else C.stem_forward
        y, saved, code = fwd(x, weight, bias, running_mean, running_var, nbt, training, momentum, eps, need_grad,
                             lw.fwd if training else torch.empty(0, dtype=torch.float32, device=x.device), kernel_arg(sync, C))
        ctx.work, ctx.sync = lw, sync
        if need_grad:
            if not training:
                raise RuntimeError("fused stem: backward through eval-mode batch norm is not supported")
            ctx.save_for_backward(x, code, weight, saved)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        from .. import _ext
        C = _ext.lib()
        x, code, weight, saved = ctx.saved_tensors
        _ext.note_launch(3)
        dx, dw, db = C.stem_backward(dy, x, code, weight, saved, ctx.work.bwd(), kernel_arg(ctx.sync, C))
        return (dx, dw, db) + (None,) * 9


def can_fuse_stem(x, weight, running_mean) -> bool:
    c = x.size(1) if x.dim() == 4 else 0
    return (x.is_cuda and x.dim() == 4 and c % 8 == 0 and c >= 8 and 256 % (c // 8) == 0 and weight is not None
            and running_mean is not None and x.dtype in (torch.float32, torch.bfloat16, torch.float16)
            and x.is_contiguous(memory_format=torch.channels_last) and x.size(2) >= 2 and x.size(3) >= 2)


def bn_relu_maxpool(x, weight, bias, running_mean, running_var, training=True, momentum=0.1, eps=1e-5, fused=None,
                    num_batches_tracked=None, sync=None):
    """maxpool(relu(bn(x))); ``sync`` (a ``SyncContext``, see ``ops/sync_bn.py``) synchronises the training statistics."""
    sync = effective(sync, training)
    ok = can_fuse_stem(x, weight, running_mean)
    need_grad = torch.is_grad_enabled() and (x.requires_grad or (weight is not None and weight.requires_grad))
    if need_grad and not training:
        ok = False
    use = ok if fused is None else (fused and ok)
    if momentum is None and training:   # cumulative average (see batch_norm_unfused)
        use = False
    if not use or (sync is not None and sync.native is None):
        return batch_norm_unfused(x, weight, bias, running_mean, running_var, training, momentum, eps, num_batches_tracked, sync,
                                  lambda y: F.max_pool2d(F.relu(y), kernel_size=3, stride=2, padding=1))
    if momentum is None:                # eval mode: the factor is not used
        momentum = 0.0
    return _StemFn.apply(x, weight, bias, running_mean, running_var, num_batches_tracked, training, float(momentum), float(eps), need_grad,
                         sync, None)
