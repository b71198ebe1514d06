"""``conv1x1_bn_act``: 1x1 convolution -> BatchNorm (+ residual) (+ ReLU) with the BN statistics produced by the GEMM.

The convolution runs as a hand-written wgmma GEMM (``csrc/gemm_bnstats.cu``: TMA -> smem -> ``wgmma.mma_async`` -> registers)
whose epilogue reduces the per-channel sum / sum of squares of the stored bf16 output, so BatchNorm only needs its
apply pass.  Backward: cuDNN dgrad / wgrad for the convolution, the fused BN backward kernels for the rest.
Falls back to ``F.conv2d`` + :func:`bn_act` whenever the fast path does not apply (CPU, fp32/fp16, stride != 1, odd shapes).
"""
from __future__ import annotations

import torch

from .bn_act import _BnActFn, _can_fuse, workspace


class _Conv1x1Stats(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, stats):
        from .. import _ext
        _ext.note_launch(2)                     # GEMM + statistics combine
        y = _ext.lib().conv1x1_bnstats(x, weight, stats)
        ctx.save_for_backward(x, weight)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, weight = ctx.saved_tensors
        dy = dy.contiguous(memory_format=torch.channels_last)
        dx, dw, _ = torch.ops.aten.convolution_backward(dy, x, weight, None, (1, 1), (0, 0), (1, 1), False, (0, 0), 1,
                                                        (ctx.needs_input_grad[0], ctx.needs_input_grad[1], False))
        return dx, dw, None


def can_fuse_conv1x1(x, conv) -> bool:
    w = conv.weight
    return (x.is_cuda and x.dtype == torch.bfloat16 and w.dtype == torch.bfloat16 and x.dim() == 4
            and conv.kernel_size == (1, 1) and conv.stride == (1, 1) and conv.padding == (0, 0) and conv.groups == 1 and conv.bias is None
            and x.is_contiguous(memory_format=torch.channels_last) and x.size(1) % 64 == 0 and w.size(0) % 64 == 0
            and x.size(0) * x.size(2) * x.size(3) >= 128)


def conv1x1_bn_act(x, conv, bn, residual=None, enabled=True, split=False):
    """relu?(bn(conv1x1(x)) + residual) for a ``nn.Conv2d`` and a :class:`BNAct` module (``split``: see ``bn_act``)."""
    training = bn.training or not bn.track_running_stats
    if not (enabled and training and can_fuse_conv1x1(x, conv) and bn.fused is not False):
        return bn(conv(x), residual, split) if split else bn(conv(x), residual)
    nc = conv.weight.size(0)
    ws = workspace(x.device)
    work, gen = ws.take(4 * nc)
    y = _Conv1x1Stats.apply(x, conv.weight, work[: 2 * nc])
    if not _can_fuse(y, bn.weight, residual, bn.running_mean):
        return bn(y, residual, split) if split else bn(y, residual)   # (cannot happen for the shapes accepted above)
    need_grad = torch.is_grad_enabled() and (y.requires_grad or bn.weight.requires_grad)
    nbt = bn.num_batches_tracked if (bn.training and bn.track_running_stats) else None
    out = _BnActFn.apply(y, residual, bn.weight, bn.bias, bn.running_mean, bn.running_var, nbt, True,
                         0.1 if bn.momentum is None else float(bn.momentum), float(bn.eps), bn.relu, need_grad, (work, gen),
                         bool(split and need_grad))
    if split and not isinstance(out, tuple):
        return out, out
    return out
