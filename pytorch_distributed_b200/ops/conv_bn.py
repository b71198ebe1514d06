"""``conv1x1_bn_act``: 1x1 convolution -> BatchNorm (+ residual) (+ ReLU) with the BN statistics produced by the GEMM.

The convolution runs as a hand-written wgmma GEMM (``csrc/gemm_bnstats.cu``: TMA -> smem -> ``wgmma.mma_async`` -> registers)
whose epilogue reduces the per-channel sum / sum of squares of the stored 16-bit output, so BatchNorm only needs its
apply pass.  Backward: cuDNN dgrad / wgrad for the convolution, the fused BN backward kernels for the rest.

Training-mode steps take the GEMM when the activations and the weights are both bf16 or both fp16 (a model cast to
bf16 / fp16, e.g. ``amp`` O2 / O3), and under ``torch.autocast("cuda")`` with a bf16 or fp16 autocast dtype (``amp`` O1,
fp32 weights): there the weight is cast to the autocast dtype through autograd, as autocast's own ``F.conv2d`` would,
so the fp32 parameter still receives an fp32 gradient.  Everything else - eval mode, CPU, fp32 activations, stride != 1,
odd shapes, ``PTD_FUSED_CONV1X1=0`` - runs ``F.conv2d`` + :func:`bn_act`.

The backward of a pair on one rank (:class:`_Conv1x1BnFn`) runs the BN reduction pass and then ``conv1x1_bn_backward``'s
wgmma data-gradient GEMM, which forms BN's dx from g and y in shared memory as it loads its A operand: dx is written once,
for cuDNN's weight gradient, instead of being written by the BN apply pass and read back by cuDNN's dgrad.  dx has the
bits of the apply pass.  It is taken where it is faster (``tools/dgrad_probe.py``): up to 256 input channels, i.e. one or
two 128-wide n-tiles.  With more, every n-tile re-forms the same dx tiles and the few m-tiles of those small late-stage
activations leave too few CTAs per n-tile, so cuDNN's dgrad wins.  Synchronised BatchNorm, a block output without
``split`` (the apply would also write the residual gradient) and ``PTD_FUSED_DGRAD=0`` keep the two-op backward.
"""
from __future__ import annotations

import os

import torch
from torch.autograd.function import once_differentiable

from .bn_act import _BnActFn, _can_fuse, workspace
from .sync_bn import kernel_arg

FUSED_DGRAD = os.environ.get("PTD_FUSED_DGRAD", "1") == "1"
DGRAD_MAX_CIN = 256                # widest conv input the fused backward is faster for (module docstring)


class _Conv1x1Stats(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, stats, sync=None):
        from .. import _ext
        _ext.note_launch(2)                     # GEMM + statistics combine (or cross-rank exchange)
        C = _ext.lib()
        y = C.conv1x1_bnstats(x, weight, stats, kernel_arg(sync, C))
        ctx.save_for_backward(x, weight)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        x, weight = ctx.saved_tensors
        dy = dy.contiguous(memory_format=torch.channels_last)
        dx, dw, _ = torch.ops.aten.convolution_backward(dy, x, weight, None, (1, 1), (0, 0), (1, 1), False, (0, 0), 1,
                                                        (ctx.needs_input_grad[0], ctx.needs_input_grad[1], False))
        return dx, dw, None, None


class _Conv1x1BnFn(torch.autograd.Function):
    """relu?(bn(conv1x1(x)) (+ residual)) of one rank: forward as ``_Conv1x1Stats`` + ``_BnActFn``, backward through
    ``conv1x1_bn_backward`` (reduction pass + fused data-gradient GEMM) and cuDNN's weight gradient fed with its dx.
    ``split``: two aliases of the output, whose gradients arrive separately (the residual gradient is their masked sum)."""

    @staticmethod
    def forward(ctx, x, weight, residual, bn_weight, bias, running_mean, running_var, nbt, momentum, eps, relu, lw, split):
        from .. import _ext
        C = _ext.lib()
        ctx.set_materialize_grads(False)
        _ext.note_launch(3)                     # GEMM + statistics combine + apply
        y = C.conv1x1_bnstats(x, weight, lw.fwd, None)
        out, saved, mask = C.bn_act_forward(y, residual, bn_weight, bias, running_mean, running_var, nbt, True, momentum, eps, relu,
                                            True, lw.fwd, True, None)
        ctx.save_for_backward(x, weight, y, mask if relu else None, bn_weight, saved)
        ctx.relu, ctx.has_res, ctx.work = relu, residual is not None, lw
        if split:
            return out, out.view_as(out)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, dy, dy2=None):
        from .. import _ext
        none = (None,) * 9
        if dy is None:
            dy, dy2 = dy2, None
        if dy is None:
            return (None,) * 4 + none
        x, weight, y, mask, bn_weight, saved = ctx.saved_tensors
        C = _ext.lib()
        work = ctx.work.bwd()
        if ctx.has_res and dy2 is None:         # one alias of a split output unused: the apply writes the residual gradient
            _ext.note_launch(3)
            dy_bn, dres, dgamma, dbeta = C.bn_act_backward(dy, y, mask, bn_weight, saved, ctx.relu, True, work)
            dx, dw, _ = torch.ops.aten.convolution_backward(dy_bn, x, weight, None, (1, 1), (0, 0), (1, 1), False, (0, 0), 1,
                                                            (ctx.needs_input_grad[0], ctx.needs_input_grad[1], False))
            return (dx, dw, dres, dgamma, dbeta) + (None,) * 8
        _ext.note_launch(3)                     # reduce + combine + fused dgrad GEMM
        dx, dy_bn, g, dgamma, dbeta = C.conv1x1_bn_backward(dy, dy2, y, mask, bn_weight, saved, weight, ctx.relu, work)
        dw = None
        if ctx.needs_input_grad[1]:
            dw = torch.ops.aten.convolution_backward(dy_bn, x, weight, None, (1, 1), (0, 0), (1, 1), False, (0, 0), 1,
                                                     (False, True, False))[1]
        return (dx, dw, (g if ctx.has_res else None), dgamma, dbeta) + (None,) * 8


GEMM_DTYPES = (torch.bfloat16, torch.float16)


def autocast_gemm_dtype():
    """The dtype CUDA autocast runs convolutions in when it is enabled and one the GEMM takes (bf16 / fp16), else None."""
    if torch.is_autocast_enabled("cuda"):
        dt = torch.get_autocast_dtype("cuda")
        if dt in GEMM_DTYPES:
            return dt
    return None


def gemm_weight(w, autocast_dtype):
    """The weight the GEMM multiplies by: ``w`` itself, or its autocast copy (a differentiable cast)."""
    return w if autocast_dtype is None or w.dtype == autocast_dtype else w.to(autocast_dtype)


def can_fuse_conv1x1(x, conv) -> bool:
    w = conv.weight
    wdt = autocast_gemm_dtype() or w.dtype
    return (x.is_cuda and x.dtype in GEMM_DTYPES and wdt == x.dtype and w.is_floating_point() and x.dim() == 4
            and conv.kernel_size == (1, 1) and conv.stride == (1, 1) and conv.padding == (0, 0) and conv.groups == 1 and conv.bias is None
            and x.is_contiguous(memory_format=torch.channels_last) and x.size(1) % 64 == 0 and w.size(0) % 64 == 0
            and x.size(0) * x.size(2) * x.size(3) >= 128)


def conv1x1_bn_act(x, conv, bn, residual=None, enabled=True, split=False):
    """relu?(bn(conv1x1(x)) + residual) for a ``nn.Conv2d`` and a :class:`BNAct` module (``split``: see ``bn_act``).
    A synchronised ``bn`` (``SyncBNAct``) exchanges the GEMM's statistics across the ranks before the apply pass."""
    training = bn.training or not bn.track_running_stats
    sync = bn.sync_context()
    if not (enabled and training and can_fuse_conv1x1(x, conv) and bn.fused is not False and (sync is None or sync.native is not None)
            and bn.momentum is not None):       # momentum=None (cumulative average) runs the unfused BatchNorm
        return bn(conv(x), residual, split) if split else bn(conv(x), residual)
    lw = workspace(x.device).layer(conv.weight.size(0), sync)
    need_grad = torch.is_grad_enabled() and (x.requires_grad or conv.weight.requires_grad or bn.weight.requires_grad)
    if (FUSED_DGRAD and need_grad and sync is None and (residual is None or split) and x.size(1) <= DGRAD_MAX_CIN
            and bn.weight is not None and bn.running_mean is not None
            and (residual is None or (residual.dtype == x.dtype and residual.is_contiguous(memory_format=torch.channels_last)
                                      and residual.shape == (x.size(0), conv.weight.size(0), x.size(2), x.size(3))))):
        nbt = bn.num_batches_tracked if (bn.training and bn.track_running_stats) else None
        out = _Conv1x1BnFn.apply(x, gemm_weight(conv.weight, autocast_gemm_dtype()), residual, bn.weight, bn.bias, bn.running_mean,
                                 bn.running_var, nbt, float(bn.momentum), float(bn.eps), bn.relu, lw, bool(split))
        return out if (not split or isinstance(out, tuple)) else (out, out)
    y = _Conv1x1Stats.apply(x, gemm_weight(conv.weight, autocast_gemm_dtype()), lw.fwd, sync)
    if not _can_fuse(y, bn.weight, residual, bn.running_mean):
        return bn(y, residual, split) if split else bn(y, residual)   # (cannot happen for the shapes accepted above)
    need_grad = torch.is_grad_enabled() and (y.requires_grad or bn.weight.requires_grad)
    nbt = bn.num_batches_tracked if (bn.training and bn.track_running_stats) else None
    out = _BnActFn.apply(y, residual, bn.weight, bn.bias, bn.running_mean, bn.running_var, nbt, True,
                         float(bn.momentum), float(bn.eps), bn.relu, need_grad, lw,
                         bool(split and need_grad), sync)
    if split and not isinstance(out, tuple):
        return out, out
    return out
