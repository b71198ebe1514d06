"""ResNet stem convolution (7x7 / stride 2 / pad 3 / C_in = 3) as im2col + the wgmma GEMM, fused with the stem tail.

cuDNN runs this layer on legacy kernels (C_in = 3 fits no tensor-core tile).  Here
(``csrc/stem_conv.cu``, ``csrc/gemm_bnstats.cu``):

    A  = im2col(x)                    [M, 192] bf16 / fp16, one 384-byte row per output pixel, k = r*24 + s*3 + c
    y  = A @ Wp^T  (+ BN statistics)  persistent wgmma GEMM; the sums BatchNorm needs come out of its epilogue
    -> BN + ReLU + MaxPool            ``stem_forward_pre`` (the statistics pass of the fused stem tail is skipped)
    dW = unpack(dY^T @ A)             library GEMM over the saved A

On by default for training-mode forwards (``PTD_STEM_GEMM=0`` / ``models.resnet.STEM_GEMM = False`` restores cuDNN).  It
runs when the image and the weight are both bf16 or both fp16 (a model cast to bf16 / fp16, e.g. ``amp`` O2 / O3), and
under ``torch.autocast("cuda")`` with a bf16 or fp16 autocast dtype (``amp`` O1, fp32 weights and images): there the
image and the weight are cast to the autocast dtype (the weight through autograd, so the fp32 parameter receives an fp32
gradient), as autocast's own ``F.conv2d`` would.  Eval mode keeps cuDNN.  The PyTorch functions below define the layout
and are what the CPU tests check against ``F.conv2d``.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F
from torch.autograd.function import once_differentiable

from .bn_act import workspace
from .sync_bn import kernel_arg
from .conv_bn import GEMM_DTYPES, autocast_gemm_dtype, gemm_weight
from .stem import _StemFn, bn_relu_maxpool, can_fuse_stem

K_PAD = 192        # GEMM K: 7 filter rows x 24 (21 real elements each) = 168, padded to 3 x 64
ROW_K = 24


def pack_stem_weight(weight: torch.Tensor) -> torch.Tensor:
    """[C_out, 3, 7, 7] -> [C_out, 192] in the k order of the im2col rows (zeros in the padding positions)."""
    co = weight.size(0)
    w = weight.permute(0, 2, 3, 1).reshape(co, 7, 21)              # (co, r, s*3 + c)
    w = F.pad(w, (0, ROW_K - 21)).reshape(co, 7 * ROW_K)
    return F.pad(w, (0, K_PAD - 7 * ROW_K)).contiguous()


def unpack_stem_weight(packed: torch.Tensor, like: torch.Tensor) -> torch.Tensor:
    """Inverse of :func:`pack_stem_weight` (drops the padding columns); result has ``like``'s shape / dtype / layout."""
    co = packed.size(0)
    w = packed[:, : 7 * ROW_K].reshape(co, 7, ROW_K)[:, :, :21].reshape(co, 7, 7, 3).permute(0, 3, 1, 2)
    out = torch.empty_like(like)
    out.copy_(w)
    return out


def im2col_reference(x: torch.Tensor) -> torch.Tensor:
    """What ``stem_im2col`` computes, in PyTorch: [N, 3, H, W] -> [N, 192, OH, OW] (channels_last), any device."""
    n, c, h, w = x.shape
    assert c == 3
    oh, ow = (h + 6 - 7) // 2 + 1, (w + 6 - 7) // 2 + 1
    cols = F.unfold(x.float(), kernel_size=7, padding=3, stride=2)                 # [N, 3*7*7, OH*OW], ordered (c, r, s)
    cols = cols.reshape(n, 3, 7, 7, oh * ow).permute(0, 4, 2, 3, 1).reshape(n, oh * ow, 7, 21)   # (r, s*3 + c)
    a = F.pad(cols, (0, ROW_K - 21)).reshape(n, oh * ow, 7 * ROW_K)
    a = F.pad(a, (0, K_PAD - 7 * ROW_K)).to(x.dtype)
    return a.reshape(n, oh, ow, K_PAD).permute(0, 3, 1, 2)


def can_use_stem_gemm(x: torch.Tensor, conv) -> bool:
    w = conv.weight
    ac = autocast_gemm_dtype()
    xdt, wdt = (ac, ac) if ac is not None and x.is_floating_point() and w.is_floating_point() else (x.dtype, w.dtype)
    return (x.is_cuda and xdt in GEMM_DTYPES and wdt == xdt and x.dim() == 4 and x.size(1) == 3
            and not x.requires_grad and conv.kernel_size == (7, 7) and conv.stride == (2, 2) and conv.padding == (3, 3)
            and conv.dilation == (1, 1) and conv.groups == 1 and conv.bias is None and w.size(0) % 64 == 0
            and x.is_contiguous(memory_format=torch.channels_last) and x.size(2) >= 7 and x.size(3) >= 7)


class _StemConvFn(torch.autograd.Function):
    """y = conv7x7s2(x, weight) through im2col + GEMM; ``stats`` (zeroed fp32 [2 * C_out]) receives sum / sum of squares."""

    @staticmethod
    def forward(ctx, x, weight, stats, emulate=False, sync=None):
        packed = pack_stem_weight(weight)
        if emulate:
            a = im2col_reference(x).contiguous(memory_format=torch.channels_last)
            rows = a.permute(0, 2, 3, 1).reshape(-1, K_PAD)
            y2 = (rows.float() @ packed.float().t()).to(x.dtype)
            if stats is not None:
                stats[: y2.size(1)] += y2.float().sum(0)
                stats[y2.size(1): 2 * y2.size(1)] += (y2.float() ** 2).sum(0)
            y = y2.reshape(a.size(0), a.size(2), a.size(3), -1).permute(0, 3, 1, 2)
        else:
            from .. import _ext
            C = _ext.lib()
            _ext.note_launch(3)                 # im2col + GEMM + statistics combine
            a = C.stem_im2col(x)
            y = C.conv1x1_bnstats(a, packed.view(packed.size(0), K_PAD, 1, 1), stats, kernel_arg(sync, C))
        ctx.save_for_backward(a, weight)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        a, weight = ctx.saved_tensors
        co = weight.size(0)
        dy2 = dy.permute(0, 2, 3, 1).reshape(-1, co)                   # [M, C_out] view of the channels_last gradient
        rows = a.permute(0, 2, 3, 1).reshape(-1, K_PAD)
        if dy2.dtype != rows.dtype:
            dy2 = dy2.to(rows.dtype)
        # [C_out, 192], a reduction over millions of output pixels: fp32 result, so that the library's split-K partial sums are
        # not rounded to 16 bits on the way (cuDNN's wgrad accumulates in fp32 too)
        if rows.is_cuda and rows.dtype != torch.float32:
            dwp = torch.mm(dy2.t(), rows, out_dtype=torch.float32)
        else:
            dwp = dy2.float().t() @ rows.float()
        return None, unpack_stem_weight(dwp, weight), None, None, None


def stem_conv_bn_relu_maxpool(x, conv, bn, emulate: bool = False):
    """maxpool(relu(bn(conv7x7(x)))) for the ResNet stem modules ``conv`` (nn.Conv2d) and ``bn`` (BNAct), training mode.
    A synchronised ``bn`` (``SyncBNAct``) exchanges the GEMM's statistics across the ranks."""
    nc = conv.weight.size(0)
    momentum = bn.momentum
    nbt = bn.num_batches_tracked if (bn.training and bn.track_running_stats) else None
    sync = bn.sync_context()
    if emulate:                                                        # CPU / test path: same op graph, PyTorch math
        y = _StemConvFn.apply(x, conv.weight, None, True)
        return bn_relu_maxpool(y, bn.weight, bn.bias, bn.running_mean, bn.running_var, training=True, momentum=momentum, eps=bn.eps,
                               fused=False, num_batches_tracked=nbt, sync=sync)
    if momentum is None:                                               # cumulative average: cuDNN + the unfused BatchNorm
        return bn_relu_maxpool(conv(x), bn.weight, bn.bias, bn.running_mean, bn.running_var, training=True, momentum=None,
                               eps=bn.eps, fused=False, num_batches_tracked=nbt, sync=sync)
    ac = autocast_gemm_dtype()
    if ac is not None and x.dtype != ac:
        x = x.to(ac)                                                   # keeps channels_last
    lw = workspace(x.device).layer(nc, sync)
    y = _StemConvFn.apply(x, gemm_weight(conv.weight, ac), lw.fwd, False, sync)   # always 5 inputs: backward returns 5 gradients
    if not can_fuse_stem(y, bn.weight, bn.running_mean):
        raise RuntimeError("stem GEMM output does not fit the fused stem tail")
    need_grad = torch.is_grad_enabled() and (y.requires_grad or bn.weight.requires_grad)
    return _StemFn.apply(y, bn.weight, bn.bias, bn.running_mean, bn.running_var, nbt, True, float(momentum), float(bn.eps), need_grad,
                         sync, lw)
