"""``bn_act``: BatchNorm2d (+ residual add) (+ ReLU) as one autograd op.

CUDA + channels_last + C % 8 == 0  -> hand-written NHWC kernels (``csrc/bn_act.cu``): statistics pass + one fused
apply pass forward, reduce pass + one fused apply pass backward.
Anything else (CPU, NCHW, odd channel counts) -> the plain PyTorch composition below, which is also the numerical
oracle in ``tests/test_bn_act.py``.

The per-call fp32 accumulators ([2C] sums for forward, [2C] for backward) come from a per-device workspace that is
zeroed ONCE per training step (one memset for all ~100 slices of a ResNet-50) instead of one ``zeros()`` per layer.

``sync=`` (an ``ops.sync_bn.SyncContext``) normalises with the statistics of the whole data-parallel batch
(``torch.nn.SyncBatchNorm`` semantics); each direction then takes ``sync_work_len(C)`` floats of the workspace.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn.functional as F
from torch.autograd.function import once_differentiable

from .sync_bn import effective, kernel_arg, work_len


def bn_act_reference(x, weight, bias, running_mean, running_var, residual=None, relu=True, training=True, momentum=0.1,
                     eps=1e-5):
    """Plain PyTorch semantics: relu(batch_norm(x) + residual)."""
    w = weight if weight is None or weight.dtype == x.dtype or x.dtype == torch.float32 else weight
    y = F.batch_norm(x, running_mean, running_var, w, bias, training, momentum, eps)
    if residual is not None:
        y = y + residual
    return F.relu(y) if relu else y


class _Workspace:
    """Bump allocator over one zeroed fp32 buffer per device; ``reset`` = a single memset per step."""

    def __init__(self, device, capacity: int = 1 << 20):
        self.buf = torch.zeros(capacity, dtype=torch.float32, device=device)
        self.used = 0
        self.generation = 0

    def reset(self):
        if self.used:
            self.buf[: self.used].zero_()
        self.used = 0
        self.generation += 1

    def take(self, n: int):
        n = (n + 31) // 32 * 32
        if self.used + n > self.buf.numel():
            return torch.zeros(n, dtype=torch.float32, device=self.buf.device), -1
        s = self.buf[self.used: self.used + n]
        self.used += n
        return s, self.generation

    def layer(self, c: int, sync) -> "_LayerWork":
        """The accumulator slices of one fused BatchNorm layer of ``c`` channels: ``work_len(c, sync)`` floats per direction."""
        wl = work_len(c, sync)
        work, gen = self.take(2 * wl)
        return _LayerWork(self, work, gen, wl)


class _LayerWork:
    """``fwd``: the slice the forward (or the GEMM producing its statistics) accumulates into; ``bwd()``: the backward's."""

    def __init__(self, ws, work, gen, wl):
        self.fwd = work[:wl]
        self._bwd = work[wl:]
        self._ws, self._gen, self._wl, self._dev = ws, gen, wl, work.device

    def bwd(self):
        """The backward's slice, handed out once.  The kernels add their sums into the slice they are given, so a second
        backward through the same graph (``retain_graph=True``, two ``autograd.grad`` calls, two losses over one trunk)
        and a backward after ``reset`` recycled the slice get fresh zeros instead."""
        work, self._bwd = self._bwd, None
        if work is None or (self._gen != -1 and self._gen != self._ws.generation):
            return torch.zeros(self._wl, dtype=torch.float32, device=self._dev)
        return work


_workspaces = {}


def workspace(device) -> _Workspace:
    ws = _workspaces.get(device)
    if ws is None:
        ws = _Workspace(device)
        _workspaces[device] = ws
    return ws


def begin_step(device) -> None:
    """Call once before a training forward pass: recycles (zeroes) the accumulator slices of the previous step."""
    if device.type == "cuda" or device in _workspaces:
        workspace(device).reset()


class _Emu:
    """Pure PyTorch (fp32 math) stand-in for the ``csrc/bn_act.cu`` entry points, same signatures and tensor contracts
    (channels_last activations seen as a row-major [M, C] matrix, 1 mask byte per 8 channels, ``saved`` = mean | invstd).
    It documents what the kernels compute and lets the CPU tests drive the autograd plumbing of :class:`_BnActFn`
    (``bn_act(..., fused="emulate")``).  Like the kernels, each reduction adds its [2C] sums into ``work[:2C]`` and the
    statistics and gradients are computed from what the slice then holds.  With ``sync`` (a ``SyncContext``) the sums
    and the row count are added over the ranks with the communicator's ``all_reduce_``."""

    is_emulation = True

    @staticmethod
    def _accumulate(work, sums):
        """``work[:2C] += sums``; returns a copy of what the slice holds afterwards (``work`` None: a fresh slice)."""
        if work is None:
            return sums.clone()
        w = work[:sums.numel()]
        w += sums
        return w.clone()

    @staticmethod
    def _rows(t):
        return t.permute(0, 2, 3, 1).reshape(-1, t.size(1))

    @staticmethod
    def _like(rows, ref):
        n, c, h, w = ref.shape
        return rows.reshape(n, h, w, c).permute(0, 3, 1, 2).to(ref.dtype).contiguous(memory_format=torch.channels_last)

    @staticmethod
    def _unpack(mask, m, c):
        bits = (mask.view(m, c // 8, 1).to(torch.int32) >> torch.arange(8, device=mask.device, dtype=torch.int32)) & 1
        return bits.reshape(m, c).bool()

    @staticmethod
    def _global_sums(sums, m, sync):
        """(global [2C] sums, global row count) of this rank's sums over the ranks of ``sync``."""
        v = torch.cat([sums.float(), sums.new_tensor([float(m)], dtype=torch.float32)])
        sync.all_reduce_sum_(v)
        c2 = sums.numel()
        return v[:c2], int(round(v[c2].item()))

    @staticmethod
    def bn_act_forward(x, residual, weight, bias, rm, rv, nbt, training, momentum, eps, relu, need_mask, work, stats_ready, sync=None):
        xr = _Emu._rows(x).float()
        m, c = xr.shape
        n = m                                 # rows the statistics cover
        saved = mask = None
        if training:                          # E[x^2] - E[x]^2 over the (global) sums, as the kernels compute it
            sums = work[:2 * c].clone() if stats_ready else _Emu._accumulate(work, torch.cat([xr.sum(0), (xr * xr).sum(0)]))
            if sync is not None:
                sums, n = _Emu._global_sums(sums, m, sync)
            mean = sums[:c] / n
            var = (sums[c:] / n - mean * mean).clamp_min(0)
            invstd = torch.rsqrt(var + eps)
            saved = torch.cat([mean, invstd])
            if rm is not None:
                rm.mul_(1 - momentum).add_(momentum * mean)
                rv.mul_(1 - momentum).add_(momentum * var * (n / (n - 1) if n > 1 else 1.0))
            if nbt is not None:
                nbt.add_(1)
        else:
            mean, invstd = rm, torch.rsqrt(rv + eps)
        v = (xr - mean) * (invstd * weight.float()) + bias.float()
        if residual is not None:
            v = v + _Emu._rows(residual).float()
        if relu:
            if need_mask:
                pos = (v > 0).view(m, c // 8, 8).to(torch.int32)
                mask = (pos << torch.arange(8, device=x.device, dtype=torch.int32)).sum(-1).to(torch.uint8).reshape(-1)
            v = v.clamp_min(0)
        return _Emu._like(v, x), saved, mask

    @staticmethod
    def _bwd_from_g(g, x, weight, saved, work, sync=None):
        xr = _Emu._rows(x).float()
        m, c = xr.shape
        mean, invstd = saved[:c], saved[c:]
        xhat = (xr - mean) * invstd
        sums = _Emu._accumulate(work, torch.cat([g.sum(0), (g * xhat).sum(0)]))
        sdz, sdzx = sums[:c], sums[c:]
        gdz, gdzx, n = sdz, sdzx, m
        if sync is not None:              # dx from the global sums; dgamma / dbeta stay this rank's
            tot, n = _Emu._global_sums(torch.cat([sdz, sdzx]), m, sync)
            gdz, gdzx = tot[:c], tot[c:]
        dx = (weight.float() * invstd) * (g - gdz / n - xhat * gdzx / n)
        return _Emu._like(dx, x), sdzx.to(weight.dtype), sdz.to(weight.dtype)

    @staticmethod
    def bn_act_backward(dy, x, mask, weight, saved, relu, has_res, work, sync=None):
        g = _Emu._rows(dy).float()
        if relu:
            g = g * _Emu._unpack(mask, *g.shape)
        dx, dw, db = _Emu._bwd_from_g(g, x, weight, saved, work, sync)
        dres = None
        if has_res:
            dres = dy if not relu else _Emu._like(g, x)
        return dx, dres, dw, db

    @staticmethod
    def bn_act_backward2(dy_a, dy_b, x, mask, weight, saved, relu, work, sync=None):
        g = (_Emu._rows(dy_a).float() + _Emu._rows(dy_b).float()).to(x.dtype).float()      # rounded like an eager add
        if relu:
            g = g * _Emu._unpack(mask, *g.shape)
        dx, dw, db = _Emu._bwd_from_g(g, x, weight, saved, work, sync)
        return dx, _Emu._like(g, x), dw, db


def _kernels(x):
    if x.is_cuda:
        from .. import _ext
        return _ext.lib()
    return _Emu


class _BnActFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, residual, weight, bias, running_mean, running_var, nbt, training, momentum, eps, relu, need_grad, pre=None,
                split=False, sync=None):
        from .. import _ext
        C = _kernels(x)
        ctx.set_materialize_grads(False)
        stats_ready = pre is not None          # the layer's slices: sums already reduced by the producing GEMM
        lw = pre if stats_ready else (workspace(x.device).layer(x.size(1), sync) if training else None)
        _ext.note_launch(1 if (stats_ready or not training) else 3)   # stats + combine (or exchange) + apply
        y, saved, mask = C.bn_act_forward(x, residual, weight, bias, running_mean, running_var, nbt, training, momentum, eps, relu,
                                          need_grad, lw.fwd if training else torch.empty(0, dtype=torch.float32, device=x.device),
                                          stats_ready, kernel_arg(sync, C))
        ctx.relu = relu
        ctx.has_res = residual is not None
        ctx.sync = sync
        ctx.work = lw
        if need_grad:
            if not training:
                raise RuntimeError("fused bn_act: backward through eval-mode batch norm is not supported")
            ctx.save_for_backward(x, mask if relu else None, weight, saved)
        if split:       # two aliases of one buffer: each consumer's gradient arrives separately in backward (no autograd add)
            return y, y.view_as(y)
        return y

    @staticmethod
    @once_differentiable            # the kernels are not differentiable: a second-order gradient raises instead of being cut
    def backward(ctx, dy, dy2=None):
        from .. import _ext
        none = (None,) * 11
        if dy is None:
            dy, dy2 = dy2, None
        if dy is None:                          # neither alias was used
            return (None, None, None, None) + none
        x, mask, weight, saved = ctx.saved_tensors
        C = _kernels(x)
        work = ctx.work.bwd()
        _ext.note_launch(3)                     # reduce + combine (or exchange) + apply
        karg = kernel_arg(ctx.sync, C)
        if dy2 is not None:                     # add + mask + reductions in one pass; g doubles as the residual gradient
            dx, dres, dw, db = C.bn_act_backward2(dy, dy2, x, mask, weight, saved, ctx.relu, work, karg)
        else:
            dx, dres, dw, db = C.bn_act_backward(dy, x, mask, weight, saved, ctx.relu, ctx.has_res, work, karg)
        return (dx, (dres if ctx.has_res else None), dw, db) + none


def _can_fuse(x, weight, residual, running_mean=True, emulate=False) -> bool:
    return ((x.is_cuda or emulate) and x.dim() == 4 and x.size(1) % 8 == 0 and x.size(1) <= 8192 and weight is not None and running_mean is not None
            and x.dtype in (torch.float32, torch.bfloat16, torch.float16)
            and x.is_contiguous(memory_format=torch.channels_last)
            and (residual is None or (residual.is_contiguous(memory_format=torch.channels_last) and residual.dtype == x.dtype
                                      and residual.shape == x.shape)))


def bn_act(x, weight, bias, running_mean, running_var, residual: Optional[torch.Tensor] = None, relu: bool = True,
           training: bool = True, momentum: Optional[float] = 0.1, eps: float = 1e-5, fused=None,
           num_batches_tracked: Optional[torch.Tensor] = None, split: bool = False, sync=None):
    """relu(batch_norm(x) + residual).  ``fused=None`` picks the CUDA kernels whenever the layout allows it;
    ``fused="emulate"`` runs the same autograd op over the PyTorch emulation of the kernels (CPU tests).
    ``split=True`` returns the result twice - two aliases of one buffer for the two consumers of a residual block's
    output - so that backward receives their gradients separately and fuses the add (``bn_act_backward2``).
    ``sync``: a ``SyncContext`` of world > 1 synchronises the training-mode statistics over the ranks.
    ``momentum=None``: cumulative average of the running statistics, as ``torch.nn.BatchNorm2d`` (unfused path)."""
    y = _bn_act(x, weight, bias, running_mean, running_var, residual, relu, training, momentum, eps, fused, num_batches_tracked, split,
                effective(sync, training))
    if split and not isinstance(y, tuple):
        return y, y
    return y


class _SyncBnCpuFn(torch.autograd.Function):
    """Synchronised BatchNorm in plain PyTorch over the communicator's ``all_reduce_`` (torch's SyncBatchNorm function has
    no CPU kernels): the same statistics contract as the fused kernels, any layout."""

    @staticmethod
    def forward(ctx, x, weight, bias, running_mean, running_var, eps, momentum, sync):
        c = x.size(1)
        xf = x.float()
        dims = [d for d in range(x.dim()) if d != 1]
        shape = [1, c] + [1] * (x.dim() - 2)
        g, n = _Emu._global_sums(torch.cat([xf.sum(dims), (xf * xf).sum(dims)]), x.numel() // c, sync)
        mean = g[:c] / n
        var = (g[c:] / n - mean * mean).clamp_min(0)
        invstd = torch.rsqrt(var + eps)
        if running_mean is not None:
            running_mean.mul_(1 - momentum).add_(momentum * mean)
            running_var.mul_(1 - momentum).add_(momentum * var * (n / (n - 1) if n > 1 else 1.0))
        xhat = (xf - mean.view(shape)) * invstd.view(shape)
        ctx.save_for_backward(xhat, weight, invstd)
        ctx.sync, ctx.dims, ctx.shape = sync, dims, shape
        return (xhat * weight.float().view(shape) + bias.float().view(shape)).to(x.dtype)

    @staticmethod
    def backward(ctx, dy):
        xhat, weight, invstd = ctx.saved_tensors
        c, shape = xhat.size(1), ctx.shape
        g = dy.float()
        sdz, sdzx = g.sum(ctx.dims), (g * xhat).sum(ctx.dims)
        tot, n = _Emu._global_sums(torch.cat([sdz, sdzx]), xhat.numel() // c, ctx.sync)
        dx = (weight.float() * invstd).view(shape) * (g - (tot[:c] / n).view(shape) - xhat * (tot[c:] / n).view(shape))
        return dx.to(dy.dtype), sdzx.to(weight.dtype), sdz.to(weight.dtype), None, None, None, None, None


def sync_batch_norm_unfused(x, weight, bias, running_mean, running_var, momentum, eps, num_batches_tracked, sync):
    """Layers the fused kernels cannot take (NCHW, C % 8 != 0, ...) and communicators other than the fused one: on CUDA
    ``torch.nn.SyncBatchNorm``'s own autograd function over the communicator's process group, on CPU the same semantics
    over the communicator's ``all_reduce_``.  ``momentum`` is the factor itself (``batch_norm_unfused`` resolves None)."""
    if not x.is_cuda:
        return _SyncBnCpuFn.apply(x, weight, bias, running_mean, running_var, eps, momentum, sync)
    if torch.cuda.is_current_stream_capturing():
        raise RuntimeError("synchronised BatchNorm on a layer the fused kernels cannot take (NCHW, C % 8 != 0, --no-fused-bn) "
                           "runs torch.distributed collectives, which a CUDA graph cannot capture")
    from torch.nn.modules._functions import SyncBatchNorm as _TorchSyncBN
    if weight is not None and weight.dtype != x.dtype:
        weight, bias = weight.to(x.dtype), bias.to(x.dtype)
    group = getattr(sync.comm, "group", None) or torch.distributed.group.WORLD
    return _TorchSyncBN.apply(x, weight, bias, running_mean, running_var, eps, momentum, group, sync.world)


def batch_norm_unfused(x, weight, bias, running_mean, running_var, training, momentum, eps, num_batches_tracked, sync, tail):
    """``tail(batch_norm(x))`` in plain PyTorch, for what the fused kernels cannot take.  ``tail`` is the rest of the op
    (residual add, ReLU, pooling); it receives the normalised tensor in the dtype the math ran in.
    ``momentum=None`` is ``torch.nn.BatchNorm2d``'s cumulative average: factor 1 / ``num_batches_tracked`` after the
    increment (a host read of the counter, as torch does), 0 without a counter."""
    if training and num_batches_tracked is not None:
        num_batches_tracked.add_(1)
        if momentum is None:
            momentum = 1.0 / float(num_batches_tracked)
    if momentum is None:
        momentum = 0.0
    if sync is not None:
        return tail(sync_batch_norm_unfused(x, weight, bias, running_mean, running_var, momentum, eps, num_batches_tracked, sync))
    if weight is not None and x.is_cuda and weight.dtype != torch.float32 and x.dtype != weight.dtype:
        weight, bias = weight.to(x.dtype), bias.to(x.dtype)
    if not x.is_cuda and x.dtype != torch.float32:
        # CPU batch_norm wants one dtype for activations and statistics: do the math in fp32 (test / debug path)
        y = F.batch_norm(x.float(), running_mean, running_var, None if weight is None else weight.float(),
                         None if bias is None else bias.float(), training, momentum, eps)
        return tail(y).to(x.dtype)
    return tail(F.batch_norm(x, running_mean, running_var, weight, bias, training, momentum, eps))


def _bn_act(x, weight, bias, running_mean, running_var, residual, relu, training, momentum, eps, fused, num_batches_tracked, split,
            sync=None):
    ok = _can_fuse(x, weight, residual, running_mean, emulate=(fused == "emulate"))
    use = ok if fused is None else (bool(fused) and ok)
    if momentum is None and training:   # cumulative average: its factor depends on num_batches_tracked (a host read)
        use = False
    if not use or (sync is not None and x.is_cuda and sync.native is None):
        def tail(y):
            if residual is not None:
                y = y + (residual if y.dtype == x.dtype else residual.to(y.dtype))
            return F.relu(y) if relu else y
        return batch_norm_unfused(x, weight, bias, running_mean, running_var, training, momentum, eps, num_batches_tracked, sync, tail)
    need_grad = torch.is_grad_enabled() and (x.requires_grad or weight.requires_grad or bias.requires_grad
                                             or (residual is not None and residual.requires_grad))
    if momentum is None:                # eval mode: the factor is not used
        momentum = 0.0
    if need_grad and not training:      # backward through frozen (eval-mode) statistics: rare, use the composition
        return bn_act_reference(x, weight.to(x.dtype) if weight.dtype != torch.float32 else weight,
                                bias.to(x.dtype) if bias.dtype != torch.float32 else bias, running_mean, running_var, residual, relu,
                                training, momentum, eps)
    return _BnActFn.apply(x, residual, weight, bias, running_mean, running_var, num_batches_tracked, training, float(momentum),
                          float(eps), relu, need_grad, None, bool(split and need_grad), sync)
