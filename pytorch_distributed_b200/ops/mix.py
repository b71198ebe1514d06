"""MixUp, CutMix and label smoothing for training (``--mixup-alpha``, ``--cutmix-alpha``, ``--label-smoothing``).

The semantics are torchvision's: ``transforms.v2.MixUp`` / ``CutMix`` (sample n is paired with sample n - 1 mod B, as
``roll(1, 0)`` does), the 50/50 ``RandomChoice`` between them of ``references/classification/train.py``, and
``nn.CrossEntropyLoss(label_smoothing=eps)`` over the mixed probability targets.

On the GPU the batch is mixed by one ``mix_batch`` pass (``csrc/mix.cu``) that also writes the paired labels and the
dominant label (what the metric kernel counts, as torchvision's ``utils.accuracy`` counts ``target.max(1)[1]``), and the
loss is ``soft_ce_fwd`` / ``soft_ce_bwd``: no ``[B, C]`` target, no fp32 copy of the logits.  Every per-step value sits in a
float[8] device tensor that ``draw()`` rewrites before each pass, so a captured CUDA graph follows the new draws.  On CPU
tensors the same operations are plain torch code with the same formulas; that code is also the reference of the GPU tests.
"""
from __future__ import annotations

import math
from typing import NamedTuple, Optional

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

MIXUP, CUTMIX = 1, 2


def cutmix_box(lam: float, r_x: int, r_y: int, H: int, W: int):
    """torchvision's ``CutMix.make_params`` for a drawn ``lam`` and centre ``(r_x, r_y)``: the box ``(x1, y1, x2, y2)``
    (columns [x1, x2), rows [y1, y2)) and the lambda adjusted to the box's area."""
    r = 0.5 * math.sqrt(1.0 - lam)
    r_w_half = int(r * W)
    r_h_half = int(r * H)
    x1 = max(r_x - r_w_half, 0)
    y1 = max(r_y - r_h_half, 0)
    x2 = min(r_x + r_w_half, W)
    y2 = min(r_y + r_h_half, H)
    return (x1, y1, x2, y2), float(1.0 - (x2 - x1) * (y2 - y1) / (W * H))


def lam_pair(lam: float):
    """(fp32(lam), fp32(1 - lam)) with 1 - lam taken in double: the two scalars torch multiplies an fp32 tensor by."""
    return float(np.float32(lam)), float(np.float32(1.0 - lam))


class MixTarget(NamedTuple):
    """The targets of one mixed batch: ``q = la onehot(y_a) + lb onehot(y_b)`` with ``la, lb = prm[1], prm[2]``, and the
    dominant label ``dom`` (its argmax, the smaller label on a tie)."""
    y_a: torch.Tensor
    y_b: torch.Tensor
    dom: torch.Tensor
    prm: torch.Tensor


def _identity_params(device) -> torch.Tensor:
    return torch.tensor([0, 1, 0, 0, 0, 0, 0, 0], dtype=torch.float32, device=device)


class _SoftCrossEntropy(torch.autograd.Function):
    @staticmethod
    def forward(ctx, z, y_a, y_b, prm, eps):
        from .. import _ext
        loss, _, lse = _ext.lib().soft_ce_fwd(z, y_a, y_b, prm, eps)
        _ext.note_launch(2)
        ctx.save_for_backward(z, y_a, y_b, prm, lse)
        ctx.eps = eps
        return loss

    @staticmethod
    def backward(ctx, g):
        from .. import _ext
        z, y_a, y_b, prm, lse = ctx.saved_tensors
        dz = _ext.lib().soft_ce_bwd(z, y_a, y_b, prm, lse, g.float(), ctx.eps)
        _ext.note_launch()
        return dz, None, None, None, None


def soft_cross_entropy(logits: torch.Tensor, target: MixTarget, eps: float) -> torch.Tensor:
    """Mean cross-entropy of ``logits`` against ``(1 - eps) q + eps / C`` (fp32 scalar).  CUDA: the fused kernels, for
    bf16 / fp16 / fp32 logits with a row stride.  CPU: torch's ``F.cross_entropy`` over the materialised target."""
    if logits.is_cuda:
        return _SoftCrossEntropy.apply(logits, target.y_a, target.y_b, target.prm, float(eps))
    la, lb = float(target.prm[1]), float(target.prm[2])
    C = logits.size(1)
    q = F.one_hot(target.y_b, C).float().mul_(lb).add_(F.one_hot(target.y_a, C).float().mul(la))
    return F.cross_entropy(logits.float(), q, label_smoothing=eps)


class SmoothedCrossEntropy(nn.Module):
    """``nn.CrossEntropyLoss(label_smoothing=eps)`` over integer targets: the soft-target kernels with lambda = 1 on the GPU."""

    def __init__(self, eps: float):
        super().__init__()
        self.eps = float(eps)
        self.register_buffer("prm", _identity_params("cpu"), persistent=False)

    def forward(self, output, target):
        if not output.is_cuda:
            return F.cross_entropy(output.float(), target, label_smoothing=self.eps)
        prm = self.prm if self.prm.device == output.device else self.prm.to(output.device)
        return soft_cross_entropy(output, MixTarget(target, target, target, prm), self.eps)


class BatchMix:
    """The training-time target policy: MixUp / CutMix draws, the mixing itself, the loss and the metric labels.

    ``draw(size)`` runs on the host before every training pass (eager or graph replay) and writes the parameters of the
    next ``apply`` into the device tensor ``prm``.  The draws come from ``numpy.random.Generator(PCG64([seed, rank,
    epoch]))``: ``set_epoch`` re-keys the stream, so a resume at an epoch boundary replays the same draws.  Without a
    seed, the seed comes from OS entropy.
    """

    def __init__(self, mixup_alpha: float = 0.0, cutmix_alpha: float = 0.0, label_smoothing: float = 0.0, num_classes: int = 1000,
                 seed: Optional[int] = None, rank: int = 0, device=None):
        for name, a in (("mixup_alpha", mixup_alpha), ("cutmix_alpha", cutmix_alpha)):
            if not (a >= 0 and math.isfinite(a)):
                raise ValueError("%s must be a finite number >= 0, got %r" % (name, a))
        if not 0.0 <= label_smoothing <= 1.0:
            raise ValueError("label_smoothing must lie in [0, 1], got %r" % (label_smoothing,))
        self.alphas = {MIXUP: float(mixup_alpha), CUTMIX: float(cutmix_alpha)}
        self.modes = [m for m in (MIXUP, CUTMIX) if self.alphas[m] > 0]
        self.label_smoothing = float(label_smoothing)
        self.num_classes = int(num_classes)
        self.seed = (int(seed) if seed is not None else np.random.SeedSequence().entropy) % (1 << 128)
        self.rank = int(rank)
        self.device = torch.device(device) if device is not None else torch.device("cpu")
        self.prm = _identity_params(self.device)       # rewritten by draw()
        self._identity = _identity_params(self.device)  # lambda = 1: integer targets
        self.last = {"mode": 0, "lam": 1.0, "box": (0, 0, 0, 0), "la": 1.0, "lb": 0.0}
        self.criterion = SmoothedCrossEntropy(self.label_smoothing).to(self.device)
        self._static = None                             # (key, out, y_b, dom) of the first batch shape
        self.set_epoch(0)

    @property
    def mixing(self) -> bool:
        return bool(self.modes)

    def set_epoch(self, epoch: int) -> None:
        self.rng = np.random.Generator(np.random.PCG64([self.seed, self.rank, int(epoch)]))

    def draw(self, size) -> dict:
        """Draw the next pass's mode, lambda and (CutMix) box for images of ``size = (H, W)``; returns them."""
        if not self.modes:
            return self.last
        mode = self.modes[0] if len(self.modes) == 1 else (MIXUP if self.rng.random() < 0.5 else CUTMIX)
        lam = float(self.rng.beta(self.alphas[mode], self.alphas[mode]))
        box, lam_t = (0, 0, 0, 0), lam
        if mode == CUTMIX:
            H, W = int(size[0]), int(size[1])
            r_x, r_y = int(self.rng.integers(W)), int(self.rng.integers(H))
            box, lam_t = cutmix_box(lam, r_x, r_y, H, W)
        la, lb = lam_pair(lam_t)
        self.last = {"mode": mode, "lam": lam_t, "box": box, "la": la, "lb": lb}
        host = torch.tensor([mode, la, lb, *box, 0], dtype=torch.float32)
        self.prm.copy_(host, non_blocking=self.prm.is_cuda)
        return self.last

    def _buffers(self, images, target):
        key = (images.shape, images.stride(), images.dtype, images.device)
        if self._static is not None and self._static[0] == key:
            return self._static[1:]
        bufs = (torch.empty_like(images), torch.empty_like(target), torch.empty_like(target))
        if self._static is None:
            self._static = (key,) + bufs
        return bufs

    def apply(self, images: torch.Tensor, target: torch.Tensor):
        """Mix the batch with its ``roll(1, 0)`` neighbour; returns ``(mixed images, MixTarget)``.  Without MixUp and CutMix
        (label smoothing alone) the batch passes through unchanged."""
        if not self.modes:
            return images, MixTarget(target, target, target, self._identity)
        if images.is_cuda:
            from .. import _ext
            out, y_b, dom = self._buffers(images, target)
            _ext.lib().mix_batch(images, out, target, y_b, dom, self.prm)
            _ext.note_launch()
            return out, MixTarget(target, y_b, dom, self.prm)
        return self.reference_apply(images, target, self.prm)

    @staticmethod
    def reference_apply(images: torch.Tensor, target: torch.Tensor, prm: torch.Tensor):
        """The CPU path: torchvision's formulas on the fp32 upcast of ``images``, rounded once to their dtype."""
        p = prm.cpu().tolist()
        mode, la, lb = int(p[0]), p[1], p[2]
        x1, y1, x2, y2 = (int(v) for v in p[3:7])
        x = images.float()
        if mode == MIXUP:
            out = x.roll(1, 0).mul_(lb).add_(x.mul(la))
        elif mode == CUTMIX:
            out = x.clone()
            out[..., y1:y2, x1:x2] = x.roll(1, 0)[..., y1:y2, x1:x2]
        else:
            out = x.clone()
        out = out.to(images.dtype)
        y_b = target.roll(1, 0)
        dom = target if la > lb else y_b if la < lb else torch.minimum(target, y_b)
        return out, MixTarget(target, y_b, dom, prm)

    def loss(self, output: torch.Tensor, target: MixTarget) -> torch.Tensor:
        return soft_cross_entropy(output, target, self.label_smoothing)

    @staticmethod
    def metric_target(target: MixTarget) -> torch.Tensor:
        return target.dom
