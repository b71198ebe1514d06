"""Native ResNet family (resnet18/34/50/101/152, resnext, wide_resnet).

Written from scratch; parameter / buffer names match torchvision's ResNet so the
reference checkpoint layout (``state_dict`` of the unwrapped module,
/root/reference/distributed.py:219-225) is interchangeable with torchvision.

What is H100-specific: every BatchNorm is a :class:`BNAct` that runs the
hand-written NHWC kernels in ``csrc/bn_act.cu`` (statistics pass + one fused
normalise(+residual add)(+ReLU) pass, and the matching two-pass backward), so a
bottleneck block issues 3 convs + 6 elementwise kernels instead of 3 convs + ~10.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from ..ops.bn_act import begin_step, bn_act
from ..ops.conv_bn import conv1x1_bn_act
from ..ops.stem import bn_relu_maxpool
from ..ops.stem_conv import can_use_stem_gemm, stem_conv_bn_relu_maxpool

# 1x1 conv -> BN pairs run as ONE wgmma GEMM with the BN statistics in its epilogue (ops/conv_bn.py; tools/gemm_probe.py
# compares it with cuDNN conv + a separate statistics pass over the ResNet-50 shapes).
# PTD_FUSED_CONV1X1=0 (or models.resnet.FUSED_CONV1X1 = False) restores cuDNN + bn_stats.
import os as _os
FUSED_CONV1X1 = _os.environ.get("PTD_FUSED_CONV1X1", "1") == "1"
# A block's output has two consumers (the next block's first conv and its skip connection).  With SPLIT_RESGRAD the last
# BNAct of a block hands out two aliases of its output, so the two gradients reach its backward separately and are
# summed inside the BN-backward reduction pass (csrc/bn_act.cu: bn_act_backward2) instead of by an autograd add:
# 7 instead of 9 tensor passes over the widest activations.
# PTD_SPLIT_RESGRAD=0 restores the autograd add.
SPLIT_RESGRAD = _os.environ.get("PTD_SPLIT_RESGRAD", "1") == "1"
# Stem 7x7 convolution as im2col + the wgmma GEMM with fused BN statistics instead of cuDNN's legacy C_in = 3 kernels
# (ops/stem_conv.py; tools/stem_gemm_probe.py compares the two).
# PTD_STEM_GEMM=0 restores cuDNN.
STEM_GEMM = _os.environ.get("PTD_STEM_GEMM", "1") == "1"


def _pair(x):
    """(input of the main path, input of the skip path) - the same tensor unless the producer split its output."""
    return x if isinstance(x, tuple) else (x, x)


class BNAct(nn.BatchNorm2d):
    """BatchNorm2d with optional fused residual add and ReLU: ``relu(bn(x) + residual)``."""

    def __init__(self, num_features, relu=True, fused=None, **kw):
        super().__init__(num_features, **kw)
        self.relu = relu
        self.fused = fused

    def forward(self, x, residual=None, split=False):  # type: ignore[override]
        training = self.training or not self.track_running_stats
        nbt = self.num_batches_tracked if (self.training and self.track_running_stats) else None   # bumped inside the kernel
        return bn_act(x, self.weight, self.bias, self.running_mean, self.running_var, residual=residual, relu=self.relu,
                      training=training, momentum=self.momentum, eps=self.eps, fused=self.fused,
                      num_batches_tracked=nbt, split=split, sync=self.sync_context())

    def sync_context(self):
        """The ``sync=`` handle of this layer's training-mode statistics: None (per-rank statistics)."""
        return None


def check_process_group(process_group) -> None:
    """Synchronised BatchNorm spans the whole world: a subgroup is rejected (as apex DDP rejects its unsupported arguments)."""
    import torch.distributed as dist
    if process_group is None or (dist.is_available() and dist.is_initialized() and process_group is dist.group.WORLD):
        return
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(process_group) == dist.get_world_size():
        return
    raise NotImplementedError("process_group: synchronised BatchNorm over a subgroup of the ranks is not supported; "
                              "pass None (the whole world)")


class SyncBNAct(BNAct):
    """``BNAct`` whose training-mode statistics cover the global batch of all data-parallel ranks, with the semantics of
    ``torch.nn.SyncBatchNorm``: mean / variance of the concatenated batch, running variance with the global unbiased
    factor, input gradients through the global sums, weight / bias gradients from this rank's sums (the DDP average
    then matches torch).  Eval mode and a world of 1 are plain ``BNAct``.

    The layer binds to the process's communicator (``utils.dist_ops.set_default_communicator``, registered by this
    package's DDP, apex DDP and ``hvd.init``) at its first training forward with world > 1.  With the fused communicator
    the statistics are exchanged inside the fused BatchNorm kernels (``csrc/sync_bn.cu``); layers those kernels cannot
    take, and other communicators, run ``torch.nn.SyncBatchNorm``'s autograd function over the process group.  So does
    ``momentum=None`` (cumulative average) on every communicator, the fused one included: it needs an initialised
    ``torch.distributed`` process group and cannot be captured in a CUDA graph."""

    def __init__(self, num_features, eps=1e-5, momentum=0.1, affine=True, track_running_stats=True, process_group=None, relu=False,
                 fused=None, **kw):
        check_process_group(process_group)
        super().__init__(num_features, relu=relu, fused=fused, eps=eps, momentum=momentum, affine=affine,
                         track_running_stats=track_running_stats, **kw)
        self._sync = None

    def sync_context(self):
        if not self.training:          # eval mode never synchronises (torch: need_sync = bn_training and self.training)
            return None
        if self._sync is None:
            import torch.distributed as dist
            if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
                return None
            from ..ops.sync_bn import SyncContext
            from ..utils.dist_ops import default_communicator
            comm = default_communicator()
            if comm is None:
                raise RuntimeError("SyncBatchNorm: no communicator is registered for this process; wrap the model in this "
                                   "package's DistributedDataParallel (or apex DDP, or call hvd.init()) before the first "
                                   "training forward, or call utils.dist_ops.set_default_communicator(comm)")
            self._sync = SyncContext.for_communicator(comm)
        return self._sync if self._sync.world > 1 else None

    @classmethod
    def convert_sync_batchnorm(cls, module, process_group=None):
        return convert_sync_batchnorm(module, process_group)


def _to_sync(bn: nn.modules.batchnorm._BatchNorm) -> SyncBNAct:
    new = SyncBNAct(bn.num_features, eps=bn.eps, momentum=bn.momentum, affine=bn.affine, track_running_stats=bn.track_running_stats,
                    relu=getattr(bn, "relu", False), fused=getattr(bn, "fused", None))
    new.training = bn.training
    if bn.affine:                      # the very same Parameter objects: optimizers, DDP hooks and state_dict keys stay valid
        new.weight, new.bias = bn.weight, bn.bias
    for name in ("running_mean", "running_var", "num_batches_tracked"):
        new._buffers[name] = bn._buffers.get(name)
    return new


def convert_sync_batchnorm(module: nn.Module, process_group=None) -> nn.Module:
    """Every ``nn.BatchNorm2d`` (including ``BNAct``, keeping its ReLU) and ``torch.nn.SyncBatchNorm`` of ``module`` becomes a
    :class:`SyncBNAct` sharing its Parameter and buffer objects; returns the converted module (``module`` itself unless it
    is a BatchNorm layer), like ``torch.nn.SyncBatchNorm.convert_sync_batchnorm``."""
    check_process_group(process_group)
    if isinstance(module, (nn.BatchNorm2d, nn.SyncBatchNorm)) and not isinstance(module, SyncBNAct):
        return _to_sync(module)
    for name, child in module.named_children():
        new = convert_sync_batchnorm(child, process_group)
        if new is not child:
            setattr(module, name, new)
    return module


def _conv3x3(cin, cout, stride=1, groups=1, dilation=1):
    return nn.Conv2d(cin, cout, 3, stride=stride, padding=dilation, groups=groups, bias=False, dilation=dilation)


def _conv1x1(cin, cout, stride=1):
    return nn.Conv2d(cin, cout, 1, stride=stride, bias=False)


class _Downsample(nn.Sequential):
    """conv1x1 + BN (no ReLU); indices 0/1 keep torchvision's ``downsample.0/1`` keys."""

    def __init__(self, cin, cout, stride, fused):
        super().__init__(_conv1x1(cin, cout, stride), BNAct(cout, relu=False, fused=fused))

    def forward(self, x):        # stride-1 projections (layer1) take the wgmma GEMM + fused statistics path
        return conv1x1_bn_act(x, self[0], self[1], enabled=FUSED_CONV1X1)


class BasicBlock(nn.Module):
    expansion = 1

    def __init__(self, cin, planes, stride=1, downsample=None, groups=1, base_width=64, fused=None):
        super().__init__()
        if groups != 1 or base_width != 64:
            raise ValueError("BasicBlock only supports groups=1 and base_width=64")
        self.conv1 = _conv3x3(cin, planes, stride)
        self.bn1 = BNAct(planes, relu=True, fused=fused)
        self.conv2 = _conv3x3(planes, planes)
        self.bn2 = BNAct(planes, relu=True, fused=fused)
        self.downsample = downsample
        self.stride = stride

    def forward(self, x):
        x, skip = _pair(x)
        identity = skip if self.downsample is None else self.downsample(skip)
        out = self.bn1(self.conv1(x))
        return self.bn2(self.conv2(out), identity, split=SPLIT_RESGRAD and self.training)


class Bottleneck(nn.Module):
    expansion = 4

    def __init__(self, cin, planes, stride=1, downsample=None, groups=1, base_width=64, fused=None):
        super().__init__()
        width = int(planes * (base_width / 64.0)) * groups
        self.conv1 = _conv1x1(cin, width)
        self.bn1 = BNAct(width, relu=True, fused=fused)
        self.conv2 = _conv3x3(width, width, stride, groups)
        self.bn2 = BNAct(width, relu=True, fused=fused)
        self.conv3 = _conv1x1(width, planes * self.expansion)
        self.bn3 = BNAct(planes * self.expansion, relu=True, fused=fused)
        self.downsample = downsample
        self.stride = stride

    def forward(self, x):
        x, skip = _pair(x)
        identity = skip if self.downsample is None else self.downsample(skip)
        out = conv1x1_bn_act(x, self.conv1, self.bn1, enabled=FUSED_CONV1X1)
        out = self.bn2(self.conv2(out))
        return conv1x1_bn_act(out, self.conv3, self.bn3, identity, enabled=FUSED_CONV1X1, split=SPLIT_RESGRAD and self.training)


class ResNet(nn.Module):
    def __init__(self, block, layers, num_classes=1000, groups=1, width_per_group=64, fused_bn=None,
                 zero_init_residual=False):
        super().__init__()
        self.inplanes = 64
        self.groups = groups
        self.base_width = width_per_group
        self.fused_bn = fused_bn
        self.conv1 = nn.Conv2d(3, 64, 7, stride=2, padding=3, bias=False)
        self.bn1 = BNAct(64, relu=True, fused=fused_bn)
        self.maxpool = nn.MaxPool2d(3, stride=2, padding=1)
        self.layer1 = self._make_layer(block, 64, layers[0])
        self.layer2 = self._make_layer(block, 128, layers[1], stride=2)
        self.layer3 = self._make_layer(block, 256, layers[2], stride=2)
        self.layer4 = self._make_layer(block, 512, layers[3], stride=2)
        self.avgpool = nn.AdaptiveAvgPool2d((1, 1))
        self.fc = nn.Linear(512 * block.expansion, num_classes)
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")
            elif isinstance(m, nn.BatchNorm2d):
                nn.init.constant_(m.weight, 1.0)
                nn.init.constant_(m.bias, 0.0)
        if zero_init_residual:
            for m in self.modules():
                if isinstance(m, Bottleneck):
                    nn.init.constant_(m.bn3.weight, 0.0)
                elif isinstance(m, BasicBlock):
                    nn.init.constant_(m.bn2.weight, 0.0)

    def _make_layer(self, block, planes, blocks, stride=1):
        down = None
        if stride != 1 or self.inplanes != planes * block.expansion:
            down = _Downsample(self.inplanes, planes * block.expansion, stride, self.fused_bn)
        layers = [block(self.inplanes, planes, stride, down, self.groups, self.base_width, self.fused_bn)]
        self.inplanes = planes * block.expansion
        for _ in range(1, blocks):
            layers.append(block(self.inplanes, planes, groups=self.groups, base_width=self.base_width,
                                fused=self.fused_bn))
        return nn.Sequential(*layers)

    def forward(self, x):
        if self.training:
            begin_step(x.device)      # recycle the BN accumulator workspace: one memset per step
        bn = self.bn1
        sync = bn.sync_context()
        if STEM_GEMM and bn.training and torch.is_grad_enabled() and bn.fused is not False and (
                (can_use_stem_gemm(x, self.conv1) and (sync is None or sync.native is not None) and bn.momentum is not None)
                or bn.fused == "emulate"):
            x = stem_conv_bn_relu_maxpool(x, self.conv1, bn, emulate=bn.fused == "emulate")
            x = self.layer4(self.layer3(self.layer2(self.layer1(x))))
            return self.fc(torch.flatten(self.avgpool(_pair(x)[0]), 1))
        nbt = bn.num_batches_tracked if (bn.training and bn.track_running_stats) else None
        x = bn_relu_maxpool(self.conv1(x), bn.weight, bn.bias, bn.running_mean, bn.running_var,   # fused stem tail
                            training=bn.training or not bn.track_running_stats, momentum=bn.momentum,
                            eps=bn.eps, fused=bn.fused, num_batches_tracked=nbt, sync=bn.sync_context())
        x = self.layer4(self.layer3(self.layer2(self.layer1(x))))
        x = _pair(x)[0]               # the last block has a single consumer: its second alias stays unused (gradient None)
        return self.fc(torch.flatten(self.avgpool(x), 1))


def _factory(block, layers, **fixed):
    def make(num_classes=1000, fused_bn=None, **kw):
        return ResNet(block, layers, num_classes=num_classes, fused_bn=fused_bn, **fixed, **kw)
    return make


FACTORIES = {
    "resnet18": _factory(BasicBlock, [2, 2, 2, 2]),
    "resnet34": _factory(BasicBlock, [3, 4, 6, 3]),
    "resnet50": _factory(Bottleneck, [3, 4, 6, 3]),
    "resnet101": _factory(Bottleneck, [3, 4, 23, 3]),
    "resnet152": _factory(Bottleneck, [3, 8, 36, 3]),
    "resnext50_32x4d": _factory(Bottleneck, [3, 4, 6, 3], groups=32, width_per_group=4),
    "resnext101_32x8d": _factory(Bottleneck, [3, 4, 23, 3], groups=32, width_per_group=8),
    "resnext101_64x4d": _factory(Bottleneck, [3, 4, 23, 3], groups=64, width_per_group=4),
    "wide_resnet50_2": _factory(Bottleneck, [3, 4, 6, 3], width_per_group=128),
    "wide_resnet101_2": _factory(Bottleneck, [3, 4, 23, 3], width_per_group=128),
}
