"""Input pipeline: ImageFolder loaders, synthetic ImageNet-shaped data, and the CUDA-stream prefetcher.

Reference: dataset/sampler/loader wiring at /root/reference/distributed.py:160-195 and the side-stream
``data_prefetcher`` at /root/reference/apex_distributed.py:115-169.  Deviations: ``-j/--workers`` is honoured
(SURVEY Q3), every entrypoint shards the validation set (Q6), the prefetcher never normalises twice (Q5), and a
synthetic dataset exists because neither the dev box nor the GPU boxes have ImageNet.
"""
from __future__ import annotations

import math
import os
from typing import Iterator, Optional, Tuple

import torch
import torch.distributed as dist

from .shards import StagedBatch

IMAGENET_MEAN = (0.485, 0.456, 0.406)
IMAGENET_STD = (0.229, 0.224, 0.225)
IMAGENET_TRAIN_SIZE = 1281167
IMAGENET_VAL_SIZE = 50000


class _EpochSampler:
    """Stand-in for DistributedSampler on loaders that shard by construction."""

    def __init__(self):
        self.epoch = 0

    def set_epoch(self, epoch: int) -> None:
        self.epoch = epoch


class SyntheticLoader:
    """Yields ``steps`` batches of ImageNet-shaped data from a small pool of pre-generated **pinned host** batches.

    Every step still pays the real host->device copy (the pool lives in pinned memory, exactly like the output of a
    ``DataLoader(pin_memory=True)``); only JPEG decoding is taken out of the picture.  ``raw_uint8=True`` emulates a
    loader that ships un-normalised uint8 images (the apex prefetcher's input contract).
    """

    def __init__(self, batch_size: int, steps: int, image_size: int = 224, num_classes: int = 1000, pool: int = 4,
                 seed: int = 0, raw_uint8: bool = False, pin: Optional[bool] = None, rank: int = 0):
        self.batch_size, self.steps = int(batch_size), int(steps)
        self.raw_uint8 = bool(raw_uint8)
        self.sampler = _EpochSampler()
        g = torch.Generator().manual_seed(1234 + seed * 7919 + rank * 104729)
        pin = torch.cuda.is_available() if pin is None else pin
        self.pool = []
        for _ in range(max(1, pool)):
            if raw_uint8:
                img = torch.randint(0, 256, (batch_size, 3, image_size, image_size), generator=g, dtype=torch.uint8)
            else:
                img = torch.randn(batch_size, 3, image_size, image_size, generator=g)
            tgt = torch.randint(0, num_classes, (batch_size,), generator=g, dtype=torch.int64)
            if pin:
                img, tgt = img.pin_memory(), tgt.pin_memory()
            self.pool.append((img, tgt))
        self.bytes_per_step = self.pool[0][0].numel() * self.pool[0][0].element_size() + self.pool[0][1].numel() * 8

    def __len__(self) -> int:
        return self.steps

    def __iter__(self) -> Iterator[Tuple[torch.Tensor, torch.Tensor]]:
        for i in range(self.steps):
            yield self.pool[(i + self.sampler.epoch) % len(self.pool)]


def _world():
    return (dist.get_rank(), dist.get_world_size()) if dist.is_available() and dist.is_initialized() else (0, 1)


def augmenting(args) -> bool:
    """``--auto-augment`` or ``--random-erase`` is on."""
    return getattr(args, "auto_augment", None) is not None or float(getattr(args, "random_erase", 0.0) or 0.0) > 0


def build_loaders(args, batch_size: int, distributed: bool = True, raw_uint8: bool = False):
    """(train_loader, val_loader, train_sampler, val_sampler) for this rank.  ``batch_size`` is per loader.

    With ``--auto-augment`` / ``--random-erase``: shard and synthetic training batches are uint8 (the prefetcher augments
    them on the device, ``ops/augment.py``), and ``ImageFolder`` workers run torchvision's transforms themselves."""
    rank, world = _world() if distributed else (0, 1)
    aug = augmenting(args)
    if args.data and not args.synthetic:
        from . import shards
        if shards.find_shards(args.data, "train"):          # pre-decoded shards -> native C++ loader (always uint8 batches)
            return shards.build_shard_loaders(args, batch_size, rank, world)
    use_synth = args.synthetic or not args.data or not os.path.isdir(os.path.join(args.data, "train"))
    if use_synth:
        shards = world if distributed else 1
        n_train = args.synthetic_size or IMAGENET_TRAIN_SIZE
        n_val = max(1, (args.synthetic_size or IMAGENET_VAL_SIZE * 25) // 25) if args.synthetic_size else IMAGENET_VAL_SIZE
        tsteps = args.steps_per_epoch or max(1, math.ceil(n_train / shards / batch_size))
        vsteps = args.val_steps or args.steps_per_epoch or max(1, math.ceil(n_val / shards / batch_size))
        seed = args.seed or 0
        train = SyntheticLoader(batch_size, tsteps, args.image_size, args.num_classes, seed=seed, raw_uint8=raw_uint8 or aug, rank=rank)
        val = SyntheticLoader(batch_size, vsteps, args.image_size, args.num_classes, seed=seed + 1, raw_uint8=raw_uint8, rank=rank)
        return train, val, train.sampler, val.sampler
    import torchvision.datasets as datasets
    import torchvision.transforms as transforms
    normalize = transforms.Normalize(mean=IMAGENET_MEAN, std=IMAGENET_STD)
    tail = [transforms.PILToTensor()] if raw_uint8 else [transforms.ToTensor(), normalize]
    train_ds = datasets.ImageFolder(os.path.join(args.data, "train"), transforms.Compose(train_transforms(args, raw_uint8)))
    val_ds = datasets.ImageFolder(os.path.join(args.data, "val"), transforms.Compose(
        [transforms.Resize(int(args.image_size * 256 / 224)), transforms.CenterCrop(args.image_size)] + tail))
    if distributed and world > 1:
        ts = torch.utils.data.distributed.DistributedSampler(train_ds)
        vs = torch.utils.data.distributed.DistributedSampler(val_ds)
    else:
        ts, vs = None, None
    pin = torch.cuda.is_available()
    # a captured step replays one batch shape: under --cuda-graph the ragged last training batch is dropped (validation is eager)
    train = torch.utils.data.DataLoader(train_ds, batch_size=batch_size, shuffle=(ts is None), num_workers=args.workers,
                                        pin_memory=pin, sampler=ts, persistent_workers=args.workers > 0,
                                        drop_last=bool(getattr(args, "cuda_graph", False)) and len(train_ds) >= batch_size * max(1, world))
    val = torch.utils.data.DataLoader(val_ds, batch_size=batch_size, shuffle=False, num_workers=args.workers, pin_memory=pin,
                                      sampler=vs, persistent_workers=args.workers > 0)
    return train, val, ts or _EpochSampler(), vs or _EpochSampler()


def train_transforms(args, raw_uint8: bool = False):
    """The ``ImageFolder`` training transforms: the crop and flip, then (``--auto-augment ta_wide``) TrivialAugmentWide or
    (``--auto-augment imagenet|cifar10|svhn``) AutoAugment on the crop and (``--random-erase P``) RandomErasing after
    ``Normalize``, in the order of torchvision's classification recipe.
    With ``raw_uint8`` the workers ship uint8 tensors and the prefetcher normalises and augments them."""
    import torchvision.transforms as transforms
    t = [transforms.RandomResizedCrop(args.image_size), transforms.RandomHorizontalFlip()]
    if raw_uint8:
        return t + [transforms.PILToTensor()]
    policy = getattr(args, "auto_augment", None)
    if policy == "ta_wide":
        t.append(transforms.TrivialAugmentWide(interpolation=transforms.InterpolationMode.BILINEAR))
    elif policy is not None:
        t.append(transforms.AutoAugment(transforms.AutoAugmentPolicy(policy), interpolation=transforms.InterpolationMode.BILINEAR))
    t += [transforms.ToTensor(), transforms.Normalize(mean=IMAGENET_MEAN, std=IMAGENET_STD)]
    p = float(getattr(args, "random_erase", 0.0) or 0.0)
    if p > 0:
        t.append(transforms.RandomErasing(p=p))
    return t


def _limited(loader, limit: Optional[int]):
    if limit is None:
        yield from loader
        return
    for i, b in enumerate(loader):
        if i >= limit:
            return
        yield b


class DataPrefetcher:
    """Double-buffered host->device pipeline on a side stream.

    For each batch: async copy of the pinned tensors, then ONE fused kernel (``csrc/data_ops.cu``) that applies the
    optional per-channel normalisation, casts to the compute dtype and writes channels_last - replacing the reference
    prefetcher's ``.float()``, ``sub_``, ``div_`` chain and the layout/dtype conversions the model would otherwise do.
    ``record_stream`` keeps the caching allocator from recycling a batch while the compute stream still reads it.

    ``augment`` (a :class:`~..ops.augment.BatchAugment`, training batches of uint8 pixels only): each batch's draws are made
    on the host as it is staged, copied with it, and the kernel that normalises it augments it too (``augment_normalize``;
    a staged shard batch is first resampled to uint8 on the device).
    """

    def __init__(self, loader, device, dtype: torch.dtype = torch.float32, channels_last: bool = False,
                 normalize: Optional[str] = None, limit: Optional[int] = None, augment=None):
        self.device = torch.device(device)
        self.dtype = dtype
        self.channels_last = channels_last
        self.limit = limit
        self.loader = loader
        self.cuda = self.device.type == "cuda"
        self.h2d_bytes = 0
        if normalize == "imagenet255":      # raw uint8 pixels -> normalised
            a = [1.0 / (255.0 * s) for s in IMAGENET_STD]
            b = [-m / s for m, s in zip(IMAGENET_MEAN, IMAGENET_STD)]
        elif normalize is None:
            a, b = [1.0] * 3, [0.0] * 3
        else:
            raise ValueError("unknown normalisation %r" % (normalize,))
        self._a = torch.tensor(a, dtype=torch.float32, device=self.device)
        self._b = torch.tensor(b, dtype=torch.float32, device=self.device)
        self.identity = normalize is None
        if augment is not None and normalize != "imagenet255":
            raise ValueError("augmentation needs a loader of uint8 pixels")
        self.augment = augment
        self.stream = torch.cuda.Stream(device=self.device) if self.cuda else None

    def __len__(self):
        n = len(self.loader)
        return n if self.limit is None else min(n, self.limit)

    def _convert(self, img: torch.Tensor) -> torch.Tensor:
        if self.cuda and img.dim() == 4 and img.size(1) == 3 and img.is_contiguous():
            from .. import _ext
            code = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}[self.dtype]
            _ext.note_launch()
            return _ext.lib().normalize_nhwc(img, self._a, self._b, code, self.channels_last)
        img = img.to(self.dtype)
        if not self.identity:
            img = img * self._a.view(1, -1, 1, 1).to(self.dtype) + self._b.view(1, -1, 1, 1).to(self.dtype)
        if self.channels_last and img.dim() == 4:
            img = img.contiguous(memory_format=torch.channels_last)
        return img

    def _resample(self, staged, arena: torch.Tensor) -> torch.Tensor:
        """A shard batch staged for the device resample (utils/shards.StagedBatch) -> what _convert gives for the
        host-resampled uint8 batch, bit for bit."""
        from .. import _ext
        code = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}[self.dtype]
        _ext.note_launch()
        return _ext.lib().resample_normalize(arena, staged.n, staged.out_h, staged.out_w, staged.max_rows, self._a, self._b, code,
                                             self.channels_last)

    def _stage(self, batch):
        img, tgt = batch
        staged = isinstance(img, StagedBatch)
        src = img.data if staged else img
        self.h2d_bytes += src.numel() * src.element_size() + tgt.numel() * tgt.element_size()
        if self.augment is not None:
            return self._stage_augmented(img, src, tgt, staged)
        if not self.cuda:
            if staged:
                raise RuntimeError("a batch staged for the device resample needs a CUDA prefetcher")
            return self._convert(img), tgt
        with torch.cuda.stream(self.stream):
            src = src.to(self.device, non_blocking=True)
            tgt = tgt.to(self.device, non_blocking=True)
            if hasattr(self.loader, "batch_copied"):         # ring-buffer loaders recycle the pinned slot after this event
                ev = torch.cuda.Event()
                ev.record(self.stream)
                self.loader.batch_copied(ev)
            img = self._resample(img, src) if staged else self._convert(src)
        return img, tgt

    def _stage_augmented(self, img, src, tgt, staged):
        n, _, H, W = img.shape
        prm = self.augment.draw(n, H, W)
        self.h2d_bytes += prm.numel() * 4
        if not self.cuda:
            if staged:
                raise RuntimeError("a batch staged for the device resample needs a CUDA prefetcher")
            return self.augment.apply(img, prm, self._a, self._b, self.dtype, self.channels_last), tgt
        from .. import _ext
        with torch.cuda.stream(self.stream):
            src = src.to(self.device, non_blocking=True)
            tgt = tgt.to(self.device, non_blocking=True)
            prm_d = prm.to(self.device, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(self.stream)
            if hasattr(self.loader, "batch_copied"):
                self.loader.batch_copied(ev)
            self.augment.copied(prm, ev)
            if staged:
                _ext.note_launch()
                src = _ext.lib().resample_normalize(src, img.n, img.out_h, img.out_w, img.max_rows, self._a, self._b,
                                                    _ext.lib().U8_OUT, False)
            out = self.augment.apply(src, prm_d, self._a, self._b, self.dtype, self.channels_last)
        return out, tgt

    def next(self):
        """Reference-style pull API (``data_prefetcher.next()`` in /root/reference/apex_distributed.py:160-169):
        returns ``(input, target)`` and ``(None, None)`` when the loader is exhausted."""
        if getattr(self, "_gen", None) is None:
            self._gen = iter(self)
        try:
            return next(self._gen)
        except StopIteration:
            self._gen = None
            return None, None

    def __iter__(self):
        it = iter(_limited(self.loader, self.limit))
        nxt = None
        try:
            nxt = self._stage(next(it))
        except StopIteration:
            return
        while nxt is not None:
            if self.cuda:
                torch.cuda.current_stream(self.device).wait_stream(self.stream)
                for t in nxt:
                    t.record_stream(torch.cuda.current_stream(self.device))
            cur = nxt
            try:
                nxt = self._stage(next(it))
            except StopIteration:
                nxt = None
            yield cur


data_prefetcher = DataPrefetcher   # the reference's class name
