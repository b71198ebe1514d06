"""Pre-decoded image shards + the native loader that reads them.

The reference's input path is ``ImageFolder`` + PIL transforms inside DataLoader worker processes
(/root/reference/distributed.py:160-195).  That path is kept (``utils/data.build_loaders``); this module is the
production alternative for a node that consumes ~90k images/s: JPEGs are decoded ONCE into ``*.ptds`` shards
(``tools/make_shards.py``), and training reads them through ``csrc/host/loader.cpp`` - mmap, C++ worker threads doing
RandomResizedCrop + flip (train) or Resize + CenterCrop (val) with an antialiased bilinear filter, output written as
uint8 NCHW straight into pinned ring slots.  ``DataPrefetcher`` then does the H2D copy and the fused
normalise / cast / NHWC kernel exactly as for any other uint8 loader.  On a GPU run the threads only stage the source
pixels and filter taps of each crop (:class:`StagedBatch`) and the resample runs on the GPU (csrc/resample.cu) with
the same bits as output.

Shard layout (little endian): ``b"PTDSHRD1"``, u32 records, u32 index capacity, ``capacity`` x 24-byte index entries
``(u64 offset, u32 height, u32 width, i32 label, u32 channels=3)``, then the raw HWC uint8 pixels.
"""
from __future__ import annotations

import glob
import json
import os
import struct
from collections import deque
from typing import Iterator, List, Optional, Sequence, Tuple

import numpy as np
import torch

SUFFIX = ".ptds"
_HEADER = struct.Struct("<8sII")
_ENTRY = struct.Struct("<QIIiI")
MAGIC = b"PTDSHRD1"


class ShardWriter:
    """Single-pass writer: the index region is reserved up front for ``capacity`` records."""

    def __init__(self, path: str, capacity: int):
        self.path, self.capacity = path, int(capacity)
        self._f = open(path + ".tmp", "wb")
        self._f.write(b"\0" * (_HEADER.size + _ENTRY.size * self.capacity))
        self._entries: List[Tuple[int, int, int, int]] = []

    def __len__(self) -> int:
        return len(self._entries)

    @property
    def full(self) -> bool:
        return len(self._entries) >= self.capacity

    def add(self, image_hwc: np.ndarray, label: int) -> None:
        if self.full:
            raise RuntimeError("shard is full")
        a = np.ascontiguousarray(image_hwc, dtype=np.uint8)
        if a.ndim != 3 or a.shape[2] != 3:
            raise ValueError("expected an HxWx3 uint8 image, got %r" % (a.shape,))
        off = self._f.tell()
        self._f.write(a.tobytes())
        self._entries.append((off, a.shape[0], a.shape[1], int(label)))

    def close(self) -> None:
        if self._f is None:
            return
        self._f.seek(0)
        self._f.write(_HEADER.pack(MAGIC, len(self._entries), self.capacity))
        for off, h, w, label in self._entries:
            self._f.write(_ENTRY.pack(off, h, w, label, 3))
        self._f.close()
        self._f = None
        os.replace(self.path + ".tmp", self.path)

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


def read_index(path: str) -> List[Tuple[int, int, int, int]]:
    """(offset, height, width, label) of every record - pure Python, for tools and tests."""
    with open(path, "rb") as f:
        magic, n, _cap = _HEADER.unpack(f.read(_HEADER.size))
        if magic != MAGIC:
            raise ValueError("%s is not a shard file" % path)
        raw = f.read(_ENTRY.size * n)
    return [_ENTRY.unpack_from(raw, i * _ENTRY.size)[:4] for i in range(n)]


def find_shards(data_dir: str, split: str) -> List[str]:
    return sorted(glob.glob(os.path.join(data_dir, "%s-*%s" % (split, SUFFIX))))


def _decode(job):
    path, label, max_side = job
    from PIL import Image
    try:
        with Image.open(path) as im:
            im = im.convert("RGB")                       # grey-scale / CMYK / palette files of ImageNet included
            w, h = im.size
            short = min(w, h)
            if max_side and short > max_side:            # keep the aspect ratio: RandomResizedCrop still sees the whole image
                s = max_side / short
                im = im.resize((max(1, round(w * s)), max(1, round(h * s))), Image.BILINEAR)
            return np.asarray(im, dtype=np.uint8), label
    except Exception as e:                               # unreadable file: reported and skipped, like a filtered sample
        return None, "%s: %s" % (path, e)


def write_shards(split_dir: str, out_dir: str, split: str, max_side: int = 256, per_shard: int = 4096, workers: int = 0,
                 log=None) -> List[str]:
    """Decode the ``ImageFolder`` tree ``split_dir`` into ``out_dir/<split>-NNNNN.ptds`` (labels = sorted class dirs)."""
    from torchvision.datasets import ImageFolder
    ds = ImageFolder(split_dir)
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "%s-classes.json" % split), "w") as f:
        json.dump(ds.classes, f)
    jobs = [(p, y, max_side) for p, y in ds.samples]
    paths: List[str] = []
    writer: Optional[ShardWriter] = None
    pool = None
    if workers > 0:
        import multiprocessing as mp
        pool = mp.get_context("spawn").Pool(workers)
        stream = pool.imap(_decode, jobs, chunksize=32)
    else:
        stream = map(_decode, jobs)
    try:
        for i, (arr, label) in enumerate(stream):
            if arr is None:
                (log or print)("skipped unreadable image %s" % (label,))
                continue
            if writer is None or writer.full:
                if writer is not None:
                    writer.close()
                paths.append(os.path.join(out_dir, "%s-%05d%s" % (split, len(paths), SUFFIX)))
                writer = ShardWriter(paths[-1], min(per_shard, len(jobs) - i))
            writer.add(arr, label)
            if log and (i + 1) % 10000 == 0:
                log("%s: %d / %d" % (split, i + 1, len(jobs)))
    finally:
        if writer is not None:
            writer.close()
        if pool is not None:
            pool.close()
            pool.join()
    return paths


class _Sampler:
    def __init__(self, owner):
        self._owner = owner

    def set_epoch(self, epoch: int) -> None:
        self._owner.epoch = int(epoch)


class StagedBatch:
    """A batch staged for resampling on the GPU (``ShardLoader(device_resample=True)``).

    ``data`` is the used prefix of a pinned ring-slot arena: ``n`` 32-byte descriptors, then per sample the source
    rectangle its filter taps read and the taps themselves (layout: ``StageDesc`` in csrc/host/loader.cpp).
    ``DataPrefetcher`` copies it to the device and expands it with the ``resample_normalize`` kernel into the tensor
    ``normalize_nhwc`` makes of the host-resampled ``uint8 [n, 3, out_h, out_w]`` batch, bit for bit.
    ``max_rows`` bounds the source rows one output row reads (it sizes the kernel's shared memory).
    """

    __slots__ = ("data", "n", "out_h", "out_w", "max_rows")

    def __init__(self, data: torch.Tensor, n: int, out_h: int, out_w: int, max_rows: int):
        self.data, self.n, self.out_h, self.out_w, self.max_rows = data, int(n), int(out_h), int(out_w), int(max_rows)

    @property
    def shape(self) -> Tuple[int, int, int, int]:
        return (self.n, 3, self.out_h, self.out_w)


class ShardLoader:
    """Iterable over ``(uint8 [B,3,H,W], int64 [B])`` batches living in a ring of (pinned) host buffers.

    Contract: a yielded batch stays valid while the next one is drawn and is recycled when the one after that is
    requested; when the consumer reports its copy with :meth:`batch_copied` (``DataPrefetcher`` does) the slot is
    instead held until that CUDA event has completed.
    ``sampler.set_epoch(e)`` selects the permutation of the next ``iter()``; sharding across ranks follows
    ``DistributedSampler`` (pad by wrapping, rank ``r`` takes positions ``r, r + world, ...``).

    ``device_resample=True`` yields :class:`StagedBatch` instead of the uint8 images: the worker threads only pick the
    crop box, build the filter taps and copy the source pixels those taps read, and the resample runs on the GPU.
    Crop boxes, order, labels, ids and the slot protocol are the same as in the default mode.
    """

    raw_uint8 = True            # DataPrefetcher must apply the ImageNet mean/std to these pixels

    def __init__(self, paths: Sequence[str], batch_size: int, image_size: int = 224, train: bool = True, seed: int = 0,
                 rank: int = 0, world: int = 1, workers: int = 4, depth: int = 4, drop_last: bool = False,
                 shuffle: Optional[bool] = None, pin: Optional[bool] = None, with_ids: bool = False,
                 scale: Tuple[float, float] = (0.08, 1.0), ratio: Tuple[float, float] = (3.0 / 4.0, 4.0 / 3.0),
                 device_resample: bool = False):
        from .. import _hostext
        if not paths:
            raise ValueError("no shard files given")
        depth = max(3, int(depth))
        self._L = _hostext.lib().ShardLoader(
            list(paths), int(batch_size), int(image_size), int(image_size), bool(train), int(seed) & (2 ** 63 - 1), int(rank),
            int(world), max(1, int(workers)), depth, bool(drop_last), bool(train if shuffle is None else shuffle),
            float(scale[0]), float(scale[1]), float(ratio[0]), float(ratio[1]), 256.0 / 224.0, bool(device_resample))
        pin = torch.cuda.is_available() if pin is None else pin
        self.batch_size, self.depth, self.image_size = int(batch_size), depth, int(image_size)
        self.device_resample = bool(device_resample)
        if self.device_resample:          # one staging arena per slot, sized for the largest record of these shards
            self._img = [torch.empty((self._L.stage_capacity(),), dtype=torch.uint8, pin_memory=pin) for _ in range(depth)]
        else:
            self._img = [torch.empty((batch_size, 3, image_size, image_size), dtype=torch.uint8, pin_memory=pin) for _ in range(depth)]
        self._tgt = [torch.empty((batch_size,), dtype=torch.int64, pin_memory=pin) for _ in range(depth)]
        self._ids = [torch.empty((batch_size,), dtype=torch.int64) for _ in range(depth)] if with_ids else []
        self._L.set_buffers([t.data_ptr() for t in self._img], [t.data_ptr() for t in self._tgt], [t.data_ptr() for t in self._ids])
        self.epoch = 0
        self.sampler = _Sampler(self)
        self.last_ids: Optional[torch.Tensor] = None
        self._pending: deque = deque()           # [event or None, age] of batches handed out and not yet released

    def __len__(self) -> int:
        return int(self._L.num_batches())

    @property
    def num_records(self) -> int:
        return int(self._L.size())

    @property
    def staging_bytes(self) -> int:
        """Pinned bytes of one ring slot's image buffer (the staging arena with ``device_resample``)."""
        return self._img[0].numel()

    def batch_copied(self, event) -> None:
        """The consumer enqueued its copy of the batch it received last; ``event`` completes when that copy is done."""
        if self._pending:
            self._pending[-1][0] = event

    def _reap(self, need_room: bool) -> None:
        for e in self._pending:
            e[1] += 1
        while self._pending:
            ev, age = self._pending[0]
            if ev is not None:
                if not ev.query():
                    if not (need_room and len(self._pending) >= self.depth - 1):
                        break
                    ev.synchronize()
            elif age < 2 and not (need_room and len(self._pending) >= self.depth - 1):
                break
            self._pending.popleft()
            self._L.release()

    def __iter__(self) -> Iterator[Tuple[torch.Tensor, torch.Tensor]]:
        while self._pending:                      # an abandoned epoch: wait for copies that may still read its slots
            ev = self._pending.popleft()[0]
            if ev is not None:
                ev.synchronize()
        self._L.start_epoch(self.epoch)
        try:
            while True:
                self._reap(need_room=True)
                slot, n = self._L.next()
                if slot < 0:
                    break
                self._pending.append([None, 0])
                if self._ids:
                    self.last_ids = self._ids[slot][:n]
                if self.device_resample:
                    img = StagedBatch(self._img[slot][:self._L.staged_bytes(slot)], n, self.image_size, self.image_size,
                                      self._L.stage_max_rows())
                else:
                    img = self._img[slot][:n]
                yield img, self._tgt[slot][:n]
        finally:
            self._L.stop()

    def close(self) -> None:
        self._L.stop()


def build_shard_loaders(args, batch_size: int, rank: int, world: int):
    """Train/val :class:`ShardLoader` pair for ``args.data`` holding ``train-*.ptds`` / ``val-*.ptds``."""
    train_paths, val_paths = find_shards(args.data, "train"), find_shards(args.data, "val")
    if not train_paths or not val_paths:
        raise FileNotFoundError("no train-*.ptds / val-*.ptds under %r (tools/make_shards.py writes them)" % (args.data,))
    seed = args.seed or 0
    workers = max(1, args.workers)
    # The GPU resample gives the same bits as the host one, so it is used whenever the run is on a GPU;
    # PTD_DEVICE_RESAMPLE=0 keeps the resample on the host threads (for A/B measurements).
    on_gpu = (getattr(args, "device", None) or "cuda").startswith("cuda") and torch.cuda.is_available()
    dev = on_gpu and os.environ.get("PTD_DEVICE_RESAMPLE", "1") != "0"
    # a captured step replays one batch shape: under --cuda-graph the ragged last training batch is dropped (validation is eager)
    drop = bool(getattr(args, "cuda_graph", False))
    train = ShardLoader(train_paths, batch_size, args.image_size, train=True, seed=seed, rank=rank, world=world, workers=workers,
                        drop_last=drop, device_resample=dev)
    if drop and len(train) == 0:          # fewer samples than one batch: keep them
        train = ShardLoader(train_paths, batch_size, args.image_size, train=True, seed=seed, rank=rank, world=world, workers=workers,
                            device_resample=dev)
    val = ShardLoader(val_paths, batch_size, args.image_size, train=False, seed=seed, rank=rank, world=world, workers=workers,
                      device_resample=dev)
    if dev and rank == 0 and not getattr(args, "quiet", False):
        print("=> shard loader: resampling on the GPU (%d MB pinned staging per train slot)" % (train.staging_bytes >> 20))
    return train, val, train.sampler, val.sampler
