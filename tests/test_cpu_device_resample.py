"""Staging mode of the native shard loader (``ShardLoader(device_resample=True)``) without a GPU.

A NumPy float32 emulation of the device kernel (csrc/resample.cu: sequential sums over the taps, one rounding per
multiply and per add, +0.5 / clamp / truncate) applied to the staged batches must give the host loader's uint8
batches bit for bit; the arena bound must hold for every crop box; staged slots follow the ring protocol."""
import argparse

import numpy as np
import pytest
import torch

from pytorch_distributed_b200 import _hostext
from pytorch_distributed_b200.utils import shards

DESC = np.dtype([("region", "<i8"), ("taps", "<i8"), ("rw", "<i4"), ("rh", "<i4"), ("kx", "<i4"), ("ky", "<i4")])
# 1x1, 1xN, Nx1, odd square, extreme aspect, smaller than the output (upscaling), the --max-side 256 shape
SHAPES = ((1, 1), (1, 37), (29, 1), (33, 33), (16, 400), (10, 12), (256, 341))
OUT = 32


def _write(tmp_path, n, sizes=SHAPES, split="train", seed=0):
    rng = np.random.default_rng(seed)
    path = str(tmp_path / ("%s-00000.ptds" % split))
    with shards.ShardWriter(path, n) as w:
        for i in range(n):
            h, wd = sizes[i % len(sizes)]
            w.add(rng.integers(0, 256, (h, wd, 3), dtype=np.uint8), i % 7)
    return [path]


def _taps(buf, off, out, k):
    first = np.frombuffer(buf, np.int32, out, off).astype(np.int64)
    count = np.frombuffer(buf, np.int32, out, off + 4 * out)
    w = np.frombuffer(buf, np.float32, out * k, off + 8 * out).reshape(out, k)
    return first, count, w, off + out * (8 + 4 * k)


def emulate(staged):
    """float32 NumPy model of resample_normalize's resample: staged batch -> uint8 [n, 3, out_h, out_w]."""
    assert _hostext.lib().STAGE_DESC_BYTES == DESC.itemsize
    buf = staged.data.numpy().tobytes()
    n, oh, ow = staged.n, staged.out_h, staged.out_w
    out = np.empty((n, 3, oh, ow), np.uint8)
    for i, d in enumerate(np.frombuffer(buf, DESC, n)):
        rw, rh, kx, ky = int(d["rw"]), int(d["rh"]), int(d["kx"]), int(d["ky"])
        region = np.frombuffer(buf, np.uint8, rw * rh * 3, int(d["region"])).reshape(rh, rw, 3).astype(np.float32)
        fx, cx, wx, t = _taps(buf, int(d["taps"]), ow, kx)
        fy, cy, wy, _ = _taps(buf, t, oh, ky)
        assert fx.min() >= 0 and (fx + cx).max() <= rw and fy.min() >= 0 and (fy + cy).max() <= rh
        assert cy.max() <= staged.max_rows
        rows = np.zeros((rh, ow, 3), np.float32)
        for k in range(kx):        # a masked tap adds +0.0, which leaves the non-negative sum unchanged
            wk = np.where(k < cx, wx[:, k], np.float32(0))
            rows = rows + wk[None, :, None] * region[:, np.minimum(fx + k, rw - 1), :]
        acc = np.zeros((oh, ow, 3), np.float32)
        for k in range(ky):
            wk = np.where(k < cy, wy[:, k], np.float32(0))
            acc = acc + wk[:, None, None] * rows[np.minimum(fy + k, rh - 1)]
        assert acc.dtype == np.float32
        out[i] = np.minimum(np.float32(255), np.maximum(np.float32(0), acc + np.float32(0.5))).astype(np.uint8).transpose(2, 0, 1)
    return out


@pytest.mark.parametrize("train,workers,rank,world", [(True, 1, 0, 1), (True, 5, 1, 2), (False, 1, 1, 2), (False, 5, 0, 1)])
def test_emulated_device_resample_matches_host(tmp_path, train, workers, rank, world):
    paths = _write(tmp_path, 21)
    kw = dict(train=train, seed=4, rank=rank, world=world, workers=workers, depth=3, pin=False, with_ids=True)
    host = shards.ShardLoader(paths, 4, OUT, **kw)
    dev = shards.ShardLoader(paths, 4, OUT, device_resample=True, **kw)
    for epoch in range(3):
        host.sampler.set_epoch(epoch)
        dev.sampler.set_epoch(epoch)
        sizes = []
        for (x, y), (s, t) in zip(host, dev):
            assert isinstance(s, shards.StagedBatch) and s.shape == tuple(x.shape)
            assert torch.equal(y, t) and torch.equal(host.last_ids, dev.last_ids)
            assert s.data.numel() <= dev.staging_bytes
            np.testing.assert_array_equal(emulate(s), x.numpy())
            sizes.append(s.n)
        assert len(sizes) == len(dev) and sizes[-1] < 4            # ragged last batch covered


@pytest.mark.parametrize("scale", [(0.08, 1.0), (1.0, 1.0)])
def test_arena_bound_holds_for_every_box(tmp_path, scale):
    paths = _write(tmp_path, len(SHAPES))
    ld = shards.ShardLoader(paths, 8, OUT, train=True, seed=1, workers=1, pin=False, device_resample=True, scale=scale)
    val = shards.ShardLoader(paths, 8, OUT, train=False, workers=1, pin=False, device_resample=True)
    for W, H in [(wd, h) for h, wd in SHAPES] + [(500, 375), (224, 224), (7, 300)]:
        bound = ld._L.stage_bound(W, H)
        assert max(ld._L.stage_size(0, pos, W, H) for pos in range(10000)) <= bound, (W, H)
        assert val._L.stage_size(0, 0, W, H) == val._L.stage_bound(W, H)      # val boxes are a function of the shape
    # 400x16 is outside the aspect range: no try fits and every box is the centred fallback crop (21 x 16)
    assert all(ld._L.crop_params(0, pos, 400, 16)[:4] == [189.0, 0.0, 21.0, 16.0] for pos in range(100))
    table = -(-8 * 32 // 16) * 16
    assert ld.staging_bytes == table + 8 * max(ld._L.stage_bound(wd, h) for h, wd in SHAPES)


def test_held_staged_batch_stays_intact(tmp_path):
    paths = _write(tmp_path, 40)
    ld = shards.ShardLoader(paths, 4, 12, train=False, workers=2, depth=3, pin=False, with_ids=True, device_resample=True)
    held = []
    for x, y in ld:
        held.append((x.data, x.data.clone()))
        if len(held) >= 2:                       # the previous batch must still be intact while the next one is drawn
            assert torch.equal(held[-2][0], held[-2][1])
    assert len(held) == 10


def test_cpu_runs_keep_the_host_resample(tmp_path):
    _write(tmp_path, 6, split="train")
    _write(tmp_path, 6, split="val")
    args = argparse.Namespace(data=str(tmp_path), seed=0, workers=1, image_size=OUT, cuda_graph=False, device="cpu", quiet=True)
    train, val, _, _ = shards.build_shard_loaders(args, 4, 0, 1)
    assert not train.device_resample and not val.device_resample
    from pytorch_distributed_b200.utils.data import DataPrefetcher
    staged = shards.ShardLoader(shards.find_shards(str(tmp_path), "train"), 4, OUT, pin=False, workers=1, device_resample=True)
    with pytest.raises(RuntimeError, match="CUDA prefetcher"):
        list(DataPrefetcher(staged, "cpu", normalize="imagenet255"))
