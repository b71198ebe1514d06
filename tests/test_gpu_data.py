"""Resampling shard batches on the GPU (csrc/resample.cu) against the host resample of the native loader: the kernel
output, the prefetcher output and an entrypoint run on shards."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from pytorch_distributed_b200.utils import shards
from pytorch_distributed_b200.utils.data import IMAGENET_MEAN, IMAGENET_STD, DataPrefetcher

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu
# mostly --max-side 256 records, plus 1x1, 1xN, Nx1, odd square, extreme aspect, smaller than the output, and a large
# record whose bands read more source rows than one pass of shared memory holds
SHAPES = ((256, 341),) * 6 + ((341, 256), (1, 1), (1, 37), (29, 1), (33, 33), (16, 400), (100, 120), (700, 900))


def C():
    from pytorch_distributed_b200 import _ext
    return _ext.lib()


def _write(d, split, n, seed):
    rng = np.random.default_rng(seed)
    path = os.path.join(str(d), "%s-00000.ptds" % split)
    with shards.ShardWriter(path, n) as w:
        for i in range(n):
            h, wd = SHAPES[i % len(SHAPES)]
            base = rng.integers(0, 256, (h // 4 + 1, wd // 4 + 1, 3), dtype=np.uint8)    # blocky noise: smooth and sharp edges
            img = np.repeat(np.repeat(base, 4, 0), 4, 1)[:h, :wd] ^ rng.integers(0, 8, (h, wd, 3), dtype=np.uint8)
            w.add(img, i % 10)
    return [path]


def _ab():
    a = torch.tensor([1.0 / (255.0 * s) for s in IMAGENET_STD], device="cuda")
    b = torch.tensor([-m / s for m, s in zip(IMAGENET_MEAN, IMAGENET_STD)], device="cuda")
    return a, b


@pytest.mark.parametrize("train", [True, False])
def test_device_resample_equals_host_resample(tmp_path, train):
    paths = _write(tmp_path, "train", 150, 0)
    kw = dict(train=train, seed=9, workers=4, depth=3, with_ids=True)
    host = shards.ShardLoader(paths, 64, 224, **kw)
    dev = shards.ShardLoader(paths, 64, 224, device_resample=True, **kw)
    a, b = _ab()
    batches = 0
    for epoch in range(2):
        host.sampler.set_epoch(epoch)
        dev.sampler.set_epoch(epoch)
        for (x, y), (s, t) in zip(host, dev):
            assert torch.equal(y, t) and torch.equal(host.last_ids, dev.last_ids)
            xg, sg = x.cuda(), s.data.cuda()
            for code, dtype in ((0, torch.float32), (1, torch.bfloat16), (2, torch.float16)):
                for cl in (False, True):
                    ref = C().normalize_nhwc(xg, a, b, code, cl)
                    got = C().resample_normalize(sg, s.n, 224, 224, s.max_rows, a, b, code, cl)
                    assert got.dtype == dtype and got.shape == ref.shape and got.stride() == ref.stride()
                    assert torch.equal(got, ref), (epoch, batches, dtype, cl, (got.float() - ref.float()).abs().max().item())
            batches += 1
    assert batches == 2 * 3                        # 150 = 64 + 64 + 22: the ragged last batch included


def test_prefetcher_over_device_loader_equals_host_loader(tmp_path):
    paths = _write(tmp_path, "train", 200, 1)
    outs, ids = [], []
    for device_resample in (False, True):
        ld = shards.ShardLoader(paths, 32, 96, train=True, seed=2, workers=3, depth=3, with_ids=True, device_resample=device_resample)
        pf = DataPrefetcher(ld, "cuda", dtype=torch.bfloat16, channels_last=True, normalize="imagenet255")
        got, seen = [], []
        for epoch in range(2):
            ld.sampler.set_epoch(epoch)
            for x, y in pf:
                got.append((x.clone(), y.clone()))
                seen.append(ld.last_ids.tolist())
        torch.cuda.synchronize()
        outs.append(got)
        ids.append(seen)
    assert ids[0] == ids[1] and len(outs[0]) == len(outs[1]) == 2 * 7
    for (x0, y0), (x1, y1) in zip(*outs):
        assert torch.equal(y0, y1) and torch.equal(x0, x1)
        assert x1.is_contiguous(memory_format=torch.channels_last) and x1.dtype == torch.bfloat16


def _run(cmd, env_extra=None):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="0", **(env_extra or {}))
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "MASTER_ADDR", "MASTER_PORT"):
        env.pop(k, None)
    p = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-3000:] + "\n" + p.stderr[-5000:]
    return p.stdout


def test_entrypoints_train_from_shards_on_the_gpu(tmp_path):
    data = tmp_path / "shards"
    data.mkdir()
    _write(data, "train", 160, 2)
    _write(data, "val", 70, 3)
    common = ["--data", str(data), "-a", "resnet18", "-b", "32", "--epochs", "1", "--image-size", "64", "--num-classes", "10", "-j", "2",
              "-p", "1", "--lr", "0.01", "--checkpoint-dir", str(tmp_path)]
    out = _run([sys.executable, os.path.join(ROOT, "distributed.py")] + common + ["--cuda-graph"])
    assert "=> shard loader: resampling on the GPU" in out
    assert "Epoch: [0][4/5]" in out and " * Acc@1" in out          # 160 // 32 training steps, then validation
    out = _run([sys.executable, os.path.join(ROOT, "dataparallel.py")] + common + ["--gpus", "0", "--evaluate"])
    assert "=> shard loader: resampling on the GPU" in out and " * Acc@1" in out
    out = _run([sys.executable, os.path.join(ROOT, "distributed.py")] + common + ["--evaluate"], {"PTD_DEVICE_RESAMPLE": "0"})
    assert "resampling on the GPU" not in out and " * Acc@1" in out
