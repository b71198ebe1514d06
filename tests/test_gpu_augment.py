"""TrivialAugment Wide and random erasing on the GPU (csrc/augment.cu) against the CPU path (torchvision's functional ops per
sample, ``BatchAugment.reference_apply``): every op, bin and sign on noise, gradients and the degenerate images of
AutoContrast and Equalize at several sizes; dtypes and layouts; run-to-run bits; the prefetcher with the device and the host
resample; entrypoint runs."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from pytorch_distributed_b200.ops import augment as A
from pytorch_distributed_b200.ops.augment import BatchAugment
from pytorch_distributed_b200.utils import shards
from pytorch_distributed_b200.utils.data import IMAGENET_MEAN, IMAGENET_STD, DataPrefetcher

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu
SIZES = [(224, 224), (176, 176), (33, 47), (240, 256)]      # 240 x 256 > 224^2 and below AUG_MAX_PIXELS
NAMES = A.op_names()
# bit-equal: the point ops, and Color, Contrast and Sharpness too, whose grayscale, mean and blend roundings the kernel
# writes out in torchvision's order (FMA where torch's CPU add-with-alpha uses one) and whose blur is exact in integers
EXACT = {"Identity", "Brightness", "Posterize", "Solarize", "AutoContrast", "Equalize", "Color", "Contrast", "Sharpness"}
# the geometric ops: torch's CPU grid is a float32 GEMM (base grid x rescaled theta) whose summation order and FMA use the
# kernel cannot know; a different last bit of a coordinate moves a bilinear result across a .5 rounding boundary now and
# then.  Measured on these images: at most 3.2e-5 of the pixels, each within +-1; the bound is 2e-4, each within +-1.
GEO_FRACTION = 2e-4
GEOMETRIC = {"ShearX", "ShearY", "TranslateX", "TranslateY", "Rotate"}


def C():
    from pytorch_distributed_b200 import _ext
    return _ext.lib()


def images(H, W, seed=0):
    """blocky noise (test_gpu_data._write), a smooth gradient, a constant image and a two-level image"""
    rng = np.random.default_rng(seed)
    base = rng.integers(0, 256, (3, H // 4 + 1, W // 4 + 1), dtype=np.uint8)
    noise = np.repeat(np.repeat(base, 4, 1), 4, 2)[:, :H, :W] ^ rng.integers(0, 8, (3, H, W), dtype=np.uint8)
    yy, xx = np.meshgrid(np.linspace(0, 1, H), np.linspace(0, 1, W), indexing="ij")
    grad = np.stack([255 * xx, 255 * yy, 127 * (xx + yy)]).round().astype(np.uint8)
    const = np.full((3, H, W), 91, dtype=np.uint8)
    two = np.where(rng.random((H, W)) < 0.3, 200, 17).astype(np.uint8)[None].repeat(3, 0)
    return torch.from_numpy(np.stack([noise, grad, const, two]))


def table(op, n_img, H, W):
    """every bin and sign of op ``op`` for each of ``n_img`` images: [n_img * 62, AUG_PRM]"""
    rows = []
    for k in range(n_img):
        for b in range(A.NUM_BINS):
            for neg in (False, True):
                r = np.zeros(A.AUG_PRM, dtype=np.float32)
                code = A.encode(op, b, neg, H, W)
                r[:len(code)] = code
                r[12], r[13] = op, A.magnitude(op, b, neg, H, W)
                rows.append(r)
    return torch.from_numpy(np.stack(rows))


def _ones():
    return torch.ones(3, device="cuda"), torch.zeros(3, device="cuda")


@pytest.mark.parametrize("H,W", SIZES, ids=["%dx%d" % s for s in SIZES])
def test_every_op_bin_and_sign_against_torchvision(H, W):
    imgs = images(H, W, seed=H * W)
    n_img = imgs.size(0)
    src = imgs.repeat_interleave(2 * A.NUM_BINS, 0).contiguous()
    a, b = _ones()
    stats = {}
    for op, name in enumerate(NAMES):
        prm = table(op, n_img, H, W)
        got = C().augment_normalize(src.cuda(), prm.cuda(), a, b, 0, False).cpu()
        want = BatchAugment.reference_apply(src, prm, a.cpu(), b.cpu(), torch.float32, False)
        d = (got - want).abs()
        frac, worst = float((d > 0).float().mean()), float(d.max())
        stats[name] = (frac, worst)
        if name in EXACT:
            assert torch.equal(got, want), (name, frac, worst)
        else:
            assert name in GEOMETRIC and worst <= 1.0 and frac <= GEO_FRACTION, (name, frac, worst)
    path = os.environ.get("PTD_AUG_STATS")
    if path:
        with open(path, "a") as f:
            f.write(json.dumps({"size": [H, W], "mismatch": stats}) + "\n")


def _ab():
    a = torch.tensor([1.0 / (255.0 * s) for s in IMAGENET_STD], device="cuda")
    b = torch.tensor([-m / s for m, s in zip(IMAGENET_MEAN, IMAGENET_STD)], device="cuda")
    return a, b


@pytest.mark.parametrize("H,W", [(224, 224), (33, 47)], ids=["224", "33x47"])
def test_dtypes_layouts_identity_and_erase(H, W):
    src = images(H, W).repeat(4, 1, 1, 1).contiguous().cuda()
    n = src.size(0)
    a, b = _ab()
    ident = torch.zeros(n, A.AUG_PRM)
    ident[:, 12] = NAMES.index("Identity")
    erased = ident.clone()
    rng = np.random.default_rng(3)
    for s in range(n):
        box = A.erase_params(rng, H, W)
        if box is not None:
            erased[s, 7] = 1
            erased[s, 8:12] = torch.tensor(box, dtype=torch.float32)
    assert int(erased[:, 7].sum()) >= n // 2
    mixed = table(NAMES.index("Equalize"), 1, H, W)[:n]
    mixed[:, 7:12] = erased[:, 7:12]
    for code, dtype in ((0, torch.float32), (1, torch.bfloat16), (2, torch.float16)):
        for cl in (False, True):
            ref = C().normalize_nhwc(src, a, b, code, cl)
            got = C().augment_normalize(src, ident.cuda(), a, b, code, cl)
            assert got.dtype == ref.dtype and got.shape == ref.shape and got.stride() == ref.stride()
            assert torch.equal(got, ref)
            got = C().augment_normalize(src, erased.cuda(), a, b, code, cl)
            assert got.stride() == ref.stride()
            mask = torch.zeros(n, 1, H, W, dtype=torch.bool, device="cuda")
            for s in range(n):
                if erased[s, 7]:
                    i, j, h, w = (int(v) for v in erased[s, 8:12])
                    mask[s, :, i:i + h, j:j + w] = True
            mask = mask.expand_as(got)
            assert torch.equal(got[mask], torch.zeros_like(got[mask]))
            assert torch.equal(got[~mask], ref[~mask])
            want = BatchAugment.reference_apply(src.cpu(), mixed, a.cpu(), b.cpu(), dtype, cl)
            got = C().augment_normalize(src, mixed.cuda(), a, b, code, cl)
            assert got.stride() == want.stride() and torch.equal(got.cpu(), want)


def test_identical_bits_run_to_run():
    src = images(224, 224).repeat(8, 1, 1, 1).contiguous().cuda()
    aug = BatchAugment("ta_wide", 0.5, seed=5)
    a, b = _ab()
    for _ in range(3):
        prm = aug.draw(src.size(0), 224, 224).cuda()
        x = C().augment_normalize(src, prm, a, b, 1, True)
        y = C().augment_normalize(src, prm, a, b, 1, True)
        assert torch.equal(x, y)


def test_bad_arguments_raise():
    src = images(32, 32).cuda()
    a, b = _ab()
    with pytest.raises(RuntimeError):
        C().augment_normalize(src, torch.zeros(4, 8, device="cuda"), a, b, 0, False)
    with pytest.raises(RuntimeError):
        C().augment_normalize(src, torch.zeros(4, A.AUG_PRM), a, b, 0, False)
    with pytest.raises(RuntimeError):
        C().augment_normalize(src, torch.zeros(4, A.AUG_PRM, device="cuda", dtype=torch.float64), a, b, 0, False)
    big = torch.zeros(1, 3, 257, 257, dtype=torch.uint8, device="cuda")
    with pytest.raises(RuntimeError):
        C().augment_normalize(big, torch.zeros(1, A.AUG_PRM, device="cuda"), a, b, 0, False)


def _write(d, n, seed):
    rng = np.random.default_rng(seed)
    path = os.path.join(str(d), "train-00000.ptds")
    shapes = ((256, 341), (341, 256), (33, 33), (100, 120), (700, 900))
    with shards.ShardWriter(path, n) as w:
        for i in range(n):
            h, wd = shapes[i % len(shapes)]
            base = rng.integers(0, 256, (h // 4 + 1, wd // 4 + 1, 3), dtype=np.uint8)
            img = np.repeat(np.repeat(base, 4, 0), 4, 1)[:h, :wd] ^ rng.integers(0, 8, (h, wd, 3), dtype=np.uint8)
            w.add(img, i % 10)
    return [path]


def test_prefetcher_device_resample_equals_host_resample(tmp_path):
    paths = _write(tmp_path, 150, 0)                     # 150 = 2 x 64 + a ragged 22
    kw = dict(train=True, seed=9, workers=4, depth=3)
    host = shards.ShardLoader(paths, 64, 224, **kw)
    dev = shards.ShardLoader(paths, 64, 224, device_resample=True, **kw)
    aug_h, aug_d = BatchAugment("ta_wide", 0.5, seed=11), BatchAugment("ta_wide", 0.5, seed=11)
    sizes = []
    for epoch in range(2):
        for ld, ag in ((host, aug_h), (dev, aug_d)):
            ld.sampler.set_epoch(epoch)
            ag.set_epoch(epoch)
        ph = DataPrefetcher(host, "cuda", torch.bfloat16, True, normalize="imagenet255", augment=aug_h)
        pd = DataPrefetcher(dev, "cuda", torch.bfloat16, True, normalize="imagenet255", augment=aug_d)
        for (x, y), (s, t) in zip(ph, pd):
            assert torch.equal(y, t) and torch.equal(x, s)
            sizes.append(x.size(0))
    assert sizes == [64, 64, 22] * 2


# ------------------------------------------------------------------------------------------------ entrypoints
FLAGS = ["--auto-augment", "ta_wide", "--random-erase", "0.25"]


def _run(cmd, tmp_path):
    e = dict(os.environ, PYTHONPATH=ROOT)
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "MASTER_ADDR", "MASTER_PORT"):
        e.pop(k, None)
    p = subprocess.run(cmd, env=e, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-3000:] + "\n" + p.stderr[-3000:]
    with open(tmp_path / "log.jsonl") as f:
        recs = [json.loads(l) for l in f if l.strip()]
    assert {"train", "val"} <= {r["phase"] for r in recs}
    assert all(np.isfinite(r["loss"]) and r["loss"] > 0 for r in recs), recs
    return p.stdout


@pytest.mark.parametrize("data", ["synthetic", "shards"])
@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_entrypoint_trains_with_both_flags(tmp_path, data, graph):
    args = ["-a", "resnet50", "-b", "32", "--steps-per-epoch", "3", "--val-steps", "1", "--epochs", "1", "--image-size", "96",
            "-p", "1", "--checkpoint-dir", str(tmp_path), "--log-jsonl", str(tmp_path / "log.jsonl"), "--mixup-alpha", "0.2"] + FLAGS
    if data == "synthetic":
        args.append("--synthetic")
    else:
        d = tmp_path / "shards"
        d.mkdir()
        _write(d, 80, 1)
        os.rename(d / "train-00000.ptds", d / "val-00000.ptds")
        _write(d, 80, 2)
        args += ["--data", str(d)]
    if graph:
        args.append("--cuda-graph")
    port = 29851 + 2 * (data == "shards") + graph
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "1", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "distributed.py")] + args
    _run(cmd, tmp_path)


@pytest.mark.multigpu
def test_ddp_world2_runs(tmp_path):
    args = ["-a", "resnet50", "-b", "32", "--synthetic", "--steps-per-epoch", "3", "--val-steps", "1", "--epochs", "1",
            "--image-size", "96", "-p", "1", "--cuda-graph", "--checkpoint-dir", str(tmp_path), "--log-jsonl",
            str(tmp_path / "log.jsonl")] + FLAGS
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29859", os.path.join(ROOT, "distributed.py")] + args
    _run(cmd, tmp_path)
