"""AutoAugment on the GPU (the two-op rows of csrc/augment.cu) against the CPU path (torchvision's functional ops per sample,
``BatchAugment.reference_apply``): every op, bin and sign in both slots; 32-column rows against 16-column rows; every
sub-policy's chain against the CPU reference applied to the kernel's own first stage; dtypes, layouts and erase boxes;
run-to-run bits; bad tables; the prefetcher with the device and the host resample; entrypoint runs."""
import json
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_gpu_augment as G  # noqa: E402

from pytorch_distributed_b200.ops import augment as A  # noqa: E402
from pytorch_distributed_b200.ops.augment import BatchAugment  # noqa: E402
from pytorch_distributed_b200.utils import shards  # noqa: E402
from pytorch_distributed_b200.utils.data import DataPrefetcher  # noqa: E402

pytestmark = pytest.mark.gpu
NAMES = A.chain_names()
AA_OPS = tuple(A._aa_policy("imagenet")._AUGMENTATION_SPACE.keys())     # the 14 ops AutoAugment's policies draw from
EXACT = G.EXACT | {"Invert"}
GEOMETRIC = G.GEOMETRIC
# the geometric ops' arithmetic is the one-op kernel's (test_gpu_augment.py), but AutoAugment's round shear magnitudes (0.1,
# 0.2, 0.3, ...) put many bilinear results exactly on a .5, where the last bit of torch's float32 grid GEMM decides the
# rounding.  Measured on these images: ShearX up to 1.22e-3 of the pixels at 33x47 (2.0e-4 at 224^2), each within +-1
GEO_FRACTION = 2.5e-3


def _row(slot_a=None, slot_b=None, H=224, W=224):
    """a two-op row; each slot (name, signed magnitude) or None for Identity"""
    r = np.zeros(A.AUG_CHAIN_PRM, dtype=np.float32)
    r[12] = r[A.COL_B + 7] = NAMES.index("Identity")
    for col, ref, e in ((0, 12, slot_a), (A.COL_B, A.COL_B + 7, slot_b)):
        if e is not None:
            code = A.op_code(e[0], e[1], H, W)
            r[col:col + len(code)] = code
            r[ref], r[ref + 1] = NAMES.index(e[0]), e[1]
    return r


def _mags(name, H, W):
    """every (bin, sign) magnitude of op ``name`` in AutoAugment's table"""
    return [A.aa_magnitude("imagenet", name, b, neg, H, W) for b in range(A.AA_NUM_BINS) for neg in (False, True)]


def _check(name, got, want, tag):
    d = (got - want).abs()
    frac, worst = float((d > 0).float().mean()), float(d.max())
    path = os.environ.get("PTD_AUG_STATS")
    if path and frac:
        with open(path, "a") as f:
            f.write(json.dumps({"case": tag, "op": name, "fraction": frac, "worst": worst}) + "\n")
    if name in EXACT:
        assert torch.equal(got, want), (name, frac, worst)
    else:
        assert name in GEOMETRIC and worst <= 1.0 and frac <= GEO_FRACTION, (name, frac, worst)


def _ones():
    return torch.ones(3, device="cuda"), torch.zeros(3, device="cuda")


@pytest.mark.parametrize("H,W", G.SIZES, ids=["%dx%d" % s for s in G.SIZES])
def test_every_op_in_both_slots_against_torchvision(H, W):
    imgs = G.images(H, W, seed=H * W + 1)
    n_img = imgs.size(0)
    k = 2 * A.AA_NUM_BINS
    src = imgs.repeat_interleave(k, 0).contiguous()
    a, b = _ones()
    for name in AA_OPS:
        mags = _mags(name, H, W) * n_img
        for slot in ("a", "b"):
            rows = [_row((name, m), None, H, W) if slot == "a" else _row(None, (name, m), H, W) for m in mags]
            prm = torch.from_numpy(np.stack(rows))
            got = G.C().augment_normalize(src.cuda(), prm.cuda(), a, b, 0, False).cpu()
            want = BatchAugment.reference_apply(src, prm, a.cpu(), b.cpu(), torch.float32, False)
            _check(name, got, want, "slot %s %dx%d" % (slot, H, W))
        if name != "Invert":            # op A with op B Identity gives the bits of the 16-column row of op A
            prm32 = torch.from_numpy(np.stack([_row((name, m), None, H, W) for m in mags]))
            prm16 = prm32[:, :A.AUG_PRM].contiguous()
            assert torch.equal(G.C().augment_normalize(src.cuda(), prm16.cuda(), a, b, 1, True),
                               G.C().augment_normalize(src.cuda(), prm32.cuda(), a, b, 1, True)), name


@pytest.mark.parametrize("policy", A.AUTOAUGMENT_POLICIES)
@pytest.mark.parametrize("H,W", [(224, 224), (33, 47)], ids=["224", "33x47"])
def test_every_sub_policy_chain_decomposed(policy, H, W):
    """the chain equals op B's CPU reference applied to the kernel's own stage 1 (op A alone, exact uint8 values in fp32)"""
    imgs = G.images(H, W, seed=7)
    src = imgs.repeat_interleave(4, 0).contiguous()             # x the four sign patterns
    n = src.size(0)
    a, b = _ones()
    table = A.chain_table(policy, H, W)
    for i, sub in enumerate(A.sub_policies(policy)):
        full = torch.from_numpy(table[[16 * i + 12 + (s & 3) for s in range(n)]])    # both entries applied
        stage1 = full.clone()
        stage1[:, A.COL_B:] = 0
        stage1[:, A.COL_B + 7] = NAMES.index("Identity")
        x1 = G.C().augment_normalize(src.cuda(), stage1.cuda(), a, b, 0, False).cpu()
        assert torch.equal(x1, x1.round().clamp(0, 255))
        only_b = full.clone()
        only_b[:, :7] = 0
        only_b[:, 12:14] = torch.tensor([NAMES.index("Identity"), 0.0])
        got = G.C().augment_normalize(src.cuda(), full.cuda(), a, b, 0, False).cpu()
        want = BatchAugment.reference_apply(x1.to(torch.uint8), only_b, a.cpu(), b.cpu(), torch.float32, False)
        name_a, name_b = sub[0][0], sub[1][0]
        _check(name_b, got, want, "%s[%d] %dx%d" % (policy, i, H, W))
        if name_a in EXACT and name_b in EXACT:
            assert torch.equal(got, BatchAugment.reference_apply(src, full, a.cpu(), b.cpu(), torch.float32, False)), sub


@pytest.mark.parametrize("H,W", [(224, 224), (33, 47)], ids=["224", "33x47"])
def test_dtypes_layouts_skipped_rows_and_erase(H, W):
    src = G.images(H, W).repeat(4, 1, 1, 1).contiguous().cuda()
    n = src.size(0)
    a, b = G._ab()
    skipped = torch.from_numpy(np.stack([_row(None, None, H, W)] * n))
    mixed = torch.from_numpy(A.chain_table("imagenet", H, W)[[(37 * s) % 400 for s in range(n)]])
    rng = np.random.default_rng(5)
    for s in range(n):
        box = A.erase_params(rng, H, W)
        if box is not None and s % 3:
            mixed[s, 7] = 1
            mixed[s, 8:12] = torch.tensor(box, dtype=torch.float32)
    exact = [s for s in range(n) if all(NAMES[int(mixed[s, c])] in EXACT for c in (12, A.COL_B + 7))]
    assert int(mixed[:, 7].sum()) >= n // 2 and len(exact) >= n // 2
    for code, dtype in ((0, torch.float32), (1, torch.bfloat16), (2, torch.float16)):
        for cl in (False, True):
            ref = G.C().normalize_nhwc(src, a, b, code, cl)
            got = G.C().augment_normalize(src, skipped.cuda(), a, b, code, cl)
            assert got.dtype == ref.dtype and got.stride() == ref.stride() and torch.equal(got, ref)
            got = G.C().augment_normalize(src, mixed.cuda(), a, b, code, cl)
            want = BatchAugment.reference_apply(src.cpu(), mixed, a.cpu(), b.cpu(), dtype, cl)
            assert got.stride() == want.stride()
            assert torch.equal(got.cpu()[exact], want[exact])
            for s in range(n):
                if mixed[s, 7]:
                    i, j, h, w = (int(v) for v in mixed[s, 8:12])
                    assert torch.equal(got[s, :, i:i + h, j:j + w].float().cpu(), torch.zeros(3, h, w))


def test_identical_bits_run_to_run():
    src = G.images(224, 224).repeat(8, 1, 1, 1).contiguous().cuda()
    a, b = G._ab()
    for policy in A.AUTOAUGMENT_POLICIES:
        aug = BatchAugment(policy, 0.5, seed=5)
        for _ in range(2):
            prm = aug.draw(src.size(0), 224, 224).cuda()
            assert torch.equal(G.C().augment_normalize(src, prm, a, b, 1, True), G.C().augment_normalize(src, prm, a, b, 1, True))


def test_bad_tables_raise():
    src = G.images(32, 32).cuda()
    a, b = G._ab()
    for bad in (torch.zeros(4, 24, device="cuda"), torch.zeros(4, 33, device="cuda"), torch.zeros(4, A.AUG_CHAIN_PRM),
                torch.zeros(4, A.AUG_CHAIN_PRM, device="cuda", dtype=torch.float64), torch.zeros(3, A.AUG_CHAIN_PRM, device="cuda")):
        with pytest.raises(RuntimeError):
            G.C().augment_normalize(src, bad, a, b, 0, False)
    big = torch.zeros(1, 3, 257, 257, dtype=torch.uint8, device="cuda")
    with pytest.raises(RuntimeError):
        G.C().augment_normalize(big, torch.zeros(1, A.AUG_CHAIN_PRM, device="cuda"), a, b, 0, False)
    assert G.C().AUG_CHAIN_PRM == A.AUG_CHAIN_PRM


def test_largest_image_chains_statistics_ops():
    """at AUG_MAX_PIXELS, op B's statistic over op A's output still matches torchvision"""
    H, W = 241, 273                                             # 65,793 pixels
    src = G.images(H, W, seed=3)[:2].contiguous()
    a, b = _ones()
    prm = torch.from_numpy(np.stack([_row(("Invert", 0.0), ("Equalize", 0.0), H, W), _row(("Solarize", 0.4), ("AutoContrast", 0.0), H, W)]))
    got = G.C().augment_normalize(src.cuda(), prm.cuda(), a, b, 0, False).cpu()
    assert torch.equal(got, BatchAugment.reference_apply(src, prm, a.cpu(), b.cpu(), torch.float32, False))


def test_prefetcher_device_resample_equals_host_resample(tmp_path):
    paths = G._write(tmp_path, 150, 0)
    kw = dict(train=True, seed=9, workers=4, depth=3)
    host = shards.ShardLoader(paths, 64, 224, **kw)
    dev = shards.ShardLoader(paths, 64, 224, device_resample=True, **kw)
    aug_h, aug_d = BatchAugment("imagenet", 0.5, seed=11), BatchAugment("imagenet", 0.5, seed=11)
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


FLAGS = ["--auto-augment", "imagenet", "--random-erase", "0.2"]


@pytest.mark.parametrize("data", ["synthetic", "shards"])
@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_entrypoint_trains_with_autoaugment(tmp_path, data, graph):
    args = ["-a", "resnet50", "-b", "32", "--steps-per-epoch", "3", "--val-steps", "1", "--epochs", "1", "--image-size", "96",
            "-p", "1", "--checkpoint-dir", str(tmp_path), "--log-jsonl", str(tmp_path / "log.jsonl"), "--mixup-alpha", "0.2"] + FLAGS
    if data == "synthetic":
        args.append("--synthetic")
    else:
        d = tmp_path / "shards"
        d.mkdir()
        G._write(d, 80, 1)
        os.rename(d / "train-00000.ptds", d / "val-00000.ptds")
        G._write(d, 80, 2)
        args += ["--data", str(d)]
    if graph:
        args.append("--cuda-graph")
    port = 29951 + 2 * (data == "shards") + graph
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "1", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(G.ROOT, "distributed.py")] + args
    G._run(cmd, tmp_path)


@pytest.mark.multigpu
def test_ddp_world2_runs(tmp_path):
    args = ["-a", "resnet50", "-b", "32", "--synthetic", "--steps-per-epoch", "3", "--val-steps", "1", "--epochs", "1",
            "--image-size", "96", "-p", "1", "--cuda-graph", "--checkpoint-dir", str(tmp_path), "--log-jsonl",
            str(tmp_path / "log.jsonl")] + FLAGS
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29959", os.path.join(G.ROOT, "distributed.py")] + args
    G._run(cmd, tmp_path)
