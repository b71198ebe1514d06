"""TrivialAugment Wide and random erasing on the CPU: the CLI, the draws against torchvision's distributions, the op and
magnitude mapping against ``TrivialAugmentWide._apply_image_or_video_transform``, the ImageFolder transform list, a gloo
world-2 run and a resume."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
from scipy import stats

from pytorch_distributed_b200 import cli
from pytorch_distributed_b200.ops import augment as A
from pytorch_distributed_b200.ops.augment import BatchAugment
from pytorch_distributed_b200.utils import data as D

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FLAGS = ["--auto-augment", "ta_wide", "--random-erase", "0.25"]


def test_cli_defaults_bounds_and_policies():
    a = cli.parse_args("distributed", [])
    assert a.auto_augment is None and a.random_erase == 0.0
    a = cli.parse_args("apex_distributed", FLAGS)
    assert a.auto_augment == "ta_wide" and a.random_erase == 0.25
    for p in ("0", "1", "0.1"):
        assert cli.parse_args("distributed", ["--random-erase", p]).random_erase == float(p)
    for bad in (["--random-erase", "-0.01"], ["--random-erase", "1.5"], ["--auto-augment", "ra"], ["--auto-augment", "ta"]):
        with pytest.raises(SystemExit):
            cli.parse_args("distributed", bad)
    with pytest.raises(ValueError):
        BatchAugment("augmix")


def _draws(aug, batches=40, n=256, H=224, W=224):
    return np.concatenate([aug.draw(n, H, W).numpy().copy() for _ in range(batches)])


def test_op_bin_sign_and_erase_rate_distributions():
    aug = BatchAugment("ta_wide", 0.3, seed=1)
    t = _draws(aug)
    ops = t[:, 12].astype(int)
    assert stats.chisquare(np.bincount(ops, minlength=14)).pvalue > 1e-3
    # the bin of the ops with a table: recovered from the magnitude
    for name in ("Brightness", "Rotate", "Posterize"):
        op = A.op_names().index(name)
        sel = t[ops == op]
        table = [A.magnitude(op, b, False, 224, 224) for b in range(A.NUM_BINS)]
        bins = []
        for m in np.abs(sel[:, 13]):
            cand = [b for b, v in enumerate(table) if np.float32(v) == np.float32(m)]
            bins.append(cand[0])
        counts = np.bincount(bins, minlength=A.NUM_BINS)
        if name != "Posterize":                     # Posterize's table repeats values
            assert stats.chisquare(counts).pvalue > 1e-3, name
    signed = [A.op_names().index(n) for n in ("ShearX", "Brightness", "Color")]
    m = t[np.isin(ops, signed)][:, 13]
    m = m[m != 0]
    assert stats.binomtest(int((m < 0).sum()), len(m), 0.5).pvalue > 1e-3
    n_erase = int(t[:, 7].sum())
    # a try fails now and then (h or w too large): the box rate is p times the chance that one of 10 tries fits (~1)
    assert stats.binomtest(n_erase, len(t), 0.3).pvalue > 1e-4


def test_erase_box_matches_torchvision_get_params():
    from torchvision.transforms.v2 import RandomErasing
    H, W = 224, 176
    rng = np.random.default_rng(0)
    ours = [A.erase_params(rng, H, W) for _ in range(4000)]
    ours = [b for b in ours if b is not None]
    torch.manual_seed(0)
    re = RandomErasing(p=1.0)
    img = torch.zeros(3, H, W)
    theirs = []
    for _ in range(4000):
        p = re.make_params([img])
        if p["v"] is not None:
            theirs.append((p["i"], p["j"], p["h"], p["w"]))
    oa = np.array(ours, dtype=float)
    ta = np.array(theirs, dtype=float)
    assert stats.ks_2samp(oa[:, 2] * oa[:, 3], ta[:, 2] * ta[:, 3]).pvalue > 1e-3           # area
    assert stats.ks_2samp(oa[:, 2] / oa[:, 3], ta[:, 2] / ta[:, 3]).pvalue > 1e-3           # aspect
    assert stats.ks_2samp(oa[:, 0] / (H - oa[:, 2] + 1), ta[:, 0] / (H - ta[:, 2] + 1)).pvalue > 1e-3
    assert all(i + h <= H and j + w <= W for i, j, h, w in ours)


def test_epoch_replay_and_rank_streams():
    a, b = BatchAugment("ta_wide", 0.5, seed=3), BatchAugment("ta_wide", 0.5, seed=3)
    e0 = _draws(a, 3, 32)
    a.set_epoch(1)
    e1 = _draws(a, 3, 32)
    b.set_epoch(1)
    assert np.array_equal(_draws(b, 3, 32), e1)
    b.set_epoch(0)
    assert np.array_equal(_draws(b, 3, 32), e0)
    assert not np.array_equal(e0, e1)
    r1 = BatchAugment("ta_wide", 0.5, seed=3, rank=1)
    assert not np.array_equal(_draws(r1, 3, 32), e0)


def _noise(H, W, seed=0):
    return torch.from_numpy(np.random.default_rng(seed).integers(0, 256, (3, H, W), dtype=np.uint8))


@pytest.mark.parametrize("H,W", [(32, 32), (20, 27)])
def test_op_and_magnitude_mapping_equals_torchvision(H, W):
    """reference_apply of every (op, bin, sign) is what TrivialAugmentWide applies for that draw"""
    from torchvision.transforms import InterpolationMode
    from torchvision.transforms.v2 import TrivialAugmentWide
    ta = TrivialAugmentWide(interpolation=InterpolationMode.BILINEAR)
    img = _noise(H, W)
    one, zero = torch.ones(3), torch.zeros(3)
    for op, name in enumerate(A.op_names()):
        fn, signed = ta._AUGMENTATION_SPACE[name]
        mags = fn(A.NUM_BINS, H, W)
        for b in range(A.NUM_BINS):
            for neg in (False, True):
                m = 0.0 if mags is None else float(mags[b]) * (-1 if (signed and neg) else 1)
                assert A.magnitude(op, b, neg, H, W) == m
                want = ta._apply_image_or_video_transform(img, name, m, interpolation=ta.interpolation, fill=ta._fill)
                prm = torch.zeros(1, A.AUG_PRM)
                code = A.encode(op, b, neg, H, W)
                prm[0, :len(code)] = torch.tensor(code)
                prm[0, 12], prm[0, 13] = op, A.magnitude(op, b, neg, H, W)
                got = BatchAugment.reference_apply(img[None], prm, one, zero, torch.float32, False)
                assert torch.equal(got[0], want.float()), (name, b, neg)
    with pytest.raises(ValueError):
        A.encode(14, 0, False, H, W)
    with pytest.raises(ValueError):
        A.encode(1, 31, False, H, W)
    with pytest.raises(ValueError):
        BatchAugment("ta_wide").draw(2, 300, 300)


def test_imagefolder_transforms_follow_the_recipe():
    import torchvision.transforms as T
    ns = argparse.Namespace(image_size=224, auto_augment=None, random_erase=0.0)
    assert [type(t) for t in D.train_transforms(ns)] == [T.RandomResizedCrop, T.RandomHorizontalFlip, T.ToTensor, T.Normalize]
    ns = argparse.Namespace(image_size=224, auto_augment="ta_wide", random_erase=0.1)
    ts = D.train_transforms(ns)
    assert [type(t) for t in ts] == [T.RandomResizedCrop, T.RandomHorizontalFlip, T.TrivialAugmentWide, T.ToTensor, T.Normalize,
                                     T.RandomErasing]
    assert ts[2].interpolation == T.InterpolationMode.BILINEAR and ts[-1].p == 0.1 and ts[-1].value == 0


def test_flags_off_leave_the_loaders_unchanged():
    ns = cli.parse_args("distributed", ["--synthetic", "-b", "4", "--image-size", "16", "--steps-per-epoch", "2"])
    assert not D.augmenting(ns)
    tr, va, _, _ = D.build_loaders(ns, 4, distributed=False)
    assert not tr.raw_uint8 and tr.pool[0][0].dtype == torch.float32
    ns = cli.parse_args("distributed", ["--synthetic", "-b", "4", "--image-size", "16", "--steps-per-epoch", "2", "--random-erase", "0.1"])
    tr, va, _, _ = D.build_loaders(ns, 4, distributed=False)
    assert tr.raw_uint8 and tr.pool[0][0].dtype == torch.uint8 and not va.raw_uint8
    from pytorch_distributed_b200 import driver
    assert driver.make_batch_augment(cli.parse_args("distributed", []), torch.device("cpu"), 0) is None


def test_cpu_prefetcher_applies_the_reference():
    ld = D.SyntheticLoader(4, 2, 24, 10, raw_uint8=True, pin=False)
    aug, ref = BatchAugment("ta_wide", 0.5, seed=2), BatchAugment("ta_wide", 0.5, seed=2)
    pf = D.DataPrefetcher(ld, "cpu", torch.float32, False, normalize="imagenet255", augment=aug)
    for (x, _), (raw, _) in zip(pf, ld):
        prm = ref.draw(4, 24, 24)
        assert torch.equal(x, BatchAugment.reference_apply(raw, prm, pf._a, pf._b, torch.float32, False))


def _env(extra=None):
    env = dict(os.environ, OMP_NUM_THREADS="1", PYTHONPATH=ROOT, **(extra or {}))
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "MASTER_ADDR", "MASTER_PORT"):
        env.pop(k, None)
    return env


def _torchrun(n, argv, port, env=None):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(n), "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "distributed.py")] + argv
    p = subprocess.run(cmd, env=_env(env), cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-3000:] + "\n" + p.stderr[-3000:]
    return p.stdout


def _records(path):
    with open(path) as f:
        return [json.loads(l) for l in f if l.strip()]


def _shards(d):
    from pytorch_distributed_b200.utils import shards
    d.mkdir(exist_ok=True)
    rng = np.random.default_rng(0)
    for split, n in (("train", 24), ("val", 8)):
        with shards.ShardWriter(str(d / ("%s-00000.ptds" % split)), n) as w:
            for i in range(n):
                w.add(rng.integers(0, 256, (40 + i, 48, 3), dtype=np.uint8), i % 10)
    return str(d)


def _common(d, log, data):
    d.mkdir(exist_ok=True)
    return ["-a", "resnet18", "-b", "8", "--data", data, "--image-size", "32", "--num-classes", "10", "-p", "1", "--device", "cpu",
            "--checkpoint-dir", str(d), "--quiet", "--seed", "0", "--log-jsonl", str(log), "--steps-per-epoch", "2",
            "--val-steps", "1", "-j", "1"] + FLAGS


def test_distributed_gloo_world2_on_shards(tmp_path):
    log = tmp_path / "log.jsonl"
    out = _torchrun(2, _common(tmp_path / "ck", log, _shards(tmp_path / "data")) + ["--epochs", "1"], 29871)
    assert out.count(" * Acc@1 ") == 2
    recs = _records(log)
    train = [r for r in recs if r["phase"] == "train"]
    assert len(train) == 2 and all(np.isfinite(r["loss"]) and r["loss"] > 0 for r in recs)


def test_resume_at_epoch_boundary_replays_the_draws(tmp_path):
    env = {"PTD_SAVE_OPTIMIZER": "1"}
    data = _shards(tmp_path / "data")
    full, half = tmp_path / "full.jsonl", tmp_path / "half.jsonl"
    _torchrun(1, _common(tmp_path / "full", full, data) + ["--epochs", "2"], 29873, env)
    _torchrun(1, _common(tmp_path / "half", half, data) + ["--epochs", "1"], 29875, env)
    ck = str(tmp_path / "half" / "checkpoint.pth.tar")
    _torchrun(1, _common(tmp_path / "half", half, data) + ["--epochs", "2", "--resume", ck], 29877, env)
    a = [r["loss"] for r in _records(full) if r["phase"] == "train"]
    b = [r["loss"] for r in _records(half) if r["phase"] == "train"]
    assert len(a) == len(b) == 2 and a == b
