"""AutoAugment on the CPU: the CLI, the draws against torchvision's distributions and tables, epoch replay and rank streams,
TrivialAugment Wide's tables unchanged, every sub-policy's encoded row against torchvision's two
``_apply_image_or_video_transform`` calls, the ImageFolder transform list, a CPU prefetcher run, a gloo world-2 run and a
resume."""
import argparse
import hashlib
import os
import sys

import numpy as np
import pytest
import torch
from scipy import stats

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_cpu_augment as T  # noqa: E402

from pytorch_distributed_b200 import cli  # noqa: E402
from pytorch_distributed_b200.ops import augment as A  # noqa: E402
from pytorch_distributed_b200.ops.augment import BatchAugment  # noqa: E402
from pytorch_distributed_b200.utils import data as D  # noqa: E402

FLAGS = ["--auto-augment", "imagenet", "--random-erase", "0.25"]
# sha256 of the TrivialAugment Wide tables below, recorded before AutoAugment was added: its draws and encoding are unchanged
TA_WIDE_SHA256 = "b3204f1b84d5f7351f30f9e2488aa76eb497efc36dab2905046c457a84a28fb2"


def test_cli_accepts_the_three_policies():
    for p in A.AUTOAUGMENT_POLICIES:
        assert cli.parse_args("distributed", ["--auto-augment", p]).auto_augment == p
        assert BatchAugment(p).width == A.AUG_CHAIN_PRM
    assert BatchAugment("ta_wide").width == BatchAugment(None, 0.1).width == A.AUG_PRM
    for bad in ("ra", "ta", "augmix", "IMAGENET"):
        with pytest.raises(SystemExit):
            cli.parse_args("distributed", ["--auto-augment", bad])
        with pytest.raises(ValueError):
            BatchAugment(bad)


def test_ta_wide_tables_unchanged():
    aug = BatchAugment("ta_wide", 0.25, seed=1234, rank=1)
    aug.set_epoch(2)
    h = hashlib.sha256()
    for n, H, W in ((64, 224, 224), (64, 224, 224), (37, 33, 47), (16, 176, 176)):
        t = aug.draw(n, H, W)
        assert t.shape == (n, A.AUG_PRM)
        h.update(t.numpy().tobytes())
    assert h.hexdigest() == TA_WIDE_SHA256


def _find_entry(row, k):
    """(name, magnitude) of entry k (0: op A, 1: op B) of a row, None when not applied"""
    name = A.chain_names()[int(row[12 if k == 0 else A.COL_B + 7])]
    return None if name == "Identity" else (name, float(row[13 if k == 0 else A.COL_B + 8]))


@pytest.mark.parametrize("policy", A.AUTOAUGMENT_POLICIES)
def test_draw_distributions(policy):
    H, W = 224, 160
    aug = BatchAugment(policy, 0.0, seed=1)
    subs = A.sub_policies(policy)
    # which sub-policy a row came from is not stored: recover it by drawing the same stream's sub-policy indices again
    rng = np.random.Generator(np.random.PCG64([aug.seed, 0, 0, A.STREAM_ID]))
    rows, picks = [], []
    for _ in range(40):
        rows.append(aug.draw(256, H, W).numpy().copy())
        picks.append(rng.integers(0, len(subs), 256))
        rng.random((256, 2))
        rng.random((256, 2))
    rows, picks = np.concatenate(rows), np.concatenate(picks)
    assert stats.chisquare(np.bincount(picks, minlength=len(subs))).pvalue > 1e-3
    negs, signed_n = 0, 0
    for i, sub in enumerate(subs):
        sel = rows[picks == i]
        for k, (name, p, idx) in enumerate(sub):
            hits = [_find_entry(r, k) for r in sel]
            applied = [h for h in hits if h is not None]
            if p == 0.0:
                assert not applied, (sub, k)
            elif p < 1.0:
                assert stats.binomtest(len(applied), len(sel), p).pvalue > 1e-4, (policy, i, k)
            else:
                assert len(applied) == len(sel)
            mag = A.aa_magnitude(policy, name, idx, False, H, W)
            fn, signed = A._aa_policy(policy)._AUGMENTATION_SPACE[name]
            table = fn(10, H, W)
            assert mag == (0.0 if table is None else float(table[idx]))
            for got_name, m in applied:
                assert got_name == name and np.float32(abs(m)) == np.float32(mag)
                if signed and mag != 0:
                    signed_n += 1
                    negs += m < 0
    assert stats.binomtest(negs, signed_n, 0.5).pvalue > 1e-3


def test_epoch_replay_and_rank_streams():
    a, b = BatchAugment("cifar10", 0.5, seed=3), BatchAugment("cifar10", 0.5, seed=3)
    e0 = T._draws(a, 3, 32)
    a.set_epoch(1)
    e1 = T._draws(a, 3, 32)
    b.set_epoch(1)
    assert np.array_equal(T._draws(b, 3, 32), e1)
    b.set_epoch(0)
    assert np.array_equal(T._draws(b, 3, 32), e0)
    assert not np.array_equal(e0, e1)
    assert not np.array_equal(T._draws(BatchAugment("cifar10", 0.5, seed=3, rank=1), 3, 32), e0)


@pytest.mark.parametrize("H,W", [(32, 32), (20, 27)])
@pytest.mark.parametrize("policy", A.AUTOAUGMENT_POLICIES)
def test_every_sub_policy_and_sign_equals_torchvision(policy, H, W):
    """reference_apply of each of the 400 encoded rows is what AutoAugment applies for that outcome"""
    pol = A._aa_policy(policy)
    img = T._noise(H, W, seed=H)
    one, zero = torch.ones(3), torch.zeros(3)
    table = A.chain_table(policy, H, W)
    assert table.shape == (400, A.AUG_CHAIN_PRM)
    got = BatchAugment.reference_apply(img[None].expand(400, -1, -1, -1), torch.from_numpy(table), one, zero, torch.float32, False)
    for i, sub in enumerate(A.sub_policies(policy)):
        for applied in range(4):
            for signs in range(4):
                want = img
                for k, (name, _, idx) in enumerate(sub):
                    if applied >> k & 1:
                        fn, signed = pol._AUGMENTATION_SPACE[name]
                        mags = fn(10, H, W)
                        m = 0.0 if mags is None else float(mags[idx])
                        if signed and signs >> k & 1:
                            m *= -1
                        want = pol._apply_image_or_video_transform(want, name, m, interpolation=pol.interpolation, fill=pol._fill)
                assert torch.equal(got[16 * i + 4 * applied + signs], want.float()), (policy, i, applied, signs)


def test_vectorised_table_equals_per_sample_encoding():
    aug = BatchAugment("svhn", 0.3, seed=4)
    H, W = 33, 47
    t = aug.draw(200, H, W).numpy()
    for r in t:
        for k, col, ref in ((0, 0, 12), (1, A.COL_B, A.COL_B + 7)):
            e = _find_entry(r, k)
            code = (A.K_IDENTITY,) if e is None else A.op_code(e[0], e[1], H, W)
            assert np.array_equal(r[col:col + 7], np.float32(list(code) + [0] * (7 - len(code))))
    assert np.all(t[:, 14:16] == 0) and np.all(t[:, A.COL_B + 9:] == 0)
    # encode() is op_code() of TrivialAugmentWide's magnitude
    for op, name in enumerate(A.op_names()):
        for b in (0, 17, 30):
            assert A.encode(op, b, True, H, W) == A.op_code(name, A.magnitude(op, b, True, H, W), H, W)


def test_imagefolder_transforms_follow_the_recipe():
    import torchvision.transforms as TV
    for p in A.AUTOAUGMENT_POLICIES:
        ts = D.train_transforms(argparse.Namespace(image_size=224, auto_augment=p, random_erase=0.2))
        assert [type(t) for t in ts] == [TV.RandomResizedCrop, TV.RandomHorizontalFlip, TV.AutoAugment, TV.ToTensor, TV.Normalize,
                                         TV.RandomErasing]
        assert ts[2].policy == TV.AutoAugmentPolicy(p) and ts[2].interpolation == TV.InterpolationMode.BILINEAR
        assert ts[-1].p == 0.2


def test_cpu_prefetcher_applies_the_reference():
    ld = D.SyntheticLoader(4, 2, 24, 10, raw_uint8=True, pin=False)
    aug, ref = BatchAugment("imagenet", 0.5, seed=2), BatchAugment("imagenet", 0.5, seed=2)
    pf = D.DataPrefetcher(ld, "cpu", torch.float32, False, normalize="imagenet255", augment=aug)
    for (x, _), (raw, _) in zip(pf, ld):
        prm = ref.draw(4, 24, 24)
        assert prm.shape == (4, A.AUG_CHAIN_PRM)
        assert torch.equal(x, BatchAugment.reference_apply(raw, prm, pf._a, pf._b, torch.float32, False))


def _common(d, log, data):
    return T._common(d, log, data)[:-len(T.FLAGS)] + FLAGS


def test_distributed_gloo_world2_on_shards(tmp_path):
    log = tmp_path / "log.jsonl"
    out = T._torchrun(2, _common(tmp_path / "ck", log, T._shards(tmp_path / "data")) + ["--epochs", "1"], 29971)
    assert out.count(" * Acc@1 ") == 2
    recs = T._records(log)
    train = [r for r in recs if r["phase"] == "train"]
    assert len(train) == 2 and all(np.isfinite(r["loss"]) and r["loss"] > 0 for r in recs)


def test_resume_at_epoch_boundary_replays_the_draws(tmp_path):
    env = {"PTD_SAVE_OPTIMIZER": "1"}
    data = T._shards(tmp_path / "data")
    full, half = tmp_path / "full.jsonl", tmp_path / "half.jsonl"
    T._torchrun(1, _common(tmp_path / "full", full, data) + ["--epochs", "2"], 29973, env)
    T._torchrun(1, _common(tmp_path / "half", half, data) + ["--epochs", "1"], 29975, env)
    ck = str(tmp_path / "half" / "checkpoint.pth.tar")
    T._torchrun(1, _common(tmp_path / "half", half, data) + ["--epochs", "2", "--resume", ck], 29977, env)
    a = [r["loss"] for r in T._records(full) if r["phase"] == "train"]
    b = [r["loss"] for r in T._records(half) if r["phase"] == "train"]
    assert len(a) == len(b) == 2 and a == b
