"""MixUp / CutMix / label smoothing (``--mixup-alpha``, ``--cutmix-alpha``, ``--label-smoothing``) without a GPU: the command
line, the draws (distribution, mode choice, CutMix box, streams), the CPU path against torchvision and float64, and gloo
runs of distributed.py (finite loss at world 2, resume at an epoch boundary = uninterrupted run)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from pytorch_distributed_b200 import cli, driver
from pytorch_distributed_b200.ops.mix import CUTMIX, MIXUP, BatchMix, MixTarget, cutmix_box, lam_pair

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FLAGS = ["--label-smoothing", "0.1", "--mixup-alpha", "0.2", "--cutmix-alpha", "1.0"]


def test_cli_defaults_and_ranges():
    a = cli.parse_args("distributed", [])
    assert (a.label_smoothing, a.mixup_alpha, a.cutmix_alpha) == (0.0, 0.0, 0.0)
    b = cli.parse_args("distributed", FLAGS)
    assert (b.label_smoothing, b.mixup_alpha, b.cutmix_alpha) == (0.1, 0.2, 1.0)
    assert {k: v for k, v in vars(a).items() if k not in ("label_smoothing", "mixup_alpha", "cutmix_alpha")} == \
        {k: v for k, v in vars(b).items() if k not in ("label_smoothing", "mixup_alpha", "cutmix_alpha")}
    assert cli.parse_args("distributed", ["--label-smoothing", "1"]).label_smoothing == 1.0
    for bad in (["--label-smoothing", "-0.1"], ["--label-smoothing", "1.5"], ["--label-smoothing", "nan"],
                ["--mixup-alpha", "-1"], ["--mixup-alpha", "inf"], ["--cutmix-alpha", "nan"], ["--cutmix-alpha", "-0.5"]):
        with pytest.raises(SystemExit):
            cli.parse_args("distributed", bad)


def test_no_flag_means_no_batch_mix():
    args = cli.parse_args("distributed", [])
    assert driver.make_batch_mix(args, torch.device("cpu"), 0) is None

    class St:
        batch_mix = None
    step = driver.TrainStep(St(), None, torch.nn.CrossEntropyLoss(), None, None)
    assert step.batch_mix is None and isinstance(step.criterion, torch.nn.CrossEntropyLoss)
    bm = driver.make_batch_mix(cli.parse_args("distributed", ["--label-smoothing", "0.1"]), torch.device("cpu"), 0)
    assert bm is not None and not bm.mixing and bm.label_smoothing == 0.1


@pytest.mark.parametrize("alpha", [0.2, 1.0])
def test_lambda_is_beta_distributed(alpha):
    from scipy import stats
    bm = BatchMix(mixup_alpha=alpha, num_classes=10, seed=3)
    lam = np.array([bm.draw((8, 8))["lam"] for _ in range(10000)])
    assert stats.kstest(lam, stats.beta(alpha, alpha).cdf).pvalue > 1e-3


def test_mode_choice_is_fair():
    bm = BatchMix(mixup_alpha=0.2, cutmix_alpha=1.0, num_classes=10, seed=5)
    n = 10000
    k = sum(bm.draw((32, 32))["mode"] == MIXUP for _ in range(n))
    assert abs(k - n / 2) < 5 * (n * 0.25) ** 0.5          # five binomial standard deviations
    assert {BatchMix(mixup_alpha=1.0, seed=1).draw((4, 4))["mode"] for _ in range(5)} == {MIXUP}
    assert {BatchMix(cutmix_alpha=1.0, seed=1).draw((4, 4))["mode"] for _ in range(5)} == {CUTMIX}


@pytest.mark.parametrize("H,W", [(224, 224), (97, 131)])
def test_cutmix_box_matches_torchvision(monkeypatch, H, W):
    from torchvision.transforms import v2
    cm = v2.CutMix(alpha=1.0, num_classes=10)
    cases = []
    for lam in (0.0, 1e-9, 0.3, 0.5, 0.7, 0.99, 1.0):
        for r_x in (0, 1, W // 2, W - 2, W - 1):
            for r_y in (0, H // 3, H // 2, H - 1):
                cases.append((lam, r_x, r_y))
    seen_empty = seen_full = False
    for lam, r_x, r_y in cases:
        class Dist:
            def sample(self, shape):
                return torch.tensor(lam, dtype=torch.float64)
        draws = iter([torch.tensor([r_x]), torch.tensor([r_y])])
        monkeypatch.setattr(cm, "_dist", Dist())
        monkeypatch.setattr(torch, "randint", lambda *a, **k: next(draws))
        want = cm.make_params([torch.zeros(1, 3, H, W)])
        monkeypatch.undo()
        box, lam_adj = cutmix_box(lam, r_x, r_y, H, W)
        assert box == want["box"] and lam_adj == want["lam_adjusted"], (lam, r_x, r_y)
        seen_empty |= (box[2] - box[0]) * (box[3] - box[1]) == 0
        seen_full |= box == (0, 0, W, H)
    assert seen_empty and seen_full == (H % 2 == 0 and W % 2 == 0)     # an odd side is never covered whole


def test_streams_rekey_per_epoch_and_rank():
    def stream(seed, rank, epoch, n=20):
        bm = BatchMix(mixup_alpha=0.2, cutmix_alpha=1.0, seed=seed, rank=rank)
        bm.set_epoch(epoch)
        return [tuple(sorted(bm.draw((16, 16)).items())) for _ in range(n)]
    bm = BatchMix(mixup_alpha=0.2, cutmix_alpha=1.0, seed=7, rank=1)
    bm.set_epoch(3)
    first = [tuple(sorted(bm.draw((16, 16)).items())) for _ in range(20)]
    bm.set_epoch(4)
    bm.set_epoch(3)
    assert [tuple(sorted(bm.draw((16, 16)).items())) for _ in range(20)] == first == stream(7, 1, 3)
    assert stream(7, 0, 3) != first and stream(7, 1, 4) != first and stream(8, 1, 3) != first
    assert BatchMix(mixup_alpha=1.0).seed != BatchMix(mixup_alpha=1.0).seed        # no seed: OS entropy


def _batch(B=6, H=9, W=11, C=10, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, 3, H, W, generator=g), torch.randint(0, C, (B,), generator=g)


def _soft_labels(t: MixTarget, C):
    la, lb = float(t.prm[1]), float(t.prm[2])
    return F.one_hot(t.y_b, C).float().mul_(lb).add_(F.one_hot(t.y_a, C).float().mul(la))


@pytest.mark.parametrize("mode", [MIXUP, CUTMIX])
def test_cpu_apply_equals_torchvision(mode):
    from torchvision.transforms import v2
    x, y = _batch()
    y[3] = y[2]                                             # one row whose two labels agree
    bm = BatchMix(mixup_alpha=0.2 if mode == MIXUP else 0.0, cutmix_alpha=1.0 if mode == CUTMIX else 0.0, num_classes=10, seed=11)
    for _ in range(20):
        p = bm.draw(x.shape[-2:])
        out, t = bm.apply(x, y)
        if mode == MIXUP:
            tv, params = v2.MixUp(alpha=0.2, num_classes=10), {"lam": p["lam"]}
        else:
            tv, params = v2.CutMix(alpha=1.0, num_classes=10), {"box": p["box"], "lam_adjusted": p["lam"]}
        params.update(labels=y, batch_size=x.shape[0])
        assert torch.equal(out, tv.transform(x, params))
        q = tv.transform(y, params)
        assert torch.equal(_soft_labels(t, 10), q)
        assert torch.equal(t.y_b, y.roll(1, 0))
        top = q.max(dim=1).values
        first_max = (q == top[:, None]).float().argmax(dim=1)    # first index of the row maximum
        assert torch.equal(t.dom, first_max)


def test_dominant_label_on_ties():
    y = torch.tensor([4, 2, 9, 9])
    prm = torch.tensor([MIXUP, 0.5, 0.5, 0, 0, 0, 0, 0])
    _, t = BatchMix.reference_apply(torch.zeros(4, 3, 2, 2), y, prm)
    assert t.dom.tolist() == [4, 2, 2, 9]                   # pairs (4, 9), (2, 4), (9, 2), (9, 9): the smaller label


@pytest.mark.parametrize("eps", [0.0, 0.1])
@pytest.mark.parametrize("lam", [1.0, 0.5, 0.3])
def test_cpu_loss_matches_float64(eps, lam):
    C = 10
    x, y = _batch(B=8, C=C, seed=2)
    la, lb = lam_pair(lam)
    t = MixTarget(y, y.roll(1, 0), y, torch.tensor([MIXUP, la, lb, 0, 0, 0, 0, 0]))
    bm = BatchMix(label_smoothing=eps, num_classes=C)
    z = (torch.randn(8, C, generator=torch.Generator().manual_seed(4)) * 3).requires_grad_()
    loss = bm.loss(z, t)
    loss.backward()
    z64 = z.detach().double().requires_grad_()
    q64 = _soft_labels(t, C).double()
    ref = F.cross_entropy(z64, q64, label_smoothing=eps)
    ref.backward()
    assert abs(float(loss.detach()) - float(ref)) <= 1e-5 * (1 + abs(float(ref)))
    assert torch.allclose(z.grad.double(), z64.grad, rtol=1e-5, atol=1e-7)
    # integer targets (validation): the smoothed criterion is torch's
    out = bm.criterion(z.detach(), y)
    assert torch.equal(out, torch.nn.CrossEntropyLoss(label_smoothing=eps)(z.detach(), y))


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


def _common(d, log):
    d.mkdir(exist_ok=True)
    return ["-a", "resnet18", "-b", "8", "--synthetic", "--image-size", "32", "--num-classes", "10", "-p", "1", "--device", "cpu",
            "--checkpoint-dir", str(d), "--quiet", "--seed", "0", "--log-jsonl", str(log), "--steps-per-epoch", "2",
            "--val-steps", "1"] + FLAGS


def test_distributed_gloo_world2_finite_loss(tmp_path):
    log = tmp_path / "log.jsonl"
    out = _torchrun(2, _common(tmp_path / "ck", log) + ["--epochs", "1"], 29771)
    assert out.count(" * Acc@1 ") == 2
    recs = _records(log)
    train = [r for r in recs if r["phase"] == "train"]
    val = [r for r in recs if r["phase"] == "val"]
    assert len(train) == 2 and len(val) == 2
    assert all(np.isfinite(r["loss"]) and r["loss"] > 0 for r in train + val)


def test_resume_at_epoch_boundary_replays_the_draws(tmp_path):
    env = {"PTD_SAVE_OPTIMIZER": "1"}
    full, half = tmp_path / "full.jsonl", tmp_path / "half.jsonl"
    _torchrun(1, _common(tmp_path / "full", full) + ["--epochs", "2"], 29773, env)
    _torchrun(1, _common(tmp_path / "half", half) + ["--epochs", "1"], 29775, env)
    ck = str(tmp_path / "half" / "checkpoint.pth.tar")
    _torchrun(1, _common(tmp_path / "half", half) + ["--epochs", "2", "--resume", ck], 29777, env)
    a = [r["loss"] for r in _records(full) if r["phase"] == "train"]
    b = [r["loss"] for r in _records(half) if r["phase"] == "train"]
    assert len(a) == len(b) == 2 and a == b
