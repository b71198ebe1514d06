"""MixUp / CutMix / label smoothing on the GPU (``csrc/mix.cu``): ``mix_batch`` bit for bit against the CPU path (itself equal
to torchvision's transforms), the soft-target cross-entropy against float64 ``F.cross_entropy``, eager and CUDA-graph training
steps bit for bit, and the entrypoints."""
import json
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

from pytorch_distributed_b200.ops.mix import CUTMIX, MIXUP, BatchMix, MixTarget, lam_pair

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DTYPES = {"fp32": torch.float32, "bf16": torch.bfloat16, "fp16": torch.float16}
FLAGS = ["--label-smoothing", "0.1", "--mixup-alpha", "0.2", "--cutmix-alpha", "1.0"]


def C():
    from pytorch_distributed_b200 import _ext
    return _ext.lib()


def _prm(mode, lam, box=(0, 0, 0, 0)):
    la, lb = lam_pair(lam)
    return torch.tensor([mode, la, lb, *box, 0], dtype=torch.float32)


def _cases(H, W):
    """(mode, lam, box): random draws of both kinds, a lambda = 0.5 tie, and boxes that are empty, whole, one pixel, or have
    edges on odd columns (inside a 16-byte vector in both layouts)."""
    bm = BatchMix(mixup_alpha=0.2, cutmix_alpha=1.0, seed=1)
    out = []
    for _ in range(4):
        d = bm.draw((H, W))
        out.append((d["mode"], d["lam"], d["box"]))
    out += [(MIXUP, 0.5, (0, 0, 0, 0)), (MIXUP, 1.0, (0, 0, 0, 0)), (CUTMIX, 0.5, (3, 1, 3, 1)), (CUTMIX, 0.0, (0, 0, W, H)),
            (CUTMIX, 0.7, (W // 2, H // 2, W // 2 + 1, H // 2 + 1)), (CUTMIX, 0.6, (1, 2, W - 3, H - 1))]
    return out


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("nhwc", [True, False], ids=["nhwc", "nchw"])
@pytest.mark.parametrize("shape", [(256, 224, 224), (1, 97, 131), (3, 97, 131), (3, 96, 100)], ids=lambda s: "x".join(map(str, s)))
def test_mix_batch_bit_equal_to_cpu(dtype, nhwc, shape):
    B, H, W = shape
    dt = DTYPES[dtype]
    g = torch.Generator().manual_seed(B * H)
    x = torch.randn(B, 3, H, W, generator=g).to(dt)
    y = torch.randint(0, 1000, (B,), generator=g)
    if B > 1:
        y[1] = y[0]                                       # a row whose two labels agree
    xd = x.cuda()
    xd = xd.contiguous(memory_format=torch.channels_last) if nhwc else xd.contiguous()
    yd = y.cuda()
    out = torch.empty_like(xd)
    yb, dom = torch.empty_like(yd), torch.empty_like(yd)
    cases = _cases(H, W)
    for mode, lam, box in (cases if B < 256 else cases[:2] + cases[-3:]):
        prm = _prm(mode, lam, box)
        C().mix_batch(xd, out, yd, yb, dom, prm.cuda())
        want, t = BatchMix.reference_apply(x, y, prm)
        assert out.is_contiguous(memory_format=torch.channels_last) == nhwc
        got = out.cpu()
        assert torch.equal(got.view(torch.int16 if dt != torch.float32 else torch.int32),
                           want.view(torch.int16 if dt != torch.float32 else torch.int32)), (mode, lam, box)
        assert torch.equal(yb.cpu(), t.y_b) and torch.equal(dom.cpu(), t.dom), (mode, lam, box)


def _ref_loss(z, t: MixTarget, eps):
    la, lb = float(t.prm[1]), float(t.prm[2])
    Cn = z.size(1)
    q = F.one_hot(t.y_b.cpu(), Cn).double().mul_(lb).add_(F.one_hot(t.y_a.cpu(), Cn).double().mul(la))
    z64 = z.detach().cpu().double().requires_grad_()
    rows = F.cross_entropy(z64, q, label_smoothing=eps, reduction="none")
    rows.mean().backward()
    return rows.detach(), z64.grad, torch.softmax(z64.detach(), 1)


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("eps", [0.0, 0.1])
@pytest.mark.parametrize("lam", [1.0, 0.5, 0.3])
@pytest.mark.parametrize("gscale", [1.0, 65536.0])
def test_soft_ce_against_float64(dtype, eps, lam, gscale):
    """fp32 evaluation with the approximate exp / log of sm_90: each row's loss within 1e-5 (1 + max |z|) of float64 (a few
    fp32 roundings of terms the size of the largest logit), and dz within g/B (2e-5 p + 1e-6) of it (the relative error of
    exp(z - lse)) plus one rounding to the logits' dtype."""
    dt = DTYPES[dtype]
    B, Cn = 256, 1000
    g = torch.Generator(device="cuda").manual_seed(7)
    full = (torch.randn(B, Cn + 24, device="cuda", generator=g) * 3).to(dt)
    z = full[:, :Cn]                                      # a row stride wider than the row
    y = torch.randint(0, Cn, (B,), device="cuda", generator=g)
    y[1] = y[0]
    la, lb = lam_pair(lam)
    t = MixTarget(y, y.roll(1, 0), y, torch.tensor([MIXUP, la, lb, 0, 0, 0, 0, 0], device="cuda"))
    loss, rows, lse = C().soft_ce_fwd(z, t.y_a, t.y_b, t.prm, eps)
    gt = torch.tensor(gscale, device="cuda")
    dz = C().soft_ce_bwd(z, t.y_a, t.y_b, t.prm, lse, gt, eps)
    ref_rows, ref_dz, p = _ref_loss(z, t, eps)
    zmax = float(z.float().abs().max())
    assert ((rows.cpu().double() - ref_rows).abs() <= 1e-5 * (1 + zmax)).all()
    assert abs(float(loss) - float(ref_rows.mean())) <= 1e-5 * (1 + zmax)
    ref_dz = ref_dz * gscale
    u = {torch.float32: 2.0 ** -24, torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}[dt]
    tiny = 2.0 ** -25 if dt == torch.float16 else 0.0    # half of fp16's subnormal spacing
    bound = gscale / B * (2e-5 * p + 1e-6) + u * ref_dz.abs() * 1.01 + tiny
    err = (dz.cpu().double() - ref_dz).abs()
    assert dz.dtype == dt and (err <= bound).all(), float((err - bound).max())
    # run to run: the same bits
    loss2, rows2, lse2 = C().soft_ce_fwd(z, t.y_a, t.y_b, t.prm, eps)
    dz2 = C().soft_ce_bwd(z, t.y_a, t.y_b, t.prm, lse2, gt, eps)
    assert torch.equal(loss, loss2) and torch.equal(rows, rows2) and torch.equal(dz.view(-1), dz2.view(-1))


def test_soft_ce_autograd_and_criterion():
    bm = BatchMix(label_smoothing=0.1, num_classes=1000, device="cuda")
    z = torch.randn(64, 1000, device="cuda").to(torch.bfloat16).requires_grad_()
    y = torch.randint(0, 1000, (64,), device="cuda")
    loss = bm.criterion(z, y)
    loss.backward()
    z64 = z.detach().double().requires_grad_()
    ref = F.cross_entropy(z64, y, label_smoothing=0.1)
    ref.backward()
    assert loss.dtype == torch.float32 and abs(float(loss.detach()) - float(ref.detach())) < 1e-4
    assert torch.allclose(z.grad.double(), z64.grad, rtol=2 ** -7, atol=1e-7)


def test_out_of_range_label_is_nan_in_its_row_only():
    B, Cn = 32, 1000
    z = torch.randn(B, Cn, device="cuda")
    y = torch.randint(0, Cn, (B,), device="cuda")
    y[5], y[9] = Cn, -1
    prm = torch.tensor([0, 1, 0, 0, 0, 0, 0, 0], dtype=torch.float32, device="cuda")
    loss, rows, lse = C().soft_ce_fwd(z, y, y, prm, 0.1)
    dz = C().soft_ce_bwd(z, y, y, prm, lse, torch.tensor(1.0, device="cuda"), 0.1)
    bad = torch.zeros(B, dtype=torch.bool)
    bad[5] = bad[9] = True
    assert torch.isnan(rows.cpu()[bad]).all() and torch.isfinite(rows.cpu()[~bad]).all()
    assert torch.isnan(dz.cpu()[bad]).all() and torch.isfinite(dz.cpu()[~bad]).all()
    assert torch.isnan(loss)


def test_apply_owns_a_fixed_buffer_for_the_static_shape():
    bm = BatchMix(mixup_alpha=0.2, num_classes=1000, seed=0, device="cuda")
    x = torch.randn(4, 3, 32, 32, device="cuda").contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 1000, (4,), device="cuda")
    bm.draw((32, 32))
    a, _ = bm.apply(x, y)
    bm.draw((32, 32))
    b, _ = bm.apply(x, y)
    c, _ = bm.apply(x[:2], y[:2])
    assert a.data_ptr() == b.data_ptr() != c.data_ptr()
    want, _ = BatchMix.reference_apply(x.cpu(), y.cpu(), bm.prm.cpu())
    assert torch.equal(b.cpu(), want)


# ------------------------------------------------------------------------------------------------ training steps
def _paths(tmp_path, runs):
    out = tmp_path / "paths.pt"
    e = dict(os.environ, PYTHONPATH=ROOT)
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "MASTER_ADDR", "MASTER_PORT"):
        e.pop(k, None)
    p = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "mix_paths.py"), str(out), json.dumps(runs)], env=e,
                       cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-3000:] + "\n" + p.stderr[-3000:]
    return torch.load(out, weights_only=False)


@pytest.mark.parametrize("argv", [FLAGS, ["--mixup-alpha", "1.0", "--larc"]], ids=["all-three", "mixup-larc"])
@pytest.mark.parametrize("accum", [1, 2])
def test_graph_replays_equal_eager_steps(tmp_path, argv, accum):
    argv = argv + ["--accum-steps", str(accum)]
    eager, graph = _paths(tmp_path, [{"argv": argv}, {"argv": argv, "graph": True}])
    assert graph["graph"] and not eager["graph"]
    lams = [s["draw"]["lam"] for s in graph["steps"] if s["graph"]]
    assert len(lams) >= 2 and len(set(lams)) == len(lams)          # new draws reach the replays
    for i, (a, b) in enumerate(zip(eager["steps"], graph["steps"])):
        assert a["draw"] == b["draw"], i
        assert torch.equal(a["mixed"], b["mixed"]), i
        assert a["metrics"] == b["metrics"], i
    assert torch.equal(eager["master"], graph["master"])


# ------------------------------------------------------------------------------------------------ entrypoints
COMMON = ["-a", "resnet50", "-b", "32", "--synthetic", "--steps-per-epoch", "4", "--val-steps", "1", "--epochs", "1",
          "--image-size", "96", "-p", "1"] + FLAGS


def _run(cmd, tmp_path):
    e = dict(os.environ, PYTHONPATH=ROOT)
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "MASTER_ADDR", "MASTER_PORT"):
        e.pop(k, None)
    p = subprocess.run(cmd, env=e, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-3000:] + "\n" + p.stderr[-3000:]
    with open(tmp_path / "log.jsonl") as f:
        recs = [json.loads(l) for l in f if l.strip()]
    assert {"train", "val"} <= {r["phase"] for r in recs}
    assert all(torch.isfinite(torch.tensor(r["loss"])) and r["loss"] > 0 for r in recs), recs
    return p.stdout


@pytest.mark.parametrize("script,extra,port", [
    ("distributed.py", ["--cuda-graph"], 29831),
    ("distributed.py", ["--cuda-graph", "--accum-steps", "2", "--model-ema"], 29832),
    ("apex_distributed.py", ["--cuda-graph", "--opt-level", "O2", "--precision", "fp16"], 29833),
    ("apex_distributed.py", ["--opt-level", "O1"], 29834),
    ("horovod_distributed.py", ["--cuda-graph"], 29835),
    ("dataparallel.py", [], None),
], ids=["ddp-graph", "ddp-accum2-ema", "apex-o2", "apex-o1", "horovod", "dataparallel"])
def test_entrypoint_runs(script, extra, port, tmp_path):
    args = COMMON + extra + ["--checkpoint-dir", str(tmp_path), "--log-jsonl", str(tmp_path / "log.jsonl")]
    if port is None:
        cmd = [sys.executable, os.path.join(ROOT, script), "--gpus", "0"] + args
    else:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "1", "--master-addr", "127.0.0.1",
               "--master-port", str(port), os.path.join(ROOT, script)] + args
    _run(cmd, tmp_path)


@pytest.mark.multigpu
def test_ddp_world2_runs(tmp_path):
    args = COMMON + ["--cuda-graph", "--sync-bn", "--checkpoint-dir", str(tmp_path), "--log-jsonl", str(tmp_path / "log.jsonl")]
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29839", os.path.join(ROOT, "distributed.py")] + args
    _run(cmd, tmp_path)
