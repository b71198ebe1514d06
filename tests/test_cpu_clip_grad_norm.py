"""Global-norm gradient clipping (``--clip-grad-norm``) without a GPU: the command line, FusedSGD's CPU path against
``torch.optim.SGD`` after ``torch.nn.utils.clip_grad_norm_`` in float64, NaN and infinite norms, loss scaling and a skipped
step, the order against LARC, changing max_norm between steps, and gloo world-2 runs of distributed.py."""
import json
import os
import subprocess
import sys

import pytest
import torch

from pytorch_distributed_b200 import cli
from pytorch_distributed_b200.apex.parallel.LARC import LARC
from pytorch_distributed_b200.ops.fused_sgd import FusedSGD
from pytorch_distributed_b200.parallel.amp import LossScaler

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_cli_flag():
    assert cli.parse_args("distributed", []).clip_grad_norm is None
    assert cli.parse_args("distributed", ["--clip-grad-norm", "1.0"]).clip_grad_norm == 1.0
    assert cli.parse_args("apex_distributed", ["--clip-grad-norm", "0.25"]).clip_grad_norm == 0.25
    for bad in ("0", "-1", "nan", "inf", "x"):
        with pytest.raises(SystemExit):
            cli.parse_args("distributed", ["--clip-grad-norm", bad])


def test_set_clip_grad_norm_validates():
    p = torch.nn.Parameter(torch.ones(3))
    opt = FusedSGD([p], lr=0.1)
    assert opt.grad_norm() is None and opt.clipped_steps() is None
    for bad in (0.0, -1.0, float("nan"), float("inf")):
        with pytest.raises(ValueError):
            opt.set_clip_grad_norm(bad)
    with pytest.raises(ValueError):
        FusedSGD([p], lr=0.1, clip_grad_norm=0.0)
    opt.set_clip_grad_norm(2.0)
    opt.set_clip_grad_norm(None)


def _model(dtype, seed=0):
    torch.manual_seed(seed)
    return torch.nn.Sequential(torch.nn.Linear(16, 32), torch.nn.ReLU(), torch.nn.Linear(32, 4)).to(dtype)


def _groups(model, two_groups, wd):
    ps = list(model.parameters())
    if not two_groups:
        return [{"params": ps}]
    return [{"params": ps[:2]}, {"params": ps[2:], "weight_decay": 0.0 if wd else 1e-3, "lr": 0.05}]


def _batches(n, seed=1, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(8, 16, generator=g) * scale, torch.randn(8, 4, generator=g)) for _ in range(n)]


def _loss(model, x, y):
    return (model(x.to(next(model.parameters()).dtype)) - y.to(next(model.parameters()).dtype)).square().mean()


def _torch_run(model, groups, batches, max_norms, larc=False, **kw):
    opt = torch.optim.SGD(groups, **kw)
    if larc:
        opt = LARC(opt, trust_coefficient=0.02, clip=True)
    norms = []
    for (x, y), mn in zip(batches, max_norms):
        opt.zero_grad()
        _loss(model, x, y).backward()
        norms.append(float(torch.nn.utils.clip_grad_norm_(model.parameters(), mn)) if mn is not None else None)
        opt.step()
    return norms


def _fused_run(model, groups, batches, max_norms, larc=False, **kw):
    opt = FusedSGD(groups, clip_grad_norm=max_norms[0], **kw)
    if larc:
        opt = LARC(opt, trust_coefficient=0.02, clip=True)
    norms = []
    for (x, y), mn in zip(batches, max_norms):
        opt.set_clip_grad_norm(mn)
        opt.zero_grad()
        _loss(model, x, y).backward()
        opt.step()
        norms.append(float(opt.grad_norm()) if mn is not None else None)
    return opt, norms


def _check_close(m32, m64, tol=2e-5):
    for a, b in zip(m32.parameters(), m64.parameters()):
        err = (a.detach().double() - b.detach()).abs().max().item()
        assert err <= tol * (1 + b.detach().abs().max().item()), err


@pytest.mark.parametrize("max_norm", [0.05, 1e3])
@pytest.mark.parametrize("nesterov,wd,two_groups", [(False, 0.0, False), (True, 1e-2, False), (False, 1e-2, True)])
def test_reference_path_matches_torch_float64(max_norm, nesterov, wd, two_groups):
    """0.05 clips every step, 1e3 none.  FusedSGD's fp32 CPU path against torch.optim.SGD + clip_grad_norm_ in float64."""
    batches = _batches(4)
    kw = dict(lr=0.1, momentum=0.9, weight_decay=wd, nesterov=nesterov)
    m32, m64 = _model(torch.float32), _model(torch.float64)
    opt, got = _fused_run(m32, _groups(m32, two_groups, wd), batches, [max_norm] * 4, **kw)
    want = _torch_run(m64, _groups(m64, two_groups, wd), batches, [max_norm] * 4, **kw)
    _check_close(m32, m64)
    for a, b in zip(got, want):
        assert abs(a - b) <= 1e-5 * b
    assert int(opt.clipped_steps()) == (4 if max_norm < 1 else 0)
    assert all(p.grad is not None for p in m32.parameters())      # the gradients themselves are left unclipped


def test_set_clip_grad_norm_between_steps():
    batches = _batches(5)
    norms = [0.05, 0.2, None, 1e3, 0.01]
    m32, m64 = _model(torch.float32), _model(torch.float64)
    opt, got = _fused_run(m32, m32.parameters(), batches, norms, lr=0.1, momentum=0.9)
    want = _torch_run(m64, m64.parameters(), batches, norms, lr=0.1, momentum=0.9)
    _check_close(m32, m64)
    assert int(opt.clipped_steps()) == sum(1 for g, mn in zip(want, norms) if mn is not None and mn / (g + 1e-6) < 1)


def test_nan_norm_gives_nan_weights_like_torch():
    for opt_kind in ("fused", "torch"):
        m = _model(torch.float32)
        opt = FusedSGD(m.parameters(), lr=0.1, clip_grad_norm=1.0) if opt_kind == "fused" else torch.optim.SGD(m.parameters(), lr=0.1)
        _loss(m, *_batches(1)[0]).backward()
        m[0].weight.grad[0, 0] = float("nan")
        if opt_kind == "torch":
            torch.nn.utils.clip_grad_norm_(m.parameters(), 1.0)
        opt.step()
        assert all(torch.isnan(p).all() for p in m.parameters()), opt_kind
        if opt_kind == "fused":
            assert torch.isnan(opt.grad_norm()) and int(opt.clipped_steps()) == 0


def test_infinite_norm_gives_zero_gradient():
    """Finite gradients whose squares overflow fp32: the norm is inf, the coefficient 0, the step leaves p unchanged."""
    m = _model(torch.float32)
    before = [p.detach().clone() for p in m.parameters()]
    opt = FusedSGD(m.parameters(), lr=0.1, momentum=0.9, clip_grad_norm=1.0)
    for p in m.parameters():
        p.grad = torch.full_like(p, 1e30)
    opt.step()
    assert opt.grad_norm() == float("inf") and int(opt.clipped_steps()) == 1
    for a, b in zip(before, m.parameters()):
        assert torch.equal(a, b)


def test_loss_scaler_scaled_gradient_and_skipped_step():
    """The norm is taken of the unscaled gradient; an overflowed step changes no weight, momentum, norm or count."""
    batches = _batches(3)
    m32, m64 = _model(torch.float32), _model(torch.float64)
    opt = FusedSGD(m32.parameters(), lr=0.1, momentum=0.9, clip_grad_norm=0.05)
    scaler = LossScaler("cpu", init_scale=1024.0)
    opt._amp = scaler
    got = []
    for x, y in batches:
        opt.zero_grad()
        (_loss(m32, x, y) * scaler.loss_scale()).backward()
        opt.step()
        got.append(float(opt.grad_norm()))
    want = _torch_run(m64, m64.parameters(), batches, [0.05] * 3, lr=0.1, momentum=0.9)
    _check_close(m32, m64)
    for a, b in zip(got, want):
        assert abs(a - b) <= 1e-5 * b
    state = [p.detach().clone() for p in m32.parameters()] + [opt.state[p]["momentum_buffer"].clone() for p in m32.parameters()]
    norm, count = opt.grad_norm().clone(), opt.clipped_steps().clone()
    opt.zero_grad()
    (_loss(m32, *batches[0]) * scaler.loss_scale()).backward()
    m32[0].weight.grad[0, 0] = float("inf")
    scaler.found_inf.fill_(1)
    opt.step()
    after = [p.detach() for p in m32.parameters()] + [opt.state[p]["momentum_buffer"] for p in m32.parameters()]
    assert all(torch.equal(a, b) for a, b in zip(state, after))
    assert torch.equal(norm, opt.grad_norm()) and torch.equal(count, opt.clipped_steps())


def test_larc_sees_the_clipped_gradient():
    """LARC(FusedSGD(clip_grad_norm)) against torch's clipping followed by LARC(torch.optim.SGD), in float64."""
    batches = _batches(4)
    kw = dict(lr=0.1, momentum=0.9, weight_decay=1e-3)
    m32, m64 = _model(torch.float32), _model(torch.float64)
    _, got = _fused_run(m32, m32.parameters(), batches, [0.05] * 4, larc=True, **kw)
    want = _torch_run(m64, m64.parameters(), batches, [0.05] * 4, larc=True, **kw)
    _check_close(m32, m64)
    for a, b in zip(got, want):
        assert abs(a - b) <= 1e-5 * b


def test_state_dict_unchanged():
    m = _model(torch.float32)
    a = FusedSGD(m.parameters(), lr=0.1, momentum=0.9)
    b = FusedSGD(m.parameters(), lr=0.1, momentum=0.9, clip_grad_norm=1.0)
    assert a.state_dict() == b.state_dict()


def _torchrun(tmp_path, name, argv, port):
    env = dict(os.environ, OMP_NUM_THREADS="1", PYTHONPATH=ROOT)
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "MASTER_ADDR", "MASTER_PORT"):
        env.pop(k, None)
    d = tmp_path / name
    d.mkdir()
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "distributed.py"), "-a", "resnet18", "-b", "8", "--synthetic",
           "--image-size", "32", "--num-classes", "10", "-p", "1", "--device", "cpu", "--checkpoint-dir", str(d), "--quiet",
           "--seed", "0", "--steps-per-epoch", "3", "--val-steps", "1", "--epochs", "1", "--log-jsonl", str(d / "log.jsonl")] + argv
    p = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-3000:] + "\n" + p.stderr[-3000:]
    recs = [json.loads(line) for line in open(d / "log.jsonl")]
    return [r for r in recs if r["phase"] == "train"], torch.load(d / "checkpoint.pth.tar", weights_only=False)["state_dict"]


def test_distributed_gloo_world2_ranks_agree_and_match_torch(tmp_path):
    fused, sd_f = _torchrun(tmp_path, "fused", ["--clip-grad-norm", "0.5"], 29771)
    stock, sd_t = _torchrun(tmp_path, "torch", ["--clip-grad-norm", "0.5", "--optimizer", "torch"], 29773)
    assert sorted(r["rank"] for r in fused) == [0, 1] and sorted(r["rank"] for r in stock) == [0, 1]
    assert fused[0]["grad_norm"] == fused[1]["grad_norm"] and fused[0]["clipped_steps"] == fused[1]["clipped_steps"] == 3
    assert stock[0]["grad_norm"] == stock[1]["grad_norm"] and stock[0]["clipped_steps"] == 3
    assert abs(fused[0]["grad_norm"] - stock[0]["grad_norm"]) <= 1e-4 * stock[0]["grad_norm"]
    for k, v in sd_t.items():
        if v.is_floating_point():
            assert torch.allclose(sd_f[k], v, rtol=1e-4, atol=1e-5), k
