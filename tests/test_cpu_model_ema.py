"""ModelEma (``--model-ema``) without a GPU: the command line, FusedSGD's CPU reference path against a float64 average, the
exact endpoints, gloo world-2 runs of distributed.py (ranks agree, checkpoint layout, resume = uninterrupted run)."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from pytorch_distributed_b200 import cli
from pytorch_distributed_b200.ops.fused_sgd import FusedSGD
from pytorch_distributed_b200.utils.ema import ModelEma, decay_pair

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -24          # fp32 unit roundoff


def test_cli_flags():
    a = cli.parse_args("distributed", [])
    assert a.model_ema is False and a.model_ema_decay == 0.9999
    a = cli.parse_args("distributed", ["--model-ema", "--model-ema-decay", "0.99"])
    assert a.model_ema and a.model_ema_decay == 0.99
    assert cli.parse_args("distributed", ["--model-ema", "--model-ema-decay", "0"]).model_ema_decay == 0.0
    for bad in (["--model-ema-decay", "0.99"], ["--model-ema", "--model-ema-decay", "1"],
                ["--model-ema", "--model-ema-decay", "-0.1"], ["--model-ema", "--model-ema-decay", "nan"]):
        with pytest.raises(SystemExit):
            cli.parse_args("distributed", bad)


def _model(seed=0):
    torch.manual_seed(seed)
    return torch.nn.Sequential(torch.nn.Linear(16, 32), torch.nn.BatchNorm1d(32), torch.nn.ReLU(), torch.nn.Linear(32, 4))


def _train(model, opt, ema, steps, seed=1, record=None):
    g = torch.Generator().manual_seed(seed)
    for _ in range(steps):
        x = torch.randn(8, 16, generator=g)
        opt.zero_grad()
        model(x).square().mean().backward()
        opt.step()
        ema.update()
        if record is not None:
            record.append({k: v.detach().clone() for k, v in model.state_dict().items()})


@pytest.mark.parametrize("decay", [0.9, 0.5, 0.9999])
def test_reference_path_matches_float64(decay):
    """The fp32 average of the CPU path against a float64 average of the same master trajectory (the one FusedSGD's
    fp32 SGD produced, itself checked against float64 SGD elsewhere).  Per step the fp32 evaluation adds at most
    u |w p| (the product) + 2 u |e| (fmaf's rounding, and the double rounding of the CPU path) to the error, which the
    decay then damps: err_k <= d err_{k-1} + u (|w p_k| + 2 |e_k|)."""
    model = _model()
    opt = FusedSGD(model.parameters(), lr=0.1, momentum=0.9, weight_decay=1e-4)
    ema = ModelEma(model, decay=decay, optimizer=opt)
    assert ema.module is not model and all(a.data_ptr() != b.data_ptr() for a, b in zip(ema.module.parameters(), model.parameters()))
    init = {k: v.detach().double().clone() for k, v in model.state_dict().items() if v.is_floating_point()}
    traj = []
    _train(model, opt, ema, 6, record=traj)
    d, w = decay_pair(decay)
    e64 = dict(init)
    bound = {k: torch.zeros_like(v) for k, v in init.items()}
    for sd in traj:
        for k in e64:
            p = sd[k].double()
            e64[k] = d * e64[k] + (1 - d) * p
            bound[k] = d * bound[k] + U * (w * p.abs() + 2 * e64[k].abs()) + abs(w - (1 - d)) * p.abs()
    got = ema.state_dict()
    for k in e64:
        err = (got[k].double() - e64[k]).abs()
        assert (err <= bound[k] * 1.0001 + 1e-30).all(), (k, float(err.max()), float(bound[k].max()))
    assert torch.equal(got["1.num_batches_tracked"], model.state_dict()["1.num_batches_tracked"])


@pytest.mark.parametrize("decay", [0.0, 1.0])
def test_endpoints_are_exact(decay):
    model = _model()
    init = {k: v.detach().clone() for k, v in model.state_dict().items()}
    opt = FusedSGD(model.parameters(), lr=0.1, momentum=0.9, weight_decay=1e-4)
    ema = ModelEma(model, decay=decay, optimizer=opt)
    _train(model, opt, ema, 3)
    got = ema.state_dict()
    want = model.state_dict() if decay == 0.0 else init
    for k, v in want.items():
        if v.is_floating_point():
            assert torch.equal(got[k], v), k


def test_torch_optimizer_update_and_sync_module():
    """A stock optimizer: update() does the averaging; sync_module() writes it into the copy, whose forward is then the
    averaged model's."""
    model = _model()
    opt = torch.optim.SGD(model.parameters(), lr=0.1, momentum=0.9)
    ema = ModelEma(model, decay=0.0, optimizer=opt)
    _train(model, opt, ema, 2)
    ema.sync_module()
    x = torch.randn(4, 16)
    model.eval()
    assert torch.equal(ema.module(x), model(x))


def test_decay_setter_and_load_state_dict():
    model = _model()
    opt = FusedSGD(model.parameters(), lr=0.1, momentum=0.9)
    ema = ModelEma(model, decay=0.5, optimizer=opt)
    ema.decay = 0.25
    assert ema.decay_pair() == (0.25, 0.75)
    with pytest.raises(ValueError):
        ema.decay = 1.5
    sd = {"module." + k: v.clone() + 1 if v.is_floating_point() else v for k, v in ema.state_dict().items()}
    ema.load_state_dict(sd)
    for k, v in ema.state_dict().items():
        assert torch.equal(v, sd["module." + k]), k


def _torchrun(tmp_path, name, argv, port, env_extra=None):
    env = dict(os.environ, OMP_NUM_THREADS="1", PYTHONPATH=ROOT, **(env_extra or {}))
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "MASTER_ADDR", "MASTER_PORT"):
        env.pop(k, None)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "tests", "mp_model_ema_checks.py"), str(tmp_path / name), "distributed"] + argv
    p = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-3000:] + "\n" + p.stderr[-3000:]
    return p.stdout


def _common(tmp_path, arch="resnet18", sub="ck"):
    d = tmp_path / sub
    d.mkdir(exist_ok=True)
    return ["-a", arch, "-b", "8", "--synthetic", "--image-size", "32", "--num-classes", "10", "-p", "1", "--device", "cpu",
            "--checkpoint-dir", str(d), "--quiet", "--model-ema", "--model-ema-decay", "0.9", "--seed", "0"]


def test_distributed_gloo_world2_ranks_agree_and_checkpoint_loads(tmp_path):
    import torchvision
    out = _torchrun(tmp_path, "out", _common(tmp_path, "resnet50") + ["--steps-per-epoch", "3", "--val-steps", "1", "--epochs", "1"],
                    29751)
    assert out.count(" * EMA Acc@1 ") == 2 and out.count(" * Acc@1 ") == 2
    r0 = torch.load(tmp_path / "out" / "rank0.pt", weights_only=False)["ema"]
    r1 = torch.load(tmp_path / "out" / "rank1.pt", weights_only=False)["ema"]
    assert r0.keys() == r1.keys()
    for k in r0:
        assert torch.equal(r0[k], r1[k]), k
    ck = torch.load(tmp_path / "ck" / "checkpoint.pth.tar", weights_only=False)
    sde = ck["state_dict_ema"]
    assert list(sde.keys()) == list(ck["state_dict"].keys())
    assert all(v.dtype == torch.float32 for v in sde.values() if v.is_floating_point())
    assert any(not torch.equal(sde[k], ck["state_dict"][k]) for k in sde if sde[k].is_floating_point())
    ref = torchvision.models.resnet50(num_classes=10)
    ref.load_state_dict(sde)


def test_resume_gives_the_uninterrupted_average(tmp_path):
    env = {"PTD_SAVE_OPTIMIZER": "1"}
    base = ["--steps-per-epoch", "2", "--val-steps", "1"]
    _torchrun(tmp_path, "full", _common(tmp_path, sub="full") + base + ["--epochs", "2"], 29753, env)
    _torchrun(tmp_path, "half", _common(tmp_path, sub="half") + base + ["--epochs", "1"], 29755, env)
    ck = str(tmp_path / "half" / "checkpoint.pth.tar")
    _torchrun(tmp_path, "resumed", _common(tmp_path, sub="half") + base + ["--epochs", "2", "--resume", ck], 29757, env)
    a = torch.load(tmp_path / "full" / "checkpoint.pth.tar", weights_only=False)
    b = torch.load(tmp_path / "half" / "checkpoint.pth.tar", weights_only=False)
    assert a["epoch"] == b["epoch"] == 2
    for key in ("state_dict", "state_dict_ema"):
        for k in a[key]:
            assert torch.equal(a[key][k], b[key][k]), (key, k)


def test_decay_pair_rounding():
    d, w = decay_pair(0.9999)
    assert d == float(np.float32(0.9999)) and w == float(np.float32(1 - d))
    assert decay_pair(0.0) == (0.0, 1.0) and decay_pair(1.0) == (1.0, 0.0)
