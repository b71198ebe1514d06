"""Synchronised BatchNorm on CPU: gloo, world 2, through the PyTorch emulation of the fused kernels (``fused="emulate"``)
and through the unfused path, against fp64 BatchNorm over the concatenated global batch; module conversion, the public
names, the command-line switch and its rejections."""
import os
import subprocess
import sys

import pytest
import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

WORKER = r'''
import sys
import torch
import torch.distributed as dist
sys.path.insert(0, sys.argv[1])
from pytorch_distributed_b200.models.resnet import SyncBNAct
from pytorch_distributed_b200.parallel.comm import TorchCommunicator
from pytorch_distributed_b200.utils.dist_ops import set_default_communicator

dist.init_process_group("gloo")
r, W = dist.get_rank(), dist.get_world_size()
set_default_communicator(TorchCommunicator(device="cpu"))
C, H = 16, 5
rows = [3, 5]                                   # per-rank batches differ
g = torch.Generator().manual_seed(0)
xg = torch.randn(sum(rows), C, H, H, generator=g, dtype=torch.float64) * 3 + 1.5
dyg = torch.randn(sum(rows), C, H, H, generator=g, dtype=torch.float64)
w0 = torch.rand(C, generator=g, dtype=torch.float64) + 0.5
b0 = torch.randn(C, generator=g, dtype=torch.float64)
lo, hi = sum(rows[:r]), sum(rows[:r + 1])
eps, mom = 1e-5, 0.1

# fp64 reference: BatchNorm over the global batch
mean = xg.mean((0, 2, 3)); var = xg.var((0, 2, 3), unbiased=False); n = xg.numel() // C
xhat = (xg - mean.view(1, C, 1, 1)) / torch.sqrt(var + eps).view(1, C, 1, 1)
y_ref = xhat * w0.view(1, C, 1, 1) + b0.view(1, C, 1, 1)
x_req = xg.clone().requires_grad_(True)
yy = torch.nn.functional.batch_norm(x_req, None, None, w0, b0, True, mom, eps)
(yy * dyg).sum().backward()
dx_ref = x_req.grad[lo:hi]
dw_ref = (dyg * xhat)[lo:hi].sum((0, 2, 3)); db_ref = dyg[lo:hi].sum((0, 2, 3))
rm_ref = mom * mean; rv_ref = (1 - mom) + mom * var * n / (n - 1)

def close(a, b, name, tol=2e-5):
    err = (a.double() - b).abs().max().item() / max(1.0, b.abs().max().item())
    assert err < tol, "%s: rank %d, mode %s, rel err %.3g" % (name, r, mode, err)

for mode in ("emulate", False):
    layer = SyncBNAct(C, eps=eps, momentum=mom, fused=mode)
    with torch.no_grad():
        layer.weight.copy_(w0); layer.bias.copy_(b0)
    x = xg[lo:hi].float()
    if mode == "emulate":
        x = x.contiguous(memory_format=torch.channels_last)
    x.requires_grad_(True)
    y = layer(x)
    if mode == "emulate":                        # backwards through a retained graph: each exchanges fresh sums, same bits
        l = (y.double() * dyg[lo:hi]).sum()
        g1 = torch.autograd.grad(l, [x, layer.weight, layer.bias], retain_graph=True)
        g2 = torch.autograd.grad(l, [x, layer.weight, layer.bias], retain_graph=True)
        assert all(torch.equal(a, b) for a, b in zip(g1, g2)), "rank %d: the second backward differs from the first" % r
    (y.double() * dyg[lo:hi]).sum().backward()
    close(y, y_ref[lo:hi], "y")
    close(x.grad, dx_ref, "dx")
    close(layer.weight.grad, dw_ref, "dgamma (rank-local)")
    close(layer.bias.grad, db_ref, "dbeta (rank-local)")
    close(layer.running_mean, rm_ref, "running_mean")
    close(layer.running_var, rv_ref, "running_var")
    assert int(layer.num_batches_tracked) == 1
    stats = [torch.zeros(2 * C) for _ in range(W)]
    dist.all_gather(stats, torch.cat([layer.running_mean, layer.running_var]))
    assert all(torch.equal(s, stats[0]) for s in stats), "running statistics differ across ranks"
    # the negative control: statistics of this rank alone are rejected by the same check
    if mode == "emulate":
        loc = xg[lo:hi]
        yl = (loc - loc.mean((0, 2, 3)).view(1, C, 1, 1)) / torch.sqrt(loc.var((0, 2, 3), unbiased=False) + eps).view(1, C, 1, 1)
        try:
            close(yl * w0.view(1, C, 1, 1) + b0.view(1, C, 1, 1), y_ref[lo:hi], "local")
            raise SystemExit("the checker accepted per-rank statistics")
        except AssertionError:
            pass
    layer.eval()                                 # eval mode never synchronises: running statistics, no collective
    with torch.no_grad():
        ye = layer(xg[lo:hi].float().contiguous(memory_format=torch.channels_last) if mode == "emulate" else xg[lo:hi].float())
    close(ye, (xg[lo:hi] - layer.running_mean.double().view(1, C, 1, 1)) /
          torch.sqrt(layer.running_var.double().view(1, C, 1, 1) + eps) * w0.view(1, C, 1, 1) + b0.view(1, C, 1, 1), "eval")
print("SYNC_BN_OK rank", r)
dist.destroy_process_group()
'''


def _env():
    env = dict(os.environ)
    env.update({"OMP_NUM_THREADS": "1", "PYTHONPATH": ROOT})
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "MASTER_ADDR", "MASTER_PORT"):
        env.pop(k, None)
    return env


def _torchrun(script, n, args, port):
    return [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(n), "--master-addr", "127.0.0.1",
            "--master-port", str(port), script] + args


def test_sync_bn_gloo_world2_matches_global_fp64(tmp_path):
    script = tmp_path / "sync_bn_worker.py"
    script.write_text(WORKER)
    p = subprocess.run(_torchrun(str(script), 2, [ROOT], 29741), env=_env(), cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stdout[-3000:] + "\n" + p.stderr[-3000:]
    assert p.stdout.count("SYNC_BN_OK") == 2


def test_distributed_py_sync_bn_gloo_world2(tmp_path):
    args = ["-a", "resnet18", "-b", "8", "--synthetic", "--steps-per-epoch", "2", "--epochs", "1", "--image-size", "32",
            "--num-classes", "10", "-p", "1", "--device", "cpu", "--sync-bn", "--checkpoint-dir", str(tmp_path)]
    p = subprocess.run(_torchrun(os.path.join(ROOT, "distributed.py"), 2, args, 29743), env=_env(), cwd=ROOT, capture_output=True,
                       text=True, timeout=600)
    assert p.returncode == 0, p.stdout[-3000:] + "\n" + p.stderr[-3000:]
    ck = torch.load(os.path.join(str(tmp_path), "checkpoint.pth.tar"), weights_only=False)
    assert int(ck["state_dict"]["bn1.num_batches_tracked"]) == 2


# ------------------------------------------------------------------ conversion
def test_convert_keeps_parameters_buffers_and_keys():
    from pytorch_distributed_b200.models import create_model
    from pytorch_distributed_b200.models.resnet import BNAct, SyncBNAct, convert_sync_batchnorm
    m = create_model("resnet18", num_classes=10)
    keys = list(m.state_dict().keys())
    params = {n: p for n, p in m.named_parameters()}
    bufs = {n: b for n, b in m.named_buffers()}
    relu = {n: mod.relu for n, mod in m.named_modules() if isinstance(mod, BNAct)}
    out = convert_sync_batchnorm(m)
    assert out is m and list(m.state_dict().keys()) == keys
    assert all(p is params[n] for n, p in m.named_parameters())
    assert all(b is bufs[n] for n, b in m.named_buffers())
    converted = {n: mod for n, mod in m.named_modules() if isinstance(mod, BNAct)}
    assert set(converted) == set(relu) and all(isinstance(mod, SyncBNAct) for mod in converted.values())
    assert all(converted[n].relu == relu[n] for n in relu)


def test_convert_torch_sync_batchnorm_and_plain_batchnorm():
    from pytorch_distributed_b200.models.resnet import SyncBNAct
    from pytorch_distributed_b200.parallel import SyncBatchNorm
    seq = nn.Sequential(nn.Conv2d(3, 8, 1), nn.SyncBatchNorm(8, momentum=0.3, eps=1e-3), nn.BatchNorm2d(8), nn.ReLU())
    seq[2].eval()
    keys = list(seq.state_dict().keys())
    w = seq[1].weight
    out = SyncBatchNorm.convert_sync_batchnorm(seq)
    assert list(out.state_dict().keys()) == keys
    assert isinstance(out[1], SyncBNAct) and out[1].weight is w and out[1].momentum == 0.3 and out[1].eps == 1e-3
    assert isinstance(out[2], SyncBNAct) and not out[2].training and out[2].relu is False
    single = SyncBatchNorm.convert_sync_batchnorm(nn.BatchNorm2d(4))
    assert isinstance(single, SyncBNAct)
    # without a process group (world 1) the layer is plain BatchNorm
    x = torch.randn(4, 8, 3, 3)
    ref = nn.functional.batch_norm(x, None, None, out[1].weight, out[1].bias, True, 0.3, 1e-3)
    torch.testing.assert_close(out[1](x), ref)


def test_cast_model_keeps_sync_layers_fp32():
    from pytorch_distributed_b200.models import create_model
    from pytorch_distributed_b200.models.resnet import SyncBNAct, convert_sync_batchnorm
    from pytorch_distributed_b200.parallel.amp import cast_model
    ref = cast_model(create_model("resnet18", num_classes=10), torch.bfloat16, keep_batchnorm_fp32=True)
    m = cast_model(convert_sync_batchnorm(create_model("resnet18", num_classes=10)), torch.bfloat16, keep_batchnorm_fp32=True)
    sync = [mod for mod in m.modules() if isinstance(mod, SyncBNAct)]
    assert sync and all(mod.running_mean.dtype == torch.float32 and mod.running_var.dtype == torch.float32 for mod in sync)
    # the same dtypes as the unsynchronised fused BatchNorm layers get (16-bit affine parameters, fp32 statistics)
    assert {n: t.dtype for n, t in m.state_dict().items()} == {n: t.dtype for n, t in ref.state_dict().items()}


def test_public_names():
    from pytorch_distributed_b200 import apex
    from pytorch_distributed_b200.models.resnet import SyncBNAct
    from pytorch_distributed_b200.parallel import SyncBatchNorm, hvd
    assert SyncBatchNorm is SyncBNAct and hvd.SyncBatchNorm is SyncBNAct and issubclass(apex.parallel.SyncBatchNorm, SyncBNAct)
    m = apex.parallel.convert_syncbn_model(nn.Sequential(nn.BatchNorm2d(8)), process_group=None, channel_last=True)
    assert isinstance(m[0], SyncBNAct)


def test_subgroup_is_rejected():
    from pytorch_distributed_b200.models.resnet import SyncBNAct, convert_sync_batchnorm
    with pytest.raises(NotImplementedError, match="process_group"):
        SyncBNAct(8, process_group=object())
    with pytest.raises(NotImplementedError, match="process_group"):
        convert_sync_batchnorm(nn.BatchNorm2d(8), process_group=object())


def test_unbound_layer_raises_clearly(monkeypatch):
    import torch.distributed as dist
    from pytorch_distributed_b200.models.resnet import SyncBNAct
    from pytorch_distributed_b200.utils import dist_ops
    monkeypatch.setattr(dist, "is_initialized", lambda: True)
    monkeypatch.setattr(dist, "get_world_size", lambda group=None: 2)
    monkeypatch.setattr(dist_ops, "_default_comm", None)
    with pytest.raises(RuntimeError, match="no communicator is registered"):
        SyncBNAct(8)(torch.randn(2, 8, 3, 3))


# ------------------------------------------------------------------ command line
def test_cli_flag_and_rejections():
    from pytorch_distributed_b200 import cli, driver
    base = ["-a", "resnet18", "--device", "cpu"]
    for entry in ("distributed", "multiprocessing_distributed", "distributed_slurm_main", "apex_distributed", "horovod_distributed",
                  "dataparallel"):
        assert cli.parse_args(entry, base).sync_bn is False
        assert cli.parse_args(entry, base + ["--sync-bn"]).sync_bn is True
    from pytorch_distributed_b200.models.resnet import SyncBNAct
    m = driver.apply_sync_bn(nn.Sequential(nn.BatchNorm2d(8)), cli.parse_args("distributed", base + ["--sync-bn"]), driver.Strategy(),
                             torch.device("cpu"))
    assert isinstance(m[0], SyncBNAct)
    keep = nn.Sequential(nn.BatchNorm2d(8))
    assert driver.apply_sync_bn(keep, cli.parse_args("distributed", base), driver.Strategy(), torch.device("cpu"))[0].__class__ is nn.BatchNorm2d
    with pytest.raises(ValueError, match="DataParallel"):
        driver.apply_sync_bn(nn.Sequential(nn.BatchNorm2d(8)), cli.parse_args("dataparallel", base + ["--sync-bn"]),
                             driver.DataParallelStrategy(), torch.device("cpu"))
    for comm in ("nccl", "gloo"):
        with pytest.raises(ValueError, match="CUDA graph"):
            driver.apply_sync_bn(nn.Sequential(nn.BatchNorm2d(8)),
                                 cli.parse_args("distributed", base + ["--sync-bn", "--cuda-graph", "--comm", comm]), driver.Strategy(),
                                 torch.device("cuda"))


def test_eval_mode_never_synchronises(monkeypatch):
    import torch.distributed as dist
    from pytorch_distributed_b200.models.resnet import SyncBNAct
    from pytorch_distributed_b200.utils import dist_ops
    monkeypatch.setattr(dist, "is_initialized", lambda: True)
    monkeypatch.setattr(dist, "get_world_size", lambda group=None: 2)
    monkeypatch.setattr(dist_ops, "_default_comm", None)
    for tracked in (True, False):
        layer = SyncBNAct(8, track_running_stats=tracked).eval()
        assert layer.sync_context() is None        # no communicator needed: nothing is exchanged
        layer(torch.randn(2, 8, 3, 3))


def test_converted_torch_sync_batchnorm_takes_non_4d_inputs():
    from pytorch_distributed_b200.models.resnet import convert_sync_batchnorm
    for shape in ((6, 8), (4, 8, 5), (2, 8, 3, 3, 3)):
        m = convert_sync_batchnorm(nn.Sequential(nn.SyncBatchNorm(8)))
        x = torch.randn(*shape)
        ref = nn.functional.batch_norm(x, None, None, m[0].weight, m[0].bias, True, 0.1, 1e-5)
        torch.testing.assert_close(m(x), ref)


def test_apex_sync_batchnorm_signature():
    from pytorch_distributed_b200 import apex
    m = apex.parallel.SyncBatchNorm(8, 1e-3, 0.2, True, True, None, True, True)
    assert m.eps == 1e-3 and m.momentum == 0.2 and m.channel_last is True and m.relu is True
    x, z = torch.randn(2, 8, 3, 3), torch.randn(2, 8, 3, 3)
    ref = torch.relu(nn.functional.batch_norm(x, None, None, m.weight, m.bias, True, 0.2, 1e-3) + z)
    torch.testing.assert_close(m(x, z), ref)
    assert apex.parallel.SyncBatchNorm(8, fuse_relu=False).relu is False


def test_cuda_graph_refused_when_layers_fall_back_to_torch():
    from pytorch_distributed_b200 import cli, driver
    base = ["-a", "resnet18", "--sync-bn", "--cuda-graph", "--comm", "fused"]
    for extra in (["--no-fused-bn"], ["--no-channels-last"]):
        with pytest.raises(ValueError, match="CUDA graph"):
            driver.apply_sync_bn(nn.Sequential(nn.BatchNorm2d(8)), cli.parse_args("distributed", base + extra), driver.Strategy(),
                                 torch.device("cuda"))


@pytest.mark.parametrize("sync", [None, object()], ids=["local", "sync"])
def test_backward_slice_recycled_by_reset_is_replaced(sync):
    """A backward that runs after ``reset`` handed its slice to the next step accumulates into fresh zeros of its own."""
    from pytorch_distributed_b200.ops.bn_act import _Workspace
    from pytorch_distributed_b200.ops.sync_bn import work_len
    ws, c = _Workspace(torch.device("cpu"), capacity=4096), 64
    wl = work_len(c, sync)
    lw = ws.layer(c, sync)
    assert lw.fwd.data_ptr() == ws.buf.data_ptr() and lw.fwd.numel() == wl
    kept = lw.bwd()
    assert kept.data_ptr() == ws.buf[wl:].data_ptr() and kept.numel() >= wl
    kept.fill_(1.0)
    ws.reset()
    fresh = lw.bwd()
    assert fresh.dtype == torch.float32 and fresh.numel() == wl and not fresh.any()
    lo, hi = ws.buf.data_ptr(), ws.buf.data_ptr() + 4 * ws.buf.numel()
    assert not lo <= fresh.data_ptr() < hi
    fresh.fill_(1.0)
    assert not ws.buf.any()
