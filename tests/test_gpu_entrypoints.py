"""Every entrypoint runs a short synthetic job on the visible GPUs (2 when available)."""
import os
import re
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]
COMMON = ["-a", "resnet18", "-b", "32", "--synthetic", "--steps-per-epoch", "4", "--val-steps", "2", "--epochs", "1", "--image-size", "64",
          "-p", "1"]


def _run(cmd, timeout=900, extra_env=None):
    env = dict(os.environ)
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "MASTER_ADDR", "MASTER_PORT"):
        env.pop(k, None)
    env.update(extra_env or {})
    p = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=timeout)
    assert p.returncode == 0, p.stdout[-3000:] + "\n" + p.stderr[-5000:]
    return p.stdout


def _torchrun(script, n, args, port):
    return [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(n), "--master-addr", "127.0.0.1",
            "--master-port", str(port), os.path.join(ROOT, script)] + args


def _finite_losses(out):
    # training losses: finite and sane; validation loss of a barely trained, randomly initialised net in eval mode (running
    # statistics a few steps old) can be huge for deep models - only require it to be a number
    vals = [float(x) for line in out.splitlines() if line.startswith("Epoch:") for x in re.findall(r"Loss (\d\.\d+e[+-]\d+)", line)]
    assert vals and all(v == v and v < 1e3 for v in vals), vals[:8]
    test = [float(x) for line in out.splitlines() if line.startswith("Test:") for x in re.findall(r"Loss (\d\.\d+e[+-]\d+)", line)]
    assert all(v == v and v != float("inf") for v in test), test[:4]


@pytest.mark.parametrize("opt_level,prec", [("O1", "fp16"), ("O2", "fp16"), ("O2", "bf16"), ("O0", "fp32")])
def test_apex_entrypoint(tmp_path, opt_level, prec):
    out = _run(_torchrun("apex_distributed.py", 2, COMMON + ["--opt-level", opt_level, "--precision", prec, "--lr", "0.01",
                                                             "--checkpoint-dir", str(tmp_path)], 29801))
    assert out.count(" * Acc@1") == 2
    _finite_losses(out)
    ck = torch.load(os.path.join(str(tmp_path), "checkpoint.pth.tar"), map_location="cpu", weights_only=False)
    assert all(v.dtype == torch.float32 for v in ck["state_dict"].values() if v.is_floating_point())


def test_horovod_entrypoint_torchrun(tmp_path):
    out = _run(_torchrun("horovod_distributed.py", 2, COMMON + ["--lr", "0.01", "--checkpoint-dir", str(tmp_path)], 29802))
    assert out.count(" * Acc@1") == 2
    _finite_losses(out)


def test_horovod_entrypoint_selfspawn(tmp_path):
    out = _run([sys.executable, os.path.join(ROOT, "horovod_distributed.py")] + COMMON +
               ["--world-size", "2", "--lr", "0.01", "--checkpoint-dir", str(tmp_path)])
    assert out.count(" * Acc@1") == 2


def test_multiprocessing_entrypoint(tmp_path):
    out = _run([sys.executable, os.path.join(ROOT, "multiprocessing_distributed.py")] + COMMON +
               ["--world-size", "2", "--lr", "0.01", "--checkpoint-dir", str(tmp_path)])
    assert out.count(" * Acc@1") == 2
    _finite_losses(out)


def test_distributed_entrypoint_cuda_graph_two_gpus(tmp_path):
    out = _run(_torchrun("distributed.py", 2, COMMON[:6] + ["8"] + COMMON[7:] + ["--cuda-graph", "--lr", "0.01", "--checkpoint-dir", str(tmp_path)], 29805))
    assert out.count(" * Acc@1") == 2
    _finite_losses(out)


@pytest.mark.parametrize("comm", ["nccl"])
def test_distributed_entrypoint_library_comm(tmp_path, comm):
    out = _run(_torchrun("distributed.py", 2, COMMON + ["--comm", comm, "--lr", "0.01", "--checkpoint-dir", str(tmp_path)], 29803))
    assert out.count(" * Acc@1") == 2


@pytest.mark.parametrize("prec", ["bf16", "fp32"])
def test_dataparallel_entrypoint(tmp_path, prec):
    out = _run([sys.executable, os.path.join(ROOT, "dataparallel.py")] + COMMON + ["--gpus", "0,1", "--precision", prec, "--lr", "0.01",
                                                                                 "--checkpoint-dir", str(tmp_path)])
    assert out.count(" * Acc@1") == 1 and os.path.exists(tmp_path / "dataparallel.csv")
    _finite_losses(out)


DP_PARITY = r'''
import copy, sys, torch
sys.path.insert(0, %r)
from pytorch_distributed_b200.models import create_model
from pytorch_distributed_b200.parallel.dp import DataParallel
from pytorch_distributed_b200.ops.fused_sgd import FusedSGD
torch.backends.cudnn.allow_tf32 = False; torch.backends.cuda.matmul.allow_tf32 = False
torch.manual_seed(0)
import os
n = min(torch.cuda.device_count(), int(os.environ.get("PTD_TEST_DP_GPUS", "2")))     # validated width; raise via the env for wider boxes
base = create_model("resnet18", num_classes=10, fused_bn=False).cuda(0)
ref = torch.nn.DataParallel(copy.deepcopy(base), device_ids=list(range(n)), output_device=0)
own = DataParallel(copy.deepcopy(base), device_ids=list(range(n)), output_device=0, wire_dtype="fp32")
print("nvls", own.engine.comm.nvls, own.engine.comm.arena.mc_error)
crit = torch.nn.CrossEntropyLoss()
o_ref = torch.optim.SGD(ref.parameters(), lr=0.05, momentum=0.9, weight_decay=1e-4)
o_own = FusedSGD(own.parameters(), lr=0.05, momentum=0.9, weight_decay=1e-4)
assert o_own.is_flat
for it in range(6):      # iterations 0-1 eager (replica threads), 2 captures the per-replica CUDA graphs, 3-5 replay them
    x = torch.randn(8 * n, 3, 64, 64, device="cuda:0"); y = torch.randint(0, 10, (8 * n,), device="cuda:0")
    with torch.no_grad():
        for a, b in zip(ref.module.parameters(), own.module.parameters()): a.copy_(b)
        for a, b in zip(ref.module.buffers(), own.module.buffers()): a.copy_(b)
        if it > 0:
            for a, b in zip(ref.module.parameters(), own.module.parameters()):
                o_ref.state[a]["momentum_buffer"].copy_(o_own.state[b]["momentum_buffer"])
    outs = []
    for m, o in ((ref, o_ref), (own, o_own)):
        o.zero_grad(); out = m(x); outs.append(out.detach()); crit(out, y).backward(); o.step()
    torch.cuda.synchronize()
    assert torch.allclose(outs[0], outs[1], rtol=1e-4, atol=1e-5), (outs[0] - outs[1]).abs().max()
    arena = own.engine.grad_arena()
    for i, ((nm, a), b) in enumerate(zip(ref.module.named_parameters(), own.engine.params)):
        off = own.engine.param_elem_off[i]
        g = arena[off:off + b.numel()].view_as(a)
        assert torch.allclose(g, a.grad, rtol=1e-3, atol=1e-6), (it, nm, (g - a.grad).abs().max().item(), a.grad.abs().max().item())
        assert torch.allclose(a, b, rtol=1e-4, atol=1e-6), (it, nm, (a - b).abs().max().item())
assert own._graphed is not None and len(own._graphed) == n, "replicas were not graphed"
# eval / other batch size fall back to the eager forward
own.eval()
with torch.no_grad():
    e = own(torch.randn(3 * n, 3, 64, 64, device="cuda:0"))
assert e.shape[0] == 3 * n and torch.isfinite(e).all()
print("DP-PARITY-OK")
'''


def test_dataparallel_matches_torch_dataparallel(tmp_path):
    script = tmp_path / "dp_parity.py"
    script.write_text(DP_PARITY % ROOT)
    out = _run([sys.executable, str(script)])
    assert "DP-PARITY-OK" in out


R50 = ["-a", "resnet50", "-b", "16", "--synthetic", "--steps-per-epoch", "6", "--val-steps", "1", "--epochs", "1", "--image-size", "64", "-p", "1",
       "--lr", "0.01"]


def test_resnet50_bottleneck_paths_ddp_graph_two_gpus(tmp_path):
    """ResNet-50 exercises the wgmma conv1x1+BN-statistics GEMM inside the captured two-stream step."""
    out = _run(_torchrun("distributed.py", 2, R50 + ["--cuda-graph", "--checkpoint-dir", str(tmp_path)], 29806))
    assert out.count(" * Acc@1") == 2
    _finite_losses(out)


def test_resnet50_dataparallel_two_gpus(tmp_path):
    """One process, two devices, replica threads: per-device kernel attributes of the wgmma GEMM path."""
    out = _run([sys.executable, os.path.join(ROOT, "dataparallel.py")] + R50 + ["--gpus", "0,1", "--checkpoint-dir", str(tmp_path)])
    assert out.count(" * Acc@1") == 1
    _finite_losses(out)
