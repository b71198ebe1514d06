"""Gradient accumulation without a GPU: the ``--accum-steps`` command line, the engine's fp32 accumulation through torch ops
(library collectives) against torch DDP + ``no_sync()`` at a gloo world of 2, the epoch length of the entrypoints, and the
guard against a step before the synchronising backward."""
import json
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from pytorch_distributed_b200 import cli  # noqa: E402


def _env():
    env = dict(os.environ, OMP_NUM_THREADS="1", PYTHONPATH=ROOT)
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "MASTER_ADDR", "MASTER_PORT"):
        env.pop(k, None)
    return env


def _run(cmd, timeout=600):
    p = subprocess.run(cmd, env=_env(), cwd=ROOT, capture_output=True, text=True, timeout=timeout)
    assert p.returncode == 0, p.stdout[-3000:] + "\n" + p.stderr[-3000:]
    return p.stdout


def _torchrun(script, n, args, port):
    return [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(n), "--master-addr", "127.0.0.1",
            "--master-port", str(port), script] + args


# ------------------------------------------------------------------------------------------------ command line
def test_cli_default_and_value():
    assert cli.parse_args("distributed", []).accum_steps == 1
    assert cli.parse_args("apex_distributed", ["--accum-steps", "4"]).accum_steps == 4
    assert cli.parse_args("horovod_distributed", ["--accum-steps", "3", "--steps-per-epoch", "3"]).accum_steps == 3


@pytest.mark.parametrize("argv", [["--accum-steps", "0"], ["--accum-steps", "-2"], ["--accum-steps", "1.5"]])
def test_cli_rejects_non_positive(argv):
    with pytest.raises(SystemExit):
        cli.parse_args("distributed", argv)


def test_cli_dataparallel_rejects_accumulation():
    assert cli.parse_args("dataparallel", ["--accum-steps", "1"]).accum_steps == 1
    for n in ("2", "8"):
        with pytest.raises(SystemExit):
            cli.parse_args("dataparallel", ["--accum-steps", n])


def test_cli_steps_per_epoch_below_accum_steps():
    with pytest.raises(SystemExit):
        cli.parse_args("distributed", ["--steps-per-epoch", "3", "--accum-steps", "4"])
    assert cli.parse_args("distributed", ["--steps-per-epoch", "4", "--accum-steps", "4"]).steps_per_epoch == 4


# ------------------------------------------------------------------------------------------------ engine vs torch DDP (gloo)
PARITY = r'''
import copy, os, sys, torch, torch.distributed as dist
sys.path.insert(0, %r)
dist.init_process_group("gloo")
rank, world = dist.get_rank(), dist.get_world_size()
from pytorch_distributed_b200.models import create_model
from pytorch_distributed_b200.parallel.ddp import DistributedDataParallel
from pytorch_distributed_b200.ops.fused_sgd import FusedSGD
torch.manual_seed(3 + rank)
base = create_model("resnet18", num_classes=10)
own = DistributedDataParallel(copy.deepcopy(base), comm="gloo", bucket_cap_mb=2.0, fp32_grad_accumulation=True)
ref = torch.nn.parallel.DistributedDataParallel(copy.deepcopy(own.module))
assert len(own.engine.buckets) > 3
crit = torch.nn.CrossEntropyLoss()
oo = FusedSGD(own.parameters(), lr=0.01, momentum=0.9, weight_decay=1e-4)
orf = torch.optim.SGD(ref.parameters(), lr=0.01, momentum=0.9, weight_decay=1e-4)
K = 3
g = torch.Generator().manual_seed(11 + rank)
for it in range(2):
    xs = [torch.randn(4, 3, 32, 32, generator=g) for _ in range(K)]
    ys = [torch.randint(0, 10, (4,), generator=g) for _ in range(K)]
    for m, o in ((own, oo), (ref, orf)):
        o.zero_grad()
        for k in range(K):
            if k < K - 1:
                with m.no_sync():
                    (crit(m(xs[k]), ys[k]) / K).backward()
                if m is own:
                    assert all(p.grad is None for p in own.parameters())    # the pass lives in the fp32 accumulator
                    assert own.engine.accum_pending
                    try:
                        oo.step()
                        raise AssertionError("step() before the synchronising backward must raise")
                    except RuntimeError as e:
                        assert "no_sync" in str(e)
            else:
                (crit(m(xs[k]), ys[k]) / K).backward()
    assert not own.engine.accum_pending and not own.engine._acc.any()
    for (n, a), b in zip(own.module.named_parameters(), ref.module.parameters()):
        assert torch.allclose(a.grad, b.grad, rtol=1e-4, atol=1e-6), (it, n, (a.grad - b.grad).abs().max())
    oo.step(); orf.step()
    for (n, a), b in zip(own.module.named_parameters(), ref.module.parameters()):
        assert torch.allclose(a, b, rtol=1e-4, atol=1e-6), (it, n, (a - b).abs().max())
    with torch.no_grad():
        for a, b in zip(ref.module.parameters(), own.module.parameters()): a.copy_(b)
        for a, b in zip(ref.module.buffers(), own.module.buffers()): a.copy_(b)
flat = torch.cat([p.detach().reshape(-1) for p in own.parameters()])
lo, hi = flat.clone(), flat.clone()
dist.all_reduce(lo, op=dist.ReduceOp.MIN); dist.all_reduce(hi, op=dist.ReduceOp.MAX)
assert torch.equal(lo, hi)
print("ACCUM-PARITY-OK", rank)
dist.destroy_process_group()
'''


def test_engine_fp32_accumulation_matches_torch_ddp_no_sync_gloo(tmp_path):
    script = tmp_path / "parity.py"
    script.write_text(PARITY % ROOT)
    out = _run(_torchrun(str(script), 2, [], 29791))
    assert out.count("ACCUM-PARITY-OK") == 2


def test_fold_and_accumulate_oracle_single_process():
    """World 1, no process group: the accumulator sums in fp32 and the fold rounds into p.grad's dtype, then clears."""
    from pytorch_distributed_b200.parallel.comm import TorchCommunicator
    from pytorch_distributed_b200.parallel.ddp import GradientEngine
    torch.manual_seed(0)
    lin = torch.nn.Linear(16, 8).to(torch.bfloat16)
    eng = GradientEngine(list(lin.parameters()), TorchCommunicator(), wire_dtype="fp32", fp32_grad_accumulation=True)
    xs = [torch.randn(4, 16, dtype=torch.bfloat16) for _ in range(3)]
    grads = []
    for x in xs:
        lin.zero_grad()
        lin(x).float().square().sum().backward()
        grads.append([p.grad.clone() for p in lin.parameters()])
    lin.zero_grad()
    for k, x in enumerate(xs):
        eng.enabled = k == len(xs) - 1
        lin(x).float().square().sum().backward()
    for i, p in enumerate(lin.parameters()):
        acc = grads[0][i].float() + grads[1][i].float()
        assert torch.equal(p.grad, (acc + grads[2][i].float()).to(torch.bfloat16))
    assert not eng._acc.any() and not eng.accum_pending


# ------------------------------------------------------------------------------------------------ entrypoints
COMMON = ["-a", "resnet18", "-b", "8", "--synthetic", "--steps-per-epoch", "7", "--val-steps", "1", "--epochs", "1",
          "--image-size", "32", "--num-classes", "10", "-p", "1", "--device", "cpu", "--accum-steps", "3", "--quiet"]


def _records(path):
    with open(path) as f:
        return [json.loads(l) for l in f if l.strip()]


@pytest.mark.parametrize("script,port", [("distributed.py", 29792), ("horovod_distributed.py", 29793)])
def test_entrypoint_epoch_holds_whole_optimizer_steps(script, port, tmp_path):
    log = tmp_path / "log.jsonl"
    _run(_torchrun(os.path.join(ROOT, script), 2, COMMON + ["--checkpoint-dir", str(tmp_path), "--log-jsonl", str(log)], port))
    train = [r for r in _records(log) if r["phase"] == "train"]
    assert sorted(r["rank"] for r in train) == [0, 1]
    for r in train:
        # 7 batches capped to the largest multiple of 3: 6 micro-batches of 8 / 2 ranks = 4 images, 2 optimizer steps
        assert r["images"] == 6 * 4 and r["accum_steps"] == 3 and r["optimizer_steps"] == 2
        assert r["loss"] == r["loss"]


def test_no_accumulation_keeps_the_record(tmp_path):
    log = tmp_path / "log.jsonl"
    argv = [a for a in COMMON if a not in ("--accum-steps", "3")]
    _run(_torchrun(os.path.join(ROOT, "distributed.py"), 1, argv + ["--checkpoint-dir", str(tmp_path), "--log-jsonl", str(log)], 29794))
    train = [r for r in _records(log) if r["phase"] == "train"]
    assert train and "accum_steps" not in train[0] and train[0]["images"] == 7 * 8
