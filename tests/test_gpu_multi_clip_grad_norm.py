"""Gradient clipping across data-parallel ranks (two or more GPUs): after several clipped steps every rank holds bit-identical
fp32 master weights, for DDP, apex O2 fp16 and horovod.  The weights are read through ``--model-ema --model-ema-decay 0``,
whose average is a bit-exact copy of the masters after every step (tests/mp_model_ema_checks.py writes it per rank)."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs 2 GPUs")]

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COMMON = ["-a", "resnet50", "--synthetic", "--steps-per-epoch", "4", "--val-steps", "1", "--epochs", "1", "--image-size", "96",
          "-p", "2", "--quiet", "--model-ema", "--model-ema-decay", "0", "--clip-grad-norm", "0.5"]
MODES = {
    "ddp": ("distributed", []),
    "ddp_graph": ("distributed", ["--cuda-graph"]),
    "apex_o2_fp16": ("apex_distributed", ["--opt-level", "O2", "--precision", "fp16"]),
    "horovod": ("horovod_distributed", []),
}


@pytest.mark.parametrize("mode", list(MODES))
def test_ranks_agree_bitwise(mode, tmp_path):
    entry, extra = MODES[mode]
    world = 2
    env = dict(os.environ, PYTHONPATH=ROOT)
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "MASTER_ADDR", "MASTER_PORT"):
        env.pop(k, None)
    out = tmp_path / "out"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world), "--master-addr", "127.0.0.1",
           "--master-port", str(29841 + list(MODES).index(mode)), os.path.join(ROOT, "tests", "mp_model_ema_checks.py"), str(out),
           entry, "-b", str(32 * world), "--checkpoint-dir", str(tmp_path)] + COMMON + extra
    p = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-3000:] + "\n" + p.stderr[-3000:]
    ranks = [torch.load(out / ("rank%d.pt" % r), weights_only=False)["ema"] for r in range(world)]
    from pytorch_distributed_b200.models import create_model
    params = {n for n, _ in create_model("resnet50").named_parameters()}
    for r in ranks[1:]:
        for k in params:
            assert torch.equal(ranks[0][k], r[k]), k
