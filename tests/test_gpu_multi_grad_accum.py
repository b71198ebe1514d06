"""Gradient accumulation across data-parallel ranks (two or more GPUs): after several optimizer steps of ``--accum-steps 3``
every rank holds bit-identical masters and momentum and a cleared fp32 accumulator, for DDP with the per-bucket update on
and off and apex O2 fp16, at world sizes 2 and 8."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs 2 GPUs")]

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COMMON = ["-a", "resnet50", "--synthetic", "--steps-per-epoch", "6", "--val-steps", "1", "--epochs", "1", "--image-size", "96",
          "-p", "2", "--quiet", "--accum-steps", "3"]
MODES = {
    "ddp_overlap": ("distributed", []),
    "ddp_no_overlap": ("distributed", ["--no-overlap-optimizer"]),
    "apex_o2_fp16": ("apex_distributed", ["--opt-level", "O2", "--precision", "fp16"]),
}


@pytest.mark.parametrize("world", [2, 8])
@pytest.mark.parametrize("mode", list(MODES))
def test_ranks_agree_bitwise(mode, world, tmp_path):
    if torch.cuda.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    entry, extra = MODES[mode]
    env = dict(os.environ, PYTHONPATH=ROOT)
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "MASTER_ADDR", "MASTER_PORT"):
        env.pop(k, None)
    out = tmp_path / "out"
    port = 29811 + 2 * list(MODES).index(mode) + (world == 8)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world), "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "tests", "mp_grad_accum_checks.py"), str(out), entry,
           "-b", str(32 * world), "--checkpoint-dir", str(tmp_path)] + COMMON + extra
    p = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-3000:] + "\n" + p.stderr[-3000:]
    ranks = [torch.load(out / ("rank%d.pt" % r), weights_only=False) for r in range(world)]
    assert len(ranks[0]["masters"]) == 161
    for r in ranks:
        assert r["fp32_accum"] and r["acc_clear"] and not r["pending"]
    for r in ranks[1:]:
        for a, b in zip(ranks[0]["masters"] + ranks[0]["momenta"], r["masters"] + r["momenta"]):
            assert torch.equal(a, b)
