"""ModelEma across data-parallel ranks (two or more GPUs): after several steps every rank holds bit-identical parameter
averages, for DDP with the per-bucket update on and off, apex O2 fp16 and horovod.  Buffer averages agree too under our
DistributedDataParallel, which broadcasts rank 0's buffers every step; apex's DDP and horovod leave each rank its own
running statistics (as apex and horovod do), and so are their averages."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs 2 GPUs")]

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COMMON = ["-a", "resnet50", "--synthetic", "--steps-per-epoch", "4", "--val-steps", "1", "--epochs", "1", "--image-size", "96",
          "-p", "2", "--quiet", "--model-ema", "--model-ema-decay", "0.9"]
MODES = {
    "ddp_overlap": ("distributed", [], True),
    "ddp_no_overlap": ("distributed", ["--no-overlap-optimizer"], True),
    "apex_o2_fp16": ("apex_distributed", ["--opt-level", "O2", "--precision", "fp16"], False),
    "horovod": ("horovod_distributed", [], False),
}


@pytest.mark.parametrize("mode", list(MODES))
def test_ranks_agree_bitwise(mode, tmp_path):
    entry, extra, buffers_agree = MODES[mode]
    world = 2
    env = dict(os.environ, PYTHONPATH=ROOT)
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "MASTER_ADDR", "MASTER_PORT"):
        env.pop(k, None)
    out = tmp_path / "out"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world), "--master-addr", "127.0.0.1",
           "--master-port", str(29821 + list(MODES).index(mode)), os.path.join(ROOT, "tests", "mp_model_ema_checks.py"), str(out),
           entry, "-b", str(32 * world), "--checkpoint-dir", str(tmp_path)] + COMMON + extra
    p = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-3000:] + "\n" + p.stderr[-3000:]
    ranks = [torch.load(out / ("rank%d.pt" % r), weights_only=False)["ema"] for r in range(world)]
    from pytorch_distributed_b200.models import create_model
    params = {n for n, _ in create_model("resnet50").named_parameters()}
    for r in ranks[1:]:
        assert r.keys() == ranks[0].keys()
        for k in r:
            if k in params or buffers_agree:
                assert torch.equal(ranks[0][k], r[k]), k
