"""Synchronised BatchNorm across real GPUs (tests/mp_sync_bn_checks.py under torchrun at 2 and 8 GPUs), and the
``--sync-bn`` entrypoints running to completion.  Skipped on a machine with fewer than 2 GPUs."""
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]


def _run(script, nproc, args=(), timeout=1200):
    port = 29300 + (os.getpid() % 300)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc), "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, script)] + list(args)
    p = subprocess.run(cmd, env=dict(os.environ), cwd=ROOT, capture_output=True, text=True, timeout=timeout)
    assert p.returncode == 0, p.stdout[-4000:] + "\n" + p.stderr[-4000:]
    return p.stdout


@pytest.mark.parametrize("nproc", [2, 8])
def test_sync_bn_matches_torch_and_replays_in_a_graph(nproc):
    if torch.cuda.device_count() < nproc:
        pytest.skip("needs %d GPUs" % nproc)
    out = _run("tests/mp_sync_bn_checks.py", nproc)
    assert out.count("PASS rank") == nproc, out[-3000:]


@pytest.mark.parametrize("entry,extra", [("distributed.py", ["--cuda-graph"]), ("apex_distributed.py", [])])
def test_sync_bn_entrypoints_complete(entry, extra, tmp_path):
    out = _run(entry, 2, args=["-a", "resnet50", "-b", "32", "--synthetic", "--steps-per-epoch", "4", "--epochs", "1",
                               "--image-size", "64", "-p", "1", "--sync-bn", "--checkpoint-dir", str(tmp_path)] + extra)
    assert " * Acc@1" in out
    ck = torch.load(os.path.join(str(tmp_path), "checkpoint.pth.tar"), map_location="cpu", weights_only=False)
    assert ck["epoch"] == 1 and int(ck["state_dict"]["bn1.num_batches_tracked"]) > 0
