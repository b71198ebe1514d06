"""Synchronised BatchNorm cost at the ResNet-50 channel counts.

    python tools/sync_bn_bench.py [--batch 256] [--iters 50] [--steps 20] [--gpus N] [--out result.json]

* per_layer_world1: with CUDA events over many launches, the training-mode forward of ``bn_act`` at each ResNet-50 BN
  shape unsynchronised and through the exchange kernel (``csrc/sync_bn.cu``) of a one-rank handle: the exchange
  kernel's own cost in place of ``combine_partials``, with no peer to wait for.
* multi_gpu (two or more GPUs; torchrun over this file): the same per-layer timing through the fused communicator of
  all ranks (the cross-GPU exchange latency), and ResNet-50 bf16 images/s of DDP training steps with and without
  ``--sync-bn``.  With one GPU it is reported as not measured.
The card name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# (C, H = W) of the ResNet-50 BatchNorm layers at 224 x 224 input
SHAPES = [(64, 112), (64, 56), (256, 56), (128, 28), (512, 28), (256, 14), (1024, 14), (512, 7), (2048, 7)]


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return {"nvidia_smi": q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unavailable",
            "torch_name": torch.cuda.get_device_name(0)}


def time_ms(fn, iters: int) -> float:
    for _ in range(3):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def per_layer(batch: int, iters: int) -> list:
    from pytorch_distributed_b200 import _ext
    from pytorch_distributed_b200.parallel import plan as P
    M = _ext.lib()
    header = P.round_up(M.SIGNAL_PAD_BYTES, 128 << 10)
    nbytes = P.round_up(header + M.SYNC_BN_AREA_BYTES, 1 << 16)
    buf = torch.zeros(nbytes, dtype=torch.uint8, device="cuda")
    arena = M.SymmArena.from_pointers(0, 1, [buf.data_ptr()], 0, nbytes, 0)
    calls = torch.zeros(M.MAX_BLOCKS, dtype=torch.int32, device="cuda")
    handle = arena.sync_bn(0, header, calls.data_ptr())
    out = []
    for c, hw in SHAPES:
        x = torch.randn(batch, c, hw, hw, device="cuda").to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
        w, b = torch.ones(c, device="cuda"), torch.zeros(c, device="cuda")
        rm, rv = torch.zeros(c, device="cuda"), torch.ones(c, device="cuda")
        plain, synced = torch.zeros(2 * c, device="cuda"), torch.zeros(4 * c + 4, device="cuda")
        t0 = time_ms(lambda: M.bn_act_forward(x, None, w, b, rm, rv, None, True, 0.1, 1e-5, True, False, plain, False), iters)
        t1 = time_ms(lambda: M.bn_act_forward(x, None, w, b, rm, rv, None, True, 0.1, 1e-5, True, False, synced, False, handle), iters)
        out.append({"C": c, "HW": hw, "batch": batch, "fwd_ms": round(t0, 4), "fwd_sync_world1_ms": round(t1, 4),
                    "exchange_overhead_us": round(1000 * (t1 - t0), 2)})
    assert arena.status() == 0
    return out


def _worker(batch: int, iters: int, steps: int) -> None:
    """One rank of the multi-GPU measurement (under torchrun): per-layer exchange latency through the fused communicator
    and ResNet-50 images/s with and without synchronised BatchNorm.  Rank 0 prints one JSON line."""
    import torch.distributed as dist
    from pytorch_distributed_b200 import _ext, cli, driver
    from pytorch_distributed_b200.models import create_model
    from pytorch_distributed_b200.ops.sync_bn import SyncContext
    from pytorch_distributed_b200.parallel.comm import FusedCommunicator
    local = int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    world, rank = dist.get_world_size(), dist.get_rank()
    M = _ext.lib()
    comm = FusedCommunicator(device=dev)
    handle = SyncContext.for_communicator(comm).native
    layers = []
    for c, hw in SHAPES:
        x = torch.randn(batch, c, hw, hw, device=dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
        w, b = torch.ones(c, device=dev), torch.zeros(c, device=dev)
        rm, rv = torch.zeros(c, device=dev), torch.ones(c, device=dev)
        plain, synced = torch.zeros(2 * c, device=dev), torch.zeros(4 * c + 4, device=dev)
        dist.barrier()
        t0 = time_ms(lambda: M.bn_act_forward(x, None, w, b, rm, rv, None, True, 0.1, 1e-5, True, False, plain, False), iters)
        dist.barrier()
        t1 = time_ms(lambda: M.bn_act_forward(x, None, w, b, rm, rv, None, True, 0.1, 1e-5, True, False, synced, False, handle), iters)
        layers.append({"C": c, "HW": hw, "batch_per_gpu": batch, "fwd_ms": round(t0, 4), "fwd_sync_ms": round(t1, 4),
                       "exchange_us": round(1000 * (t1 - t0), 2)})
    comm.check()
    e2e = {}
    for tag, extra in (("plain", []), ("sync_bn", ["--sync-bn"])):
        args = cli.parse_args("distributed", ["-a", "resnet50", "-b", str(batch * world), "--synthetic", "--quiet"] + extra)
        st = driver.Strategy()
        model = driver.apply_sync_bn(create_model("resnet50"), args, st, dev)
        model, opt = st.build(model, args, dev, local)
        crit = torch.nn.CrossEntropyLoss().to(dev)
        x = torch.randn(batch, 3, 224, 224, device=dev).to(st.input_dtype).contiguous(memory_format=torch.channels_last)
        t = torch.randint(0, 1000, (batch,), device=dev)

        def one():
            opt.zero_grad()
            st.backward(crit(st.forward(model, x).float(), t), opt)
            opt.step()
        for _ in range(5):
            one()
        dist.barrier()
        ms = time_ms(one, steps)
        e2e[tag] = {"ms_per_step": round(ms, 3), "images_per_s": round(world * batch * 1000.0 / ms, 1)}
    if rank == 0:
        print(json.dumps({"gpus": world, "per_layer": layers, "end_to_end": e2e}), flush=True)
    dist.destroy_process_group()


def multi_gpu(gpus: int, batch: int, iters: int, steps: int) -> dict:
    """The per-layer exchange latency and the end-to-end images/s at ``gpus`` GPUs (torchrun over this file)."""
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(gpus), "--master-addr", "127.0.0.1",
           "--master-port", "29517", os.path.abspath(__file__), "--worker", "--batch", str(batch), "--iters", str(iters),
           "--steps", str(steps)]
    p = subprocess.run(cmd, capture_output=True, text=True, cwd=ROOT)
    lines = [ln for ln in p.stdout.splitlines() if ln.startswith("{")]
    if p.returncode != 0 or not lines:
        raise SystemExit("multi-GPU measurement failed:\n" + p.stdout[-2000:] + p.stderr[-3000:])
    return json.loads(lines[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--gpus", type=int, default=None, help="GPUs of the multi-GPU measurement (default: all visible)")
    ap.add_argument("--worker", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sync_bn_bench needs a GPU")
    if a.worker:
        return _worker(a.batch, a.iters, a.steps)
    gpus = a.gpus or torch.cuda.device_count()
    res = {"card": card(), "gpus": gpus, "per_layer_world1": per_layer(a.batch, a.iters)}
    if gpus >= 2:
        res["multi_gpu"] = multi_gpu(gpus, a.batch, a.iters, a.steps)
    else:
        res["multi_gpu"] = "not measured: one GPU (the cross-GPU exchange and --sync-bn images/s need two or more)"
    txt = json.dumps(res, indent=1)
    print(txt)
    if a.out:
        with open(a.out, "w") as f:
            f.write(txt + "\n")


if __name__ == "__main__":
    main()
