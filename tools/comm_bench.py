"""Micro-benchmarks of the fused collectives (K1..K5) against NCCL and against their link rooflines.

    python -m torch.distributed.run --nproc-per-node 8 --master-addr 127.0.0.1 tools/comm_bench.py [sections...] > comm_bench_8gpu.md
    python tools/comm_bench.py local          # single process, all visible GPUs: K2' push / K5 reduce-to-caller (DataParallel engine)

Sections (default: all multi-process ones): k1 k1small ctas k2 k4.
Every number: device time (CUDA events on the launching stream), max over ranks, median of `reps` after warm-ups, with a
barrier + synchronize between repetitions.  Rooflines:
  all-reduce  bus bandwidth 2(W-1)/W * wire_bytes / t   vs 450 GB/s, NVLink 4 per direction per GPU (H100 SXM data sheet)
  broadcast / push / reduce-to-root   wire_bytes / t     vs the same 450 GB/s per direction per GPU (root egress or ingress)
"""
import os
import statistics
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BUS_REF, DIR_REF = 450.0, 450.0


def timed(fn, reps, device, sync, reduce_max=True):
    times = []
    for _ in range(reps):
        sync()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize(device)
        t = torch.tensor([e0.elapsed_time(e1)], device=device)
        if reduce_max and dist.is_initialized():
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        times.append(float(t.item()))
    return statistics.median(times)


def section_k1(comm_factory, dev, world, sync, say):
    """K1 at the sizes DDP sends: source dtype == wire dtype == bf16 (the headline config), fp32 -> bf16 cast-pack, and the
    in-arena ("prepacked", gradient_as_bucket_view) variant that has no pack pass at all."""
    from pytorch_distributed_b200.parallel.comm import KIND_TWO_SHOT
    say("\n## K1 two-shot all-reduce (one bucket per launch)\n")
    say("| wire MB | elements | src->wire | NVLS pack us | NVLS in-arena us | P2P pack us | NCCL us | best busbw GB/s | frac of 450 | in-arena busbw | frac | NCCL busbw |")
    say("|---:|---:|---|---:|---:|---:|---:|---:|---:|---:|---:|---:|")
    for n in (1 << 19, 1 << 20, 1 << 21, 1 << 22, 6_000_000, 1 << 23, 1 << 24, 25_600_000, 1 << 26):
        comm = comm_factory()
        for src_dt, wire, wbytes in ((torch.bfloat16, "bf16", 2), (torch.float32, "bf16", 2), (torch.float32, "fp32", 4)):
            src = torch.randn(n, device=dev).to(src_dt)
            plan = comm.make_plan([n], wire)
            arena_view = plan.arena_tensor()[:n]
            flat = src.clone() if wire == "fp32" else src.to(torch.bfloat16).clone()

            def fused(nvls, prepacked=False):
                comm.run(plan, [arena_view if prepacked else src], KIND_TWO_SHOT, comm.misc_channel, scale=1.0 / world, writeback=False,
                         nvls=nvls, prepacked=prepacked)

            def nccl():
                flat.div_(world)
                dist.all_reduce(flat)

            for _ in range(3):
                fused(True); fused(False); fused(True, True); nccl()
            t_nvls = timed(lambda: fused(True), 7, dev, sync) if comm.nvls else float("nan")
            t_pre = timed(lambda: fused(comm.nvls, True), 7, dev, sync)
            t_p2p = timed(lambda: fused(False), 7, dev, sync)
            t_nccl = timed(nccl, 7, dev, sync)
            best = min(t for t in (t_nvls, t_p2p) if t == t)
            f = 2 * (world - 1) / world * n * wbytes / 1e9
            say("| %.1f | %d | %s->%s | %.1f | %.1f | %.1f | %.1f | %.0f | %.2f | %.0f | %.2f | %.0f |" % (
                n * wbytes / 2 ** 20, n, str(src_dt).replace("torch.", ""), wire, t_nvls * 1e3, t_pre * 1e3, t_p2p * 1e3, t_nccl * 1e3,
                f / (best * 1e-3), f / (best * 1e-3) / BUS_REF, f / (t_pre * 1e-3), f / (t_pre * 1e-3) / BUS_REF, f / (t_nccl * 1e-3)))
        del comm


def section_k1small(comm_factory, dev, world, sync, say):
    """One-shot vs two-shot crossover (sets comm.ONE_SHOT_MAX_BYTES) - bf16 sources and wire."""
    from pytorch_distributed_b200.parallel.comm import KIND_ONE_SHOT, KIND_TWO_SHOT
    say("\n## K1b one-shot vs K1 two-shot (bf16, latency-bound sizes)\n")
    say("| wire KB | one-shot us | two-shot us | NCCL us |\n|---:|---:|---:|---:|")
    comm = comm_factory()
    for n in (1 << 10, 1 << 13, 1 << 15, 1 << 16, 1 << 17, 1 << 18, 1 << 19, 1 << 20, 1 << 21):
        src = torch.randn(n, device=dev).bfloat16()
        p1 = comm.make_plan([n], "bf16", double_buffer=True)
        p2 = comm.make_plan([n], "bf16")
        flat = src.clone()
        f1 = lambda: comm.run(p1, [src], KIND_ONE_SHOT, comm.misc_channel, scale=1.0 / world, writeback=False)      # noqa: E731
        f2 = lambda: comm.run(p2, [src], KIND_TWO_SHOT, comm.misc_channel, scale=1.0 / world, writeback=False)      # noqa: E731

        def nccl():
            flat.div_(world)
            dist.all_reduce(flat)

        for _ in range(3):
            f1(); f2(); nccl()
        say("| %.0f | %.1f | %.1f | %.1f |" % (n * 2 / 1024, timed(f1, 9, dev, sync) * 1e3, timed(f2, 9, dev, sync) * 1e3, timed(nccl, 9, dev, sync) * 1e3))


def section_ctas(comm_factory, dev, world, sync, say):
    from pytorch_distributed_b200.parallel.comm import KIND_TWO_SHOT
    say("\n## K1 two-shot NVLS by CTA count (bf16 source and wire)\n")
    say("| wire MB | 8 CTAs us | 16 CTAs us | 32 CTAs us | 64 CTAs us |\n|---:|---:|---:|---:|---:|")
    for n in (1 << 20, 1 << 22, 1 << 24, 1 << 26):
        comm = comm_factory()
        src = torch.randn(n, device=dev).bfloat16()
        row = []
        for c in (8, 16, 32, 64):
            pl = comm.make_plan([n], "bf16", max_ctas=c)
            fn = lambda pl=pl: comm.run(pl, [src], KIND_TWO_SHOT, comm.misc_channel, scale=1.0 / world, writeback=False)      # noqa: E731
            for _ in range(3):
                fn()
            row.append(timed(fn, 7, dev, sync) * 1e3)
        say("| %.1f | %s |" % (n * 2 / 2 ** 20, " | ".join("%.1f" % x for x in row)))
        del comm


def section_k2(comm_factory, dev, world, sync, say):
    from pytorch_distributed_b200.models import create_model
    import contextlib
    import io
    with contextlib.redirect_stdout(io.StringIO()):
        model = create_model("resnet50").to(dev)
    comm = comm_factory()
    params = [p.data for p in model.parameters()]
    bufs = [b for b in model.buffers() if b.is_floating_point()]
    big = [torch.randn(1 << 24, device=dev)]
    say("\n## K2 broadcast from rank 0 (multicast store; root egress = N bytes)\n")
    say("| tensors | MB | fused us | GB/s (root egress) | frac of 450 | NCCL (flatten + broadcast + unflatten) us |\n|---|---:|---:|---:|---:|---:|")
    for name, ts_ in (("161 ResNet-50 parameters fp32", params), ("106 BN buffers fp32", bufs), ("1 tensor fp32", big)):
        def fused_b(ts_=ts_):
            comm.broadcast_(ts_, root=0)

        def nccl_b(ts_=ts_):
            flat = torch._utils._flatten_dense_tensors(ts_)
            dist.broadcast(flat, src=0)
            for t, f in zip(ts_, torch._utils._unflatten_dense_tensors(flat, ts_)):
                t.copy_(f)

        for _ in range(3):
            fused_b(); nccl_b()
        tf, tn = timed(fused_b, 7, dev, sync), timed(nccl_b, 7, dev, sync)
        nb = sum(t.numel() * t.element_size() for t in ts_)
        say("| %s | %.2f | %.1f | %.0f | %.2f | %.1f |" % (name, nb / 2 ** 20, tf * 1e3, nb / (tf * 1e-3) / 1e9, nb / (tf * 1e-3) / 1e9 / DIR_REF, tn * 1e3))


def section_k4(comm_factory, dev, world, sync, say):
    from pytorch_distributed_b200.utils.meters import accuracy
    comm = comm_factory()
    logits = torch.randn(256, 1000, device=dev).bfloat16()
    target = torch.randint(0, 1000, (256,), device=dev)
    loss = torch.tensor(1.0, device=dev)
    out = torch.zeros(4, device=dev)

    def k4():
        comm.metrics(logits, target, loss, out)

    def ref():
        a1, a5 = accuracy(logits, target, (1, 5))
        dist.barrier()
        for t in (loss.clone(), a1, a5):
            dist.all_reduce(t)
            t /= world

    def k3():
        comm.barrier()

    for _ in range(5):
        k4(); ref(); k3()
    say("\n## Metric synchronisation per iteration (logits 256x1000 bf16) and the bare barrier\n")
    say("| path | device us |\n|---|---:|")
    say("| K4 `metrics_kernel` (top-k counting + LL all-reduce, 1 launch) | %.1f |" % (timed(k4, 15, dev, sync) * 1e3))
    say("| reference sequence: accuracy() + barrier + 3 x (clone, all_reduce, div) via NCCL | %.1f |" % (timed(ref, 15, dev, sync) * 1e3))
    say("| K3 `barrier_kernel` (signal pad, 1 CTA) | %.1f |" % (timed(k3, 15, dev, sync) * 1e3))
    comm.check()


def main_multi(sections):
    rank, local, world = int(os.environ["RANK"]), int(os.environ["LOCAL_RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    from pytorch_distributed_b200.parallel.comm import FusedCommunicator

    def factory():
        return FusedCommunicator(device=dev, arena_bytes=1 << 30)     # plans are never freed: sections take a fresh arena

    def sync():
        torch.cuda.synchronize(dev)
        dist.barrier()

    say = (lambda *a: print(*a, flush=True)) if rank == 0 else (lambda *a: None)
    probe = factory()
    say("# Fused collectives vs NCCL, %d x %s (symm=%s, nvls=%s)\n" % (world, torch.cuda.get_device_name(), probe.symm_backend, probe.nvls))
    say("Device-timed (CUDA events), max over ranks, median of 7 after 3 warm-ups.")
    del probe
    table = {"k1": section_k1, "k1small": section_k1small, "ctas": section_ctas, "k2": section_k2, "k4": section_k4}
    for s in sections or ["k1", "k1small", "ctas", "k2", "k4"]:
        table[s](factory, dev, world, sync, say)
    dist.barrier()
    dist.destroy_process_group()


def main_local():
    """Single-process engine kernels (events order the devices): K2' push (pack + multicast of the parameters to every replica's
    arena), replica unpack, K5 pack + reduce-to-caller (in-switch sum pulled by the root)."""
    from pytorch_distributed_b200.parallel.comm import KIND_PACK, KIND_PUSH, KIND_REDUCE, KIND_UNPACK
    from pytorch_distributed_b200.parallel.dp import LocalCommunicator, _TensorSet
    ndev = torch.cuda.device_count()
    devices = list(range(ndev))
    comm = LocalCommunicator(devices, 1 << 30)
    print("# Single-process engine kernels over %d x %s (nvls=%s)\n" % (ndev, torch.cuda.get_device_name(), comm.nvls))
    print("Device time on the ROOT's stream (CUDA events), median of 7 after 3 warm-ups; bf16 values.\n")
    print("| MB | K2' push us | GB/s | frac of 450 | replica unpack us | K5 pack us | K5 reduce-to-root us | GB/s (root ingress) | frac of 450 |")
    print("|---:|---:|---:|---:|---:|---:|---:|---:|---:|")
    root = torch.device("cuda", 0)

    def sync():
        for d in devices:
            torch.cuda.synchronize(d)

    for n in (1 << 20, 1 << 22, 12_800_000, 25_600_000, 1 << 26):
        per_dev = []
        for d in devices:
            with torch.cuda.device(d):
                per_dev.append([torch.randn(n, device="cuda:%d" % d).bfloat16()])
        ts = _TensorSet(comm, per_dev, "bf16")

        def run_root(kind):
            with torch.cuda.device(0):
                ts.launch(kind, 0, writeback=False)

        def run_dev1(kind):
            with torch.cuda.device(devices[-1]):
                ts.launch(kind, len(devices) - 1)

        res = {}
        for name, fn, dev_ in (("push", lambda: run_root(KIND_PUSH), root), ("unpack", lambda: run_dev1(KIND_UNPACK), torch.device("cuda", devices[-1])),
                               ("pack", lambda: run_root(KIND_PACK), root), ("reduce", lambda: run_root(KIND_REDUCE), root)):
            with torch.cuda.device(dev_):
                for _ in range(3):
                    fn()
                res[name] = timed(fn, 7, dev_, sync, reduce_max=False) * 1e3
        nb = n * 2
        print("| %.1f | %.1f | %.0f | %.2f | %.1f | %.1f | %.1f | %.0f | %.2f |" % (
            nb / 2 ** 20, res["push"], nb / res["push"] / 1e3, nb / res["push"] / 1e3 / DIR_REF, res["unpack"], res["pack"], res["reduce"],
            nb / res["reduce"] / 1e3, nb / res["reduce"] / 1e3 / DIR_REF), flush=True)


if __name__ == "__main__":
    args = sys.argv[1:]
    if args and args[0] == "local":
        main_local()
    else:
        main_multi(args)
