"""Headline benchmark: ResNet-50 training images/sec on N H100s (BASELINE.json metric / config).

    python bench.py --gpus 1 --steps 20 --warmup 5
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 --master-port P bench.py --gpus 8 ...
    python bench.py --impl reference ...        (the unmodified reference scripts from oracle/_ref, stock code path)

Own arm: the public training path of this repo (driver.Strategy.build -> DistributedDataParallel + FusedSGD, the
DataPrefetcher, the MetricPipeline) - the same objects `distributed.py` uses.
  value       device-timed (CUDA events, max over ranks) images/s of K full training steps
              (forward + loss + metric kernel + backward with fused all-reduce + optimizer), inputs already on the
              device (4 distinct 256-image bf16 NHWC batches = 154 MB > the 50 MB L2; activations are GBs).
  e2e.value   the same loop fed from PINNED HOST memory through the prefetcher (H2D of every batch inside the timed
              region) with the step's reduced loss/accuracy copied back to the host every step.
Synthetic data, random-init weights, weak scaling (256 images per GPU).
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import threading
import time

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

METRIC = "ResNet-50 images/sec (device-timed, max over ranks)"


def parse():
    p = argparse.ArgumentParser()
    p.add_argument("--gpus", type=int, default=1)
    p.add_argument("--steps", type=int, default=20)
    p.add_argument("--warmup", type=int, default=5)
    p.add_argument("--impl", default="own", choices=["own", "reference"])
    p.add_argument("--arch", default="resnet50")
    p.add_argument("--batch-per-gpu", type=int, default=256)
    p.add_argument("--precision", default="bf16")
    p.add_argument("--comm", default="auto")
    p.add_argument("--no-fused-bn", action="store_true")
    p.add_argument("--optimizer", default="fused")
    p.add_argument("--skip-e2e", action="store_true")
    p.add_argument("--no-cuda-graph", action="store_true")
    p.add_argument("--entry", default="distributed", choices=["distributed", "apex_distributed", "horovod_distributed", "dataparallel"])
    p.add_argument("--opt-level", default="O2")
    p.add_argument("--dump-outputs", metavar="DIR", default=None,
                   help="write the last timed step's results to DIR/<name>.npy (rank 0) to compare two builds")
    return p.parse_args()


# ---------------------------------------------------------------------- clocks sampling (rank 0)
class ClockSampler:
    """SM clock + throttle reasons sampled DURING the timed region (every 100 ms) through NVML in a light thread;
    falls back to an `nvidia-smi -lms` child process.  (Polling nvidia-smi itself takes driver locks and measurably
    slows an 8-rank step, so NVML is preferred.)"""
    Q = "clocks.sm,clocks.max.sm,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown," \
        "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap"
    NAMES = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]

    def __init__(self, index: int = 0):
        self.index = index
        self.sm, self.mx, self.reasons = [], [], set()
        self.proc = None
        self._stop = threading.Event()
        self.thread = None
        self.mode = None

    # ---- NVML
    def _nvml_loop(self, nv, h):
        bits = {"hw_slowdown": getattr(nv, "nvmlClocksEventReasonHwSlowdown", 0x8),
                "hw_thermal_slowdown": getattr(nv, "nvmlClocksEventReasonHwThermalSlowdown", 0x40),
                "sw_thermal_slowdown": getattr(nv, "nvmlClocksEventReasonSwThermalSlowdown", 0x20),
                "sw_power_cap": getattr(nv, "nvmlClocksEventReasonSwPowerCap", 0x4)}
        get_reasons = getattr(nv, "nvmlDeviceGetCurrentClocksEventReasons", None) or nv.nvmlDeviceGetCurrentClocksThrottleReasons
        while not self._stop.is_set():
            try:
                self.sm.append(float(nv.nvmlDeviceGetClockInfo(h, nv.NVML_CLOCK_SM)))
                self.mx.append(float(nv.nvmlDeviceGetMaxClockInfo(h, nv.NVML_CLOCK_SM)))
                r = int(get_reasons(h))
                for k, b in bits.items():
                    if r & b:
                        self.reasons.add(k)
            except Exception:  # noqa: BLE001
                pass
            self._stop.wait(0.1)

    def start(self):
        try:
            import pynvml as nv
            nv.nvmlInit()
            vis = os.environ.get("CUDA_VISIBLE_DEVICES")
            idx = int(vis.split(",")[self.index]) if vis and vis.split(",")[self.index].isdigit() else self.index
            h = nv.nvmlDeviceGetHandleByIndex(idx)
            self.mode = "nvml"
            self.thread = threading.Thread(target=self._nvml_loop, args=(nv, h), daemon=True)
            self.thread.start()
            return
        except Exception:  # noqa: BLE001
            pass
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.index), "--query-gpu=" + self.Q,
                                          "--format=csv,noheader,nounits", "-lms", "250"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.mode = "nvidia-smi"
            self.thread = threading.Thread(target=self._read, daemon=True)
            self.thread.start()
        except Exception:  # noqa: BLE001
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            f = [x.strip() for x in line.strip().split(",")]
            if len(f) < 6:
                continue
            try:
                self.sm.append(float(f[0]))
                self.mx.append(float(f[1]))
            except ValueError:
                continue
            for n, v in zip(self.NAMES, f[2:6]):
                if v.lower().startswith("active"):
                    self.reasons.add(n)

    def stop(self):
        if self.mode is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["clock sampling unavailable"]}
        if self.mode == "nvml":
            self._stop.set()
            self.thread.join(timeout=1.0)
        else:
            time.sleep(0.3)
            self.proc.terminate()
            try:
                self.proc.wait(timeout=2)
            except Exception:  # noqa: BLE001
                self.proc.kill()
        return {"sm_mhz": statistics.median(self.sm) if self.sm else None, "sm_max_mhz": max(self.mx) if self.mx else None,
                "reasons": sorted(self.reasons), "samples": len(self.sm), "source": self.mode}


DUMP_SAMPLE = 1 << 22      # state entries kept by --dump-outputs: 16 MB of float32


def dump_outputs(directory: str, model, metrics) -> None:
    """What the timed step hands its caller, after the last timed step: the reduced loss / top-1 / top-5 of that step
    (``metrics.npy``, float64) and the trained model state - every floating-point entry of ``state_dict()`` (weights
    and BatchNorm running statistics) flattened in order, of which the ``DUMP_SAMPLE`` positions drawn with a fixed
    seed are written in ascending order (``state_sample.npy``, float32)."""
    import numpy as np
    os.makedirs(directory, exist_ok=True)
    np.save(os.path.join(directory, "metrics.npy"), np.asarray(metrics.last, dtype=np.float64))
    flat = torch.cat([t.detach().reshape(-1).float() for t in model.state_dict().values() if t.is_floating_point()])
    idx = np.sort(np.random.default_rng(0).choice(flat.numel(), size=min(flat.numel(), DUMP_SAMPLE), replace=False))
    np.save(os.path.join(directory, "state_sample.npy"), flat[torch.from_numpy(idx).to(flat.device)].cpu().numpy())


def dist_env():
    if "RANK" in os.environ and "WORLD_SIZE" in os.environ:
        return int(os.environ["RANK"]), int(os.environ.get("LOCAL_RANK", 0)), int(os.environ["WORLD_SIZE"])
    return 0, 0, 1


def max_over_ranks(ms: float, device) -> float:
    if dist.is_initialized() and dist.get_world_size() > 1:
        t = torch.tensor([ms], dtype=torch.float64, device=device)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())
    return ms


def barrier_sync(device):
    torch.cuda.synchronize(device)
    if dist.is_initialized() and dist.get_world_size() > 1:
        dist.barrier()
    torch.cuda.synchronize(device)


# ====================================================================== own arm
def run_own(a):
    from pytorch_distributed_b200 import _ext, cli, driver
    from pytorch_distributed_b200.models import create_model
    from pytorch_distributed_b200.utils.data import SyntheticLoader
    from pytorch_distributed_b200.utils.meters import AverageMeter

    rank, local_rank, world = dist_env()
    dp = a.entry == "dataparallel"          # one process drives a.gpus devices (BASELINE config 5)
    assert world == a.gpus or world == 1, "launch with torchrun --nproc-per-node %d" % a.gpus
    torch.cuda.set_device(local_rank)
    device = torch.device("cuda", local_rank)
    argv = ["-a", a.arch, "-b", str(a.batch_per_gpu * (a.gpus if dp else world)), "--synthetic", "--precision", a.precision, "--comm", a.comm,
            "--optimizer", a.optimizer, "--quiet"]
    if dp:
        argv += ["--gpus", ",".join(str(i) for i in range(a.gpus))]
    if a.no_fused_bn:
        argv.append("--no-fused-bn")
    argv += os.environ.get("PTD_BENCH_ARGS", "").split()          # extra driver flags for ablations (recorded in config.opt_in)
    if a.entry == "apex_distributed":
        argv += ["--opt-level", a.opt_level]
        if a.precision == "bf16":
            argv[argv.index("--precision") + 1] = "fp16"
    args = cli.parse_args(a.entry, argv)
    st = driver.STRATEGIES[a.entry]()
    if world > 1 or a.entry == "horovod_distributed":
        st.init_process_group(args, local_rank, world)
    torch.manual_seed(0)                    # the same weights on every run: --dump-outputs compares builds
    model = create_model(args.arch, num_classes=args.num_classes, fused_bn=args.fused_bn)
    model, optimizer = st.build(model, args, device, local_rank)
    criterion = torch.nn.CrossEntropyLoss().to(device)
    # cuDNN as distributed.py runs it (algorithms picked by timing them).  --dump-outputs needs the same results on every
    # run instead: deterministic algorithms chosen by heuristics (a timed choice can differ from run to run, and so can
    # its rounding).  The JSON line records which of the two the timed steps used.
    torch.backends.cudnn.benchmark = not a.dump_outputs
    torch.backends.cudnn.deterministic = bool(a.dump_outputs)
    B = a.batch_per_gpu * (a.gpus if dp else 1)
    W, K = a.warmup, a.steps
    losses, top1, top5 = AverageMeter("Loss"), AverageMeter("Acc@1"), AverageMeter("Acc@5")
    metrics = driver.MetricPipeline(getattr(st, "comm", None), device, (losses, top1, top5), reduce=True)

    use_graph = ((not a.no_cuda_graph) and st.graph_capable and getattr(getattr(st, "comm", None), "backend", "") == "fused"
                 and hasattr(optimizer, "refresh_hyper"))
    step = driver.TrainStep(st, model, criterion, optimizer, metrics, use_graph=use_graph, warmup=2)   # captured inside warm-up

    model.train()
    # ---------------- phase A: device-resident inputs (the `value`)
    loader = SyntheticLoader(B, 4, args.image_size, args.num_classes, pool=4, rank=rank)
    pf = st.prefetcher(loader, device, args)
    resident = [(i.clone(), t.clone()) for i, t in pf]      # 4 distinct bf16 NHWC batches, staged once
    torch.cuda.synchronize(device)
    for i in range(W):
        step(*resident[i % len(resident)])
    metrics.drain()
    barrier_sync(device)
    sampler = ClockSampler(local_rank)
    if rank == 0:
        sampler.start()
    n0 = _ext.launches
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    prof = os.environ.get("PTD_PROFILE") == "1"     # ncu --profile-from-start off: capture only the timed region
    if prof:
        torch.cuda.profiler.start()
    ev0.record()
    t_host = time.perf_counter()
    for i in range(K):
        step(*resident[i % len(resident)])
    host_ms = (time.perf_counter() - t_host) * 1e3 / K      # time the host needs to ENQUEUE one step
    ev1.record()
    if prof:
        torch.cuda.synchronize(device)
        torch.cuda.profiler.stop()
    barrier_sync(device)
    launches = _ext.launches - n0
    clocks = sampler.stop() if rank == 0 else None
    metrics.drain()
    if a.dump_outputs and rank == 0:
        dump_outputs(a.dump_outputs, model, metrics)
    ms = max_over_ranks(ev0.elapsed_time(ev1), device)
    value = B * world * K / (ms / 1e3)
    # PTD_PYPROFILE=<file>: cProfile of 5 extra steps (host-side cost of a step; outside the timed region)
    if os.environ.get("PTD_PYPROFILE") and rank == 0:
        import cProfile
        import pstats
        pr = cProfile.Profile()
        pr.enable()
        for i in range(5):
            step(*resident[i % len(resident)])
        pr.disable()
        torch.cuda.synchronize(device)
        with open(os.environ["PTD_PYPROFILE"], "w") as f:
            pstats.Stats(pr, stream=f).sort_stats("cumulative").print_stats(45)
    # PTD_TIMELINE=<prefix>: 3 extra steps under torch.profiler (CUPTI kernel records, also inside graph replays), written as
    # <prefix>.rank<r>.json for tools/timeline_summary.py.  Outside the timed region: the profiler never touches a bench value.
    if os.environ.get("PTD_TIMELINE"):
        from torch.profiler import ProfilerActivity, profile
        barrier_sync(device)
        with profile(activities=[ProfilerActivity.CUDA]) as prof_tl:
            for i in range(3):
                step(*resident[i % len(resident)])
            torch.cuda.synchronize(device)
        metrics.drain()
        if rank in (0, world - 1):
            prof_tl.export_chrome_trace("%s.rank%d.json" % (os.environ["PTD_TIMELINE"], rank))
        barrier_sync(device)

    # ---------------- phase B: end to end (pinned host -> device every step, metrics back to the host every step)
    e2e = None
    if not a.skip_e2e:
        loader = SyntheticLoader(B, W + K, args.image_size, args.num_classes, pool=4, rank=rank)
        pf = st.prefetcher(loader, device, args)
        it = iter(pf)
        for _ in range(W):
            step(*next(it))
        metrics.drain()
        barrier_sync(device)
        h0, d0 = pf.h2d_bytes, metrics.d2h_bytes
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        n = 0
        for batch in it:
            step(*batch)
            n += 1
        metrics.drain()                     # the host has read every step's loss/accuracy
        e1.record()
        barrier_sync(device)
        assert n == K, (n, K)
        ms2 = max_over_ranks(e0.elapsed_time(e1), device)
        # the prefetcher stages batch i+1 while step i runs: K-1 copies + the first timed batch (staged during the
        # last warm-up step) => count K copies for K steps.
        e2e = {"value": B * world * K / (ms2 / 1e3), "unit": "images/s", "ms_per_step": ms2 / K,
               "h2d_bytes_per_step": loader.bytes_per_step, "d2h_bytes_per_step": (metrics.d2h_bytes - d0) // max(K, 1)}
    comm = getattr(st, "comm", None)
    if comm is not None:
        comm.check()
    if rank == 0:
        base = published_baseline()
        out = {
            "metric": METRIC, "value": value, "unit": "images/s", "n_gpus": a.gpus if dp else world, "steps": K, "warmup": W,
            "ms_per_step": ms / K, "higher_is_better": True, "scaling": "weak",
            "vs_baseline": (value / base) if base else None, "dtype": args.precision, "data": "synthetic",
            "config": {"model": a.arch, "global_batch": B * world, "seq_len": None, "image_size": args.image_size,
                       "parallelism": "dp%d" % (a.gpus if dp else world), "entry": a.entry, "comm": getattr(comm, "backend", "none"),
                       "nvls": bool(getattr(comm, "nvls", False)), "channels_last": bool(args.channels_last),
                       "fused_bn": args.fused_bn is not False, "optimizer": a.optimizer, "cuda_graph": step.graph is not None,
                       "l2_policy": "inputs larger than L2 (4 x 38.5 MB bf16 batches + GBs of activations per step)",
                       "bucket_cap_mb": args.bucket_cap_mb, "overlap_optimizer": bool(getattr(optimizer, "_overlap", False)),
                       "bucket_view": bool(getattr(args, "bucket_view", False)),
                       "cudnn": "deterministic" if a.dump_outputs else "benchmark",
                       "opt_in": {k: os.environ[k] for k in ("PTD_SPLIT_RESGRAD", "PTD_STEM_GEMM", "PTD_FUSED_CONV1X1", "PTD_MAX_CTAS",
                                                             "PTD_NVLS", "PTD_BENCH_ARGS", "PTD_DEFERRED_BCAST", "PTD_METRICS_SIDE",
                                                             "PTD_ONESHOT_MAX_BYTES", "PTD_HVD_STATIC") if k in os.environ}},
            "clocks": clocks, "e2e": e2e, "gpu_launches": launches, "impl": "own", "host_enqueue_ms_per_step": host_ms,
            "final_loss": losses.val,
        }
        print(json.dumps(out), flush=True)
    if dist.is_initialized():
        dist.barrier()
        dist.destroy_process_group()


def published_baseline():
    try:
        with open(os.path.join(ROOT, "BASELINE.json")) as f:
            pub = json.load(f).get("published", {})
        for v in pub.values():
            if isinstance(v, (int, float)):
                return float(v)
    except Exception:  # noqa: BLE001
        pass
    return None


# ====================================================================== reference arm
def run_reference(a):
    from oracle.run_reference import run
    run(a, METRIC, ClockSampler, published_baseline)


def _self_launch(a) -> None:
    """``python bench.py --gpus N`` without a launcher: re-run under torchrun (one rank per GPU) and pass its exit code on."""
    import socket
    import subprocess
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(a.gpus), "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.abspath(__file__)] + sys.argv[1:]
    sys.exit(subprocess.call(cmd))


if __name__ == "__main__":
    a = parse()
    if a.gpus > 1 and "RANK" not in os.environ and not (a.impl == "own" and a.entry == "dataparallel"):
        _self_launch(a)
    if a.impl == "reference":
        run_reference(a)
    else:
        run_own(a)
