"""Reference arm of bench.py: runs the UNMODIFIED reference (`oracle/_ref/distributed.py`, a byte-for-byte copy of the
reference's distributed.py - the reference is a set of scripts and is not pip-installable, see DESIGN.md) through
its own public API and stock code path:

    model = models.__dict__[arch]();  model.cuda(local_rank)
    model = torch.nn.parallel.DistributedDataParallel(model, device_ids=[local_rank])      (reference :147)
    criterion = nn.CrossEntropyLoss().cuda(local_rank);  optimizer = torch.optim.SGD(...)  (reference :151-156)
    cudnn.benchmark = True                                                                  (reference :158)
    ref.train(train_loader, model, criterion, optimizer, epoch, local_rank, args)          (reference :228-276)

i.e. exactly what the reference's `main_worker` does, minus the ImageFolder dataset (there is no ImageNet on the box):
`train_loader` is an in-memory iterable of pinned fp32 NCHW batches, the same shape/dtype a
`DataLoader(pin_memory=True)` hands to the loop.  None of this repo's models, kernels or engines are on that path.

The one runtime shim: `ref.accuracy` is replaced by an equivalent that uses `.reshape(-1)` - the reference's
`.view(-1)` raises on torch >= 1.7 (SURVEY Q1), so the stock function cannot run at all on torch 2.11.  The file on
disk is untouched (its sha256 is checked against the manifest in oracle/install_reference.py).
"""
from __future__ import annotations

import importlib.util
import json
import os
import sys

import torch
import torch.distributed as dist

HERE = os.path.dirname(os.path.abspath(__file__))
REF_DIR = os.path.join(HERE, "_ref")


def _unavailable(why: str):
    print(json.dumps({"impl": "reference", "unavailable": why}), flush=True)
    sys.exit(0)


def _load_ref():
    from oracle import install_reference as inst
    path = os.path.join(REF_DIR, "distributed.py")
    try:
        status = inst.install()            # no-op when oracle/_ref is present and matches the sha256 manifest
    except Exception as e:  # noqa: BLE001
        status = "install failed: %r" % (e,)
    bad = inst.verify()
    if bad:
        sys.stderr.write("[bench --impl reference] REFERENCE ARM UNAVAILABLE: %s; files not matching the manifest: %s\n"
                         "  run `python -c 'import __graft_entry__ as g; g.build()'` where the reference checkout is (%s or %s)\n" % (status, bad, inst.ENV, ", ".join(inst.DEFAULT_DIRS)))
        _unavailable("oracle/_ref incomplete (%s): %s" % (status, ",".join(bad)))
    argv, sys.argv = sys.argv, ["distributed.py"]
    try:
        spec = importlib.util.spec_from_file_location("ref_distributed", path)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
    finally:
        sys.argv = argv
    return mod


def _accuracy_shim(output, target, topk=(1,)):
    """reference accuracy() with .reshape instead of .view (torch>=1.7 compatibility; same values)."""
    with torch.no_grad():
        maxk = max(topk)
        batch_size = target.size(0)
        _, pred = output.topk(maxk, 1, True, True)
        pred = pred.t()
        correct = pred.eq(target.view(1, -1).expand_as(pred))
        res = []
        for k in topk:
            correct_k = correct[:k].reshape(-1).float().sum(0, keepdim=True)
            res.append(correct_k.mul_(100.0 / batch_size))
        return res


class TimedLoader:
    """In-memory stand-in for DataLoader(pin_memory=True): W + K pinned batches; brackets the K timed steps with
    barrier + synchronize + CUDA events from inside the iteration protocol, so the reference loop stays untouched."""

    def __init__(self, batch, warmup, steps, device, num_classes=1000, image_size=224, pool=4, rank=0, on_start=None):
        g = torch.Generator().manual_seed(1234 + rank * 104729)
        self.pool = []
        for _ in range(pool):
            img = torch.randn(batch, 3, image_size, image_size, generator=g).pin_memory()
            tgt = torch.randint(0, num_classes, (batch,), generator=g, dtype=torch.int64).pin_memory()
            self.pool.append((img, tgt))
        self.warmup, self.steps, self.device = warmup, steps, device
        self.ev0 = torch.cuda.Event(enable_timing=True)
        self.ev1 = torch.cuda.Event(enable_timing=True)
        self.bytes_per_step = self.pool[0][0].numel() * 4 + self.pool[0][1].numel() * 8
        self.on_start = on_start

    def __len__(self):
        return self.warmup + self.steps

    def _sync(self):
        torch.cuda.synchronize(self.device)
        if dist.is_initialized() and dist.get_world_size() > 1:
            dist.barrier()
        torch.cuda.synchronize(self.device)

    def __iter__(self):
        for i in range(self.warmup + self.steps):
            if i == self.warmup:
                self._sync()
                if self.on_start:
                    self.on_start()
                self.ev0.record()
            yield self.pool[i % len(self.pool)]
        self.ev1.record()
        self._sync()


def run(a, metric, ClockSampler, published_baseline):
    if not torch.cuda.is_available():
        _unavailable("no CUDA device")
    ref = _load_ref()
    ref.accuracy = _accuracy_shim
    rank = int(os.environ.get("RANK", 0))
    local_rank = int(os.environ.get("LOCAL_RANK", 0))
    world = int(os.environ.get("WORLD_SIZE", 1))
    if "RANK" not in os.environ:      # plain `python bench.py --impl reference` => single-rank process group
        os.environ.update(RANK="0", WORLD_SIZE="1", MASTER_ADDR="127.0.0.1", MASTER_PORT=os.environ.get("MASTER_PORT", "29533"))
    import torch.backends.cudnn as cudnn
    import torch.nn as nn
    import torchvision.models as models
    args = ref.parser.parse_args(["-a", a.arch, "-b", str(a.batch_per_gpu * world), "-p", "1000000", "--local_rank", str(local_rank)])
    args.nprocs = world               # the reference derives it from device_count(); we launch exactly `world` ranks
    dist.init_process_group(backend="nccl")
    model = models.__dict__[args.arch]()
    torch.cuda.set_device(local_rank)
    model.cuda(local_rank)
    args.batch_size = int(args.batch_size / args.nprocs)
    model = torch.nn.parallel.DistributedDataParallel(model, device_ids=[local_rank])
    criterion = nn.CrossEntropyLoss().cuda(local_rank)
    optimizer = torch.optim.SGD(model.parameters(), args.lr, momentum=args.momentum, weight_decay=args.weight_decay)
    cudnn.benchmark = True
    device = torch.device("cuda", local_rank)
    sampler = ClockSampler(local_rank)
    loader = TimedLoader(args.batch_size, a.warmup, a.steps, device, rank=rank, on_start=sampler.start if rank == 0 else None)
    devnull = open(os.devnull, "w")
    stdout, sys.stdout = sys.stdout, devnull      # the reference prints a progress line on every rank
    try:
        ref.train(loader, model, criterion, optimizer, 0, local_rank, args)
    finally:
        sys.stdout = stdout
    clocks = sampler.stop() if rank == 0 else None
    ms = loader.ev0.elapsed_time(loader.ev1)
    t = torch.tensor([ms], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    ms = float(t.item())
    value = args.batch_size * world * a.steps / (ms / 1e3)
    if rank == 0:
        base = published_baseline()
        print(json.dumps({
            "impl": "reference", "metric": metric, "value": value, "unit": "images/s", "n_gpus": world, "steps": a.steps,
            "warmup": a.warmup, "ms_per_step": ms / a.steps, "higher_is_better": True, "scaling": "weak",
            "vs_baseline": (value / base) if base else None, "dtype": "fp32 (stock reference: no autocast; cuDNN TF32 convs)",
            "data": "synthetic",
            "config": {"model": a.arch, "global_batch": args.batch_size * world, "seq_len": None, "parallelism": "dp%d" % world,
                       "entry": "distributed.py (unmodified, torch DDP + NCCL + torch.optim.SGD)",
                       "l2_policy": "inputs larger than L2 (154 MB fp32 batch per step)"},
            "clocks": clocks,
            "e2e": {"value": value, "unit": "images/s", "h2d_bytes_per_step": loader.bytes_per_step, "d2h_bytes_per_step": 12,
                    "note": "the reference loop copies every batch from pinned host memory and reads 3 scalars back per step; "
                            "its device-timed number IS end to end"},
            "gpu_launches": 0,
        }), flush=True)
    dist.barrier()
    dist.destroy_process_group()
