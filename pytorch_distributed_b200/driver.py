"""The shared training driver: ``main_worker`` / ``train`` / ``validate`` written ONCE for all entrypoints.

The reference copies these ~250 lines into each of its six scripts (/root/reference/distributed.py:129-324 and the
five siblings); the per-script differences (SURVEY section 2.3) are captured here by small :class:`Strategy` objects.

Hot-loop differences from the reference (/root/reference/distributed.py:242-276), all behaviour-preserving:
  * H2D copies run on a side stream with a fused normalise/cast/NHWC kernel (every entrypoint, not only apex);
  * accuracy + ``barrier`` + 3x ``reduce_mean`` + 3x ``.item()`` collapse into ONE low-latency kernel whose result
    is fetched asynchronously (the meters lag the GPU by at most ``--print-freq`` iterations and are drained before
    every print), so the host never stalls the device inside the loop;
  * gradient all-reduce, optimizer and loss scaling run through the fused sm_90a kernels.
Output contract (progress lines, `` * Acc@1`` summary, checkpoint files) is the reference's.
"""
from __future__ import annotations

import contextlib
import csv
import json
import os
import random
import time
import warnings
from collections import deque
from typing import Optional

import torch
import torch.distributed as dist
import torch.nn as nn

from . import cli
from .models import create_model
from .utils.checkpoint import export_ema_state_dict, export_state_dict, load_checkpoint, save_checkpoint
from .utils.data import DataPrefetcher, build_loaders
from .utils.meters import AverageMeter, ProgressMeter, accuracy, adjust_learning_rate

_DTYPES = {"fp32": torch.float32, "bf16": torch.bfloat16, "fp16": torch.float16}
_NVTX = os.environ.get("PTD_NVTX", "0") == "1"
_POISON = os.environ.get("PTD_DEBUG_POISON", "0") == "1"


def seed_everything(args) -> None:
    """/root/reference/distributed.py:116-124"""
    if args.seed is not None:
        random.seed(args.seed)
        torch.manual_seed(args.seed)
        torch.backends.cudnn.deterministic = True
        warnings.warn("You have chosen to seed training. This will turn on the CUDNN deterministic setting, "
                      "which can slow down your training considerably! You may see unexpected behavior when "
                      "restarting from checkpoints.")


def pick_device(args, local_rank: int) -> torch.device:
    want = args.device or ("cuda" if torch.cuda.is_available() else "cpu")
    if want.startswith("cuda"):
        torch.cuda.set_device(local_rank)
        return torch.device("cuda", local_rank)
    return torch.device("cpu")


# ====================================================================== metrics
class MetricPipeline:
    """Asynchronous (loss, acc1, acc5) reduction: launch now, read later.

    GPU: one K4 kernel (top-k counting + LL all-reduce over NVLink) + a 16-byte D2H copy into a pinned ring slot +
    an event.  The meters are updated when the event has completed (``poll``) or on ``drain``.
    CPU / library backends: computed eagerly with torch ops (gloo all-reduce).
    """

    def __init__(self, comm, device, meters, reduce: bool = True, depth: int = 64):
        self.comm = comm
        self.device = device
        self.losses, self.top1, self.top5 = meters
        self.reduce = reduce and comm is not None
        self.cuda = device.type == "cuda"
        self.pending = deque()
        self.d2h_bytes = 0
        self.last = (0.0, 0.0, 0.0)
        if self.cuda:
            self.ring = [torch.zeros(4, dtype=torch.float32).pin_memory() for _ in range(depth)]
            self.dev = [torch.zeros(4, dtype=torch.float32, device=device) for _ in range(depth)]
            self.slot = 0
        # the metric kernel waits for every peer's values (LL all-reduce): on the communicator's side stream that wait never
        # stalls the compute stream (PTD_METRICS_SIDE=0 puts it back in line)
        self.side = None
        if self.cuda and self.reduce and getattr(comm, "backend", "") == "fused" and os.environ.get("PTD_METRICS_SIDE", "1") == "1":
            self.side = comm.side_stream
        self._side_dirty = False

    def push(self, output, target, loss, n: int) -> None:
        if not self.cuda:
            out = torch.zeros(4)
            if self.reduce:
                self.comm.metrics(output.detach(), target, loss.detach(), out)
            else:
                a1, a5 = accuracy(output.detach(), target, topk=(1, 5))
                out[0], out[1], out[2] = loss.detach().float(), a1[0], a5[0]
            self._apply(out.tolist(), n)
            return
        dev = self.dev[self.slot]
        self.launch(output, target, loss, dev)
        self.fetch(dev, n, stream=self.side)

    def launch(self, output, target, loss, dev) -> None:
        """Enqueue the metric kernel writing into ``dev`` (capturable in a CUDA graph)."""
        lossf = loss.detach()
        if lossf.dtype != torch.float32:
            lossf = lossf.float()
        if self.side is not None:
            out = output.detach()
            ev = torch.cuda.Event()
            ev.record()
            self.side.wait_event(ev)
            with torch.cuda.stream(self.side):
                self.comm.metrics(out, target, lossf, dev)
            for t in (out, target, lossf):
                t.record_stream(self.side)
            self._side_dirty = True
        elif self.reduce and getattr(self.comm, "backend", "") == "fused":
            self.comm.metrics(output.detach(), target, lossf, dev)
        else:
            from . import _ext
            _local_metrics(_ext.lib(), output.detach(), target, lossf, dev)
            if self.reduce and self.comm.world > 1:
                self.comm.reduce_scalars_(dev[:3], average=True)

    def fetch(self, dev, n: int, stream=None) -> None:
        """16-byte D2H copy of a finished (or enqueued) metric vector into the pinned ring + completion event.
        ``stream``: the stream the metric kernel was enqueued on (None = the current one, e.g. after a graph replay)."""
        if len(self.pending) >= len(self.ring) - 1:
            self.poll(block_oldest=True)
        i = self.slot
        self.slot = (self.slot + 1) % len(self.ring)
        ev = torch.cuda.Event()
        if stream is not None:
            with torch.cuda.stream(stream):
                self.ring[i].copy_(dev, non_blocking=True)
                ev.record(stream)
        else:
            self.ring[i].copy_(dev, non_blocking=True)
            ev.record()
        self.d2h_bytes += 16
        self.pending.append((ev, i, n))

    def join(self) -> None:
        """Make the current stream wait for metric work enqueued on the side stream (needed before a capture ends and
        before buffers the kernel reads may be reused)."""
        if self.side is not None and self._side_dirty:
            torch.cuda.current_stream().wait_stream(self.side)
            self._side_dirty = False

    def _apply(self, vals, n):
        self.last = (vals[0], vals[1], vals[2])
        self.losses.update(vals[0], n)
        self.top1.update(vals[1], n)
        self.top5.update(vals[2], n)

    def poll(self, block_oldest: bool = False) -> None:
        while self.pending:
            ev, i, n = self.pending[0]
            if block_oldest:
                ev.synchronize()
                block_oldest = False
            elif not ev.query():
                break
            self.pending.popleft()
            self._apply(self.ring[i].tolist(), n)

    def drain(self) -> None:
        while self.pending:
            self.poll(block_oldest=True)


_single_arena = {}


def _local_metrics(C, output, target, loss, out):
    """K4 without peers (world == 1 arena): used by DataParallel / library-comm runs on a GPU."""
    dev = output.device.index
    a = _single_arena.get(dev)
    if a is None:
        a = C.SymmArena(dev, 0, 1, 1 << 21)
        _single_arena[dev] = a
    from . import _ext
    _ext.note_launch()
    a.launch_metrics(0, output, target, loss, out)


# ====================================================================== one optimisation step (eager or CUDA graph)
class TrainStep:
    """forward + loss + metric kernel + backward (fused bucket all-reduce on the side stream) + optimizer.

    With ``use_graph`` the whole step - several hundred kernels on two streams - is captured into ONE CUDA graph after
    ``warmup`` eager iterations and replayed afterwards: the host then enqueues a 38 MB device copy and one graph
    launch per step instead of ~900 kernels plus the autograd/hook Python, which is what bounds the step once the
    kernels are fused (bench.py reports host_enqueue_ms_per_step).  Everything the graph needs to vary is
    device-resident: hyper-parameters and loss scale (FusedSGD.hyper), signal sequence numbers (csrc/common.cuh), BN
    accumulators.  Batches of another shape (last partial batch) fall back to the eager path.

    Gradient accumulation (``st.accum_steps`` = N > 1, ``--accum-steps``): one call is one micro-batch, and every N-th call
    ends an optimizer step.  Calls 1..N-1 of a step run forward, metrics and a backward of loss / N under the strategy's
    no-sync context; call N runs the body above with loss / N.  The metrics keep the undivided loss.  Under a graph each
    of the two kinds of pass is captured the first time it comes after the warm-up and one eager optimizer step (two
    graphs, one memory pool).

    MixUp / CutMix / label smoothing (``st.batch_mix``, an :class:`~.ops.mix.BatchMix`): every pass draws its mixing
    parameters on the host first (eager, and before each replay), mixes the batch, takes the loss from
    ``batch_mix.loss`` and gives the metric kernel the dominant labels.  The ``criterion`` passed in is then unused.
    """

    def __init__(self, st, model, criterion, optimizer, metrics, use_graph: bool = False, warmup: int = 3, ema=None):
        self.st, self.model, self.criterion, self.optimizer, self.metrics = st, model, criterion, optimizer, metrics
        self.ema = ema if ema is not None else getattr(st, "model_ema", None)   # --model-ema: once per optimizer step
        self.batch_mix = getattr(st, "batch_mix", None)
        self.clip = getattr(st, "clip_grad_norm", None)      # --clip-grad-norm with --optimizer torch (FusedSGD clips inside)
        self.use_graph = bool(use_graph) and torch.cuda.is_available()
        self.warmup = warmup
        self.calls = 0
        self.accum = max(1, int(getattr(st, "accum_steps", 1) or 1))
        self.k = 0                      # pass index inside the current optimizer step
        self.eager_steps = 0            # optimizer steps run eagerly (the first one creates the optimizer's device state)
        self.graph = None               # the last pass of a step (the whole step without accumulation)
        self.graph_accum = None         # the earlier passes of a step (accumulation only)
        self.graph_launches = self.graph_accum_launches = 0
        self.static_x = self.static_y = self.static_m = None

    def _body(self, images, target, dev=None):
        nvtx = _NVTX and images.is_cuda          # PTD_NVTX=1: forward / backward(+bucket all-reduce) / optimizer ranges for nsys / ncu
        if nvtx:
            torch.cuda.nvtx.range_push("ptd.forward")
        bm = self.batch_mix
        if bm is not None:
            images, mixed = bm.apply(images, target)
        output = self.st.forward(self.model, images)
        if bm is not None:
            loss = bm.loss(output, mixed)
            target = bm.metric_target(mixed)
        else:
            loss = self.criterion(output.float() if output.dtype != torch.float32 else output, target)
        if dev is None:
            self.metrics.push(output, target, loss, images.size(0))
        else:
            self.metrics.launch(output, target, loss, dev)
        eng = getattr(self.st, "engine", None)
        if eng is not None and getattr(eng, "bucket_view", False):
            eng.zero_grads()           # bucket views: ONE memset of the arena; backward then accumulates in place (no pack pass)
        elif dev is None and self.k == 0:
            self.optimizer.zero_grad()
        if nvtx:
            torch.cuda.nvtx.range_pop()
            torch.cuda.nvtx.range_push("ptd.backward")
        if self.accum > 1:
            loss = loss / self.accum
            if self.k < self.accum - 1:
                with self.st.no_sync(self.model):
                    self.st.backward(loss, self.optimizer, last=False)
                if nvtx:
                    torch.cuda.nvtx.range_pop()
                self.metrics.join()
                return
        self.st.backward(loss, self.optimizer)
        if nvtx:
            torch.cuda.nvtx.range_pop()
            torch.cuda.nvtx.range_push("ptd.optimizer")
        if self.clip is not None:
            self.st.clip_and_step(self.optimizer, self.clip)
        else:
            self.optimizer.step()
        if self.ema is not None:
            self.ema.update()           # a fused optimizer has already averaged inside its step: no-op then
        if nvtx:
            torch.cuda.nvtx.range_pop()
        self.metrics.join()
        eng = getattr(self.st, "engine", None)
        if _POISON and eng is not None and getattr(eng, "_flat", None) is not None and getattr(eng, "fused", False):
            # PTD_DEBUG_POISON=1: a stale read of the wire arena shows up as NaN.  Only the parameters' own ranges are
            # poisoned: the alignment padding is never packed, and NaN left there would trip the all-reduce's non-finite
            # test (dynamic loss scaling) on every step
            arena = eng.grad_arena()
            for off, p in zip(eng.param_elem_off, eng.params):
                arena[off:off + p.numel()].fill_(float("nan"))

    def _static_fits(self, images):
        return self.static_x is None or (images.shape == self.static_x.shape and images.dtype == self.static_x.dtype)

    def _capture(self, images, target, last):
        if self.static_x is None:       # both graphs read the same static batch and write the same metric vector
            self.static_x, self.static_y = images.clone(), target.clone()
            self.static_m = torch.zeros(4, dtype=torch.float32, device=images.device)
        if self.k == 0:
            self.optimizer.zero_grad(set_to_none=True)
        torch.cuda.synchronize()
        from . import _ext
        n0 = _ext.launches
        g = torch.cuda.CUDAGraph()
        other = self.graph_accum if last else self.graph
        with torch.cuda.graph(g, pool=other.pool() if other is not None else None):
            self._body(self.static_x, self.static_y, self.static_m)
        n = _ext.launches - n0          # native kernels inside the graph (capture enqueues, replay runs them)
        _ext.launches = n0
        if last:
            self.graph, self.graph_launches = g, n
        else:
            self.graph_accum, self.graph_accum_launches = g, n

    def __call__(self, images, target):
        self.calls += 1
        last = self.k == self.accum - 1
        if self.batch_mix is not None:
            self.batch_mix.draw(images.shape[-2:])
        # with accumulation, capture after one eager optimizer step (it creates the optimizer's device state, a host copy
        # no capture may hold) and the earlier-pass graph first: a last pass that adds into p.grad through autograd
        # (horovod's backward_passes_per_step) must be captured reading the gradients that graph writes
        ready = self.accum == 1 or (self.eager_steps > 0 and (not last or self.graph_accum is not None))
        if (self.use_graph and ready and (self.graph if last else self.graph_accum) is None and self.calls > self.warmup
                and images.is_cuda and self._static_fits(images)):
            self._capture(images, target, last)
        graph, launches = (self.graph, self.graph_launches) if last else (self.graph_accum, self.graph_accum_launches)
        if graph is not None and self._static_fits(images):
            self.static_x.copy_(images, non_blocking=True)
            self.static_y.copy_(target, non_blocking=True)
            if last and hasattr(self.optimizer, "refresh_hyper"):
                self.optimizer.refresh_hyper()
            graph.replay()
            from . import _ext
            _ext.note_launch(launches)
            self.metrics.fetch(self.static_m, images.size(0))
        else:
            self._body(images, target)
            self.eager_steps += last
        self.k = 0 if last else self.k + 1
        self.metrics.poll()


# ====================================================================== strategies
class Strategy:
    """What differs between the reference scripts (SURVEY 2.3)."""

    name = "distributed"
    distributed = True          # one process per GPU with a process group
    shard_batch = True          # per-process batch = -b / world
    reduce_metrics = True
    raw_uint8_loader = False
    cast_params = True          # low precision = cast the model (fp32 masters in FusedSGD); False => autocast
    graph_capable = True        # the train step may be captured into a CUDA graph (--cuda-graph)
    overlap_optimizer = True    # one backward per step and nothing between backward and step: the update may ride behind each bucket
    epoch_csv: Optional[str] = None

    def init_process_group(self, args, local_rank: int, nprocs: int) -> None:
        backend = args.dist_backend or ("nccl" if (args.device or "cuda").startswith("cuda") and torch.cuda.is_available() else "gloo")
        kw = {}
        if backend == "nccl":
            kw["device_id"] = torch.device("cuda", local_rank)
        if args.dist_url:
            # multi-node launchers (Slurm) put the GLOBAL rank in args.global_rank (= node_rank * ngpus + gpu, reference
            # distributed_slurm_main.py:147); local_rank only ever selects the device
            rank = getattr(args, "global_rank", None)
            dist.init_process_group(backend=backend, init_method=args.dist_url, world_size=nprocs,
                                    rank=local_rank if rank is None else int(rank), **kw)
        else:
            dist.init_process_group(backend=backend, **kw)

    def world(self):
        return dist.get_world_size() if dist.is_initialized() else 1

    def rank(self):
        return dist.get_rank() if dist.is_initialized() else 0

    def is_saver(self, args) -> bool:
        return self.rank() == 0

    def comm_kind(self, args, device) -> str:
        if args.comm != "auto":
            return args.comm
        return "fused" if device.type == "cuda" else "gloo"

    def prepare_model(self, model, args, device):
        """Precision / layout policy for the plain-DDP style entrypoints."""
        model.to(device)
        prec = args.precision or ("bf16" if device.type == "cuda" else "fp32")
        args.precision = prec
        cl = args.channels_last if args.channels_last is not None else device.type == "cuda"
        args.channels_last = cl
        if cl:
            model.to(memory_format=torch.channels_last)
        self.autocast = None
        if prec != "fp32":
            if args.optimizer == "fused" and device.type == "cuda" and self.cast_params:
                from .parallel.amp import cast_model
                cast_model(model, _DTYPES[prec], keep_batchnorm_fp32=True)   # fp32 masters live in FusedSGD
            else:
                self.autocast = _DTYPES[prec]                                # stock optimizer: fp32 weights + autocast
        self.input_dtype = _DTYPES[prec] if (prec != "fp32" and self.autocast is None) else torch.float32
        return model

    def set_accum_steps(self, args) -> int:
        self.accum_steps = int(getattr(args, "accum_steps", 1) or 1)
        return self.accum_steps

    def no_sync(self, model):
        """Context of the backwards that only accumulate (every micro-batch of an optimizer step but the last)."""
        return model.no_sync() if hasattr(model, "no_sync") else contextlib.nullcontext()

    def make_optimizer(self, model, args):
        clip = getattr(args, "clip_grad_norm", None)
        self.clip_grad_norm = None      # --clip-grad-norm for an optimizer that does not clip inside its step (TrainStep)
        if args.optimizer == "fused":
            from .ops.fused_sgd import FusedSGD
            opt = FusedSGD(model.parameters(), args.lr, momentum=args.momentum, weight_decay=args.weight_decay,
                           overlap_backward=bool(getattr(args, "overlap_optimizer", False)) and self.overlap_optimizer,
                           clip_grad_norm=clip)
        else:
            opt = torch.optim.SGD(model.parameters(), args.lr, momentum=args.momentum, weight_decay=args.weight_decay)
            self.clip_grad_norm = clip
        if getattr(args, "larc", False):
            from .apex.parallel.LARC import LARC
            opt = LARC(opt, trust_coefficient=args.larc_trust_coefficient, clip=args.larc_clip)
        return opt

    def wrap(self, model, args, device, local_rank):
        from .parallel.ddp import DistributedDataParallel
        wire = args.wire_dtype if device.type == "cuda" else "fp32"
        model = DistributedDataParallel(model, device_ids=[local_rank] if device.type == "cuda" else None,
                                        comm=self.comm_kind(args, device), wire_dtype=wire, bucket_cap_mb=args.bucket_cap_mb,
                                        gradient_as_bucket_view=bool(getattr(args, "bucket_view", False)) and device.type == "cuda",
                                        fp32_grad_accumulation=self.set_accum_steps(args) > 1)
        self.comm = model.comm
        self.engine = model.engine
        from .utils.dist_ops import set_default_communicator
        set_default_communicator(self.comm)
        return model

    def build(self, model, args, device, local_rank):
        """Precision, wrapper and optimizer (``build_model``), then the ``--model-ema`` average of the finished model and the
        ``--label-smoothing`` / ``--mixup-alpha`` / ``--cutmix-alpha`` target policy and the ``--auto-augment`` /
        ``--random-erase`` input policy."""
        model, optimizer = self.build_model(model, args, device, local_rank)
        self.model_ema = make_model_ema(model, optimizer, args)
        self.batch_mix = make_batch_mix(args, device, self.rank() if self.distributed else 0)
        self.batch_augment = make_batch_augment(args, device, self.rank() if self.distributed else 0)
        return model, optimizer

    def build_model(self, model, args, device, local_rank):
        model = self.prepare_model(model, args, device)
        model = self.wrap(model, args, device, local_rank)
        optimizer = self.make_optimizer(model, args)
        return model, optimizer

    def forward(self, model, images):
        if self.autocast is not None:
            with torch.autocast(device_type=images.device.type, dtype=self.autocast):
                return model(images)
        return model(images)

    def backward(self, loss, optimizer, last: bool = True):
        loss.backward()

    def clip_and_step(self, optimizer, max_norm):
        """``--clip-grad-norm`` with a stock optimizer: ``clip_grad_norm_`` on the reduced, unscaled ``p.grad``, then the step."""
        self._note_clip(torch.nn.utils.clip_grad_norm_([p for g in optimizer.param_groups for p in g["params"]], max_norm), max_norm)
        optimizer.step()

    def _note_clip(self, total, max_norm):
        """The stock path's counterpart of FusedSGD.grad_norm() / clipped_steps(), on the device (no host read per step)."""
        if getattr(self, "clip_count", None) is None:
            self.clip_count = torch.zeros(1, dtype=torch.int32, device=total.device)
        self.grad_norm = total
        self.clip_count += (max_norm / (total + 1e-6) < 1).to(torch.int32)

    def clip_record(self, optimizer) -> dict:
        """``grad_norm`` of the last clipped step and ``clipped_steps`` since the previous call, for the train JSONL record (one
        host read each, after the epoch's synchronise)."""
        if hasattr(optimizer, "grad_norm") and callable(optimizer.grad_norm):
            total, count = optimizer.grad_norm(), optimizer.clipped_steps()
        else:
            total, count = getattr(self, "grad_norm", None), getattr(self, "clip_count", None)
        if total is None:
            return {"grad_norm": None, "clipped_steps": 0}
        n = int(count.item())
        seen, self._clipped_seen = getattr(self, "_clipped_seen", 0), n
        return {"grad_norm": float(total.item()), "clipped_steps": n - seen}

    def unwrapped(self, model):
        return model.module if hasattr(model, "module") else model

    def prefetcher(self, loader, device, args, limit=None, augment=None):
        """``augment``: the training loader's :class:`~.ops.augment.BatchAugment`, applied when the loader ships uint8 pixels
        (ImageFolder workers that normalise have applied torchvision's transforms already)."""
        raw = self.raw_uint8_loader or getattr(loader, "raw_uint8", False)     # native shard loader ships uint8 pixels
        return DataPrefetcher(loader, device, dtype=self.input_dtype, channels_last=bool(args.channels_last),
                              normalize="imagenet255" if raw else None, limit=limit, augment=augment if raw else None)


class ApexStrategy(Strategy):
    """/root/reference/apex_distributed.py: amp.initialize + apex DDP + scale_loss + data_prefetcher."""
    name = "apex_distributed"
    raw_uint8_loader = False

    def build_model(self, model, args, device, local_rank):
        from .apex import amp
        from .apex.parallel import DistributedDataParallel as ApexDDP
        model.to(device)
        cl = args.channels_last if args.channels_last is not None else device.type == "cuda"
        args.channels_last = cl
        if cl:
            model.to(memory_format=torch.channels_last)
        prec = args.precision or ("fp16" if device.type == "cuda" else "bf16")
        args.precision = prec
        half = _DTYPES[prec] if prec != "fp32" else torch.float16
        opt_level = "O0" if prec == "fp32" else args.opt_level
        optimizer = self.make_optimizer(model, args)
        ls = args.loss_scale if args.loss_scale == "dynamic" else float(args.loss_scale)
        model, optimizer = amp.initialize(model, optimizer, opt_level=opt_level, loss_scale=ls if opt_level != "O0" else 1.0,
                                          half_dtype=half, verbosity=0 if args.quiet else 1)
        self.amp = amp
        wire = "fp32" if device.type != "cuda" or opt_level == "O0" else ("fp16" if half == torch.float16 else "bf16")
        if args.wire_dtype != "bf16":   # explicit override
            wire = args.wire_dtype
        model = ApexDDP(model, comm=self.comm_kind(args, device), wire_dtype=wire,
                        fp32_grad_accumulation=self.set_accum_steps(args) > 1)
        self.comm = model.comm
        self.engine = model.engine
        self.autocast = None            # amp wrapped the forward already
        self.input_dtype = half if opt_level in ("O2", "O3") else torch.float32
        return model, optimizer

    def backward(self, loss, optimizer, last: bool = True):
        # apex's accumulation idiom: the earlier micro-batches leave their gradients scaled; an overflow in any of them
        # reaches the last pass's sum as inf / NaN, and the step is skipped once
        with self.amp.scale_loss(loss, optimizer, delay_unscale=not last) as scaled_loss:
            scaled_loss.backward()


class HorovodStrategy(Strategy):
    """/root/reference/horovod_distributed.py: broadcast_parameters + DistributedOptimizer(compression=fp16)."""
    name = "horovod_distributed"
    overlap_optimizer = False   # horovod semantics: step() synchronises the handles first, then updates
    cast_params = True          # 16-bit model, fp32 masters in FusedSGD (fp32 weights + autocast take the same wgmma conv / stem GEMM paths)
    # the fusion dispatcher is a host thread: not capturable - unless the static schedule replaces it after the first step
    graph_capable = os.environ.get("PTD_HVD_STATIC", "1") == "1" and os.environ.get("HOROVOD_AUTOTUNE", "0") != "1"

    def init_process_group(self, args, local_rank, nprocs):
        from .parallel import hvd
        hvd.init(comm=args.comm if args.comm != "auto" else None, device=args.device)
        self.hvd = hvd

    def world(self):
        return self.hvd.size()

    def rank(self):
        return self.hvd.rank()

    def build_model(self, model, args, device, local_rank):
        hvd = self.hvd
        model = self.prepare_model(model, args, device)
        hvd.broadcast_parameters(model.state_dict(), root_rank=0)
        # the fp32 values stashed by the bf16 cast become the optimizer's master weights: they must be rank 0's too
        inits = [p._ptd_master_init for p in model.parameters() if getattr(p, "_ptd_master_init", None) is not None]
        if inits and hvd.size() > 1:
            hvd.communicator().broadcast_(inits, root=0)
        optimizer = self.make_optimizer(model, args)
        hvd.broadcast_optimizer_state(optimizer, root_rank=0)
        comp = {"none": hvd.Compression.none, "fp16": hvd.Compression.fp16, "bf16": hvd.Compression.bf16}[args.compression]
        if device.type != "cuda":
            comp = hvd.Compression.none
        # --accum-steps N: horovod's own backward_passes_per_step (the gradients add up in p.grad, reduced every N-th pass)
        n = self.set_accum_steps(args)
        if n > 2:
            # the gradients accumulate in p.grad through autograd, which a replayed graph cannot continue from a pass
            # captured with p.grad already set (first pass of a step) or not (the others): keep such steps eager
            self.graph_capable = False
        optimizer = hvd.DistributedOptimizer(optimizer, named_parameters=model.named_parameters(), compression=comp,
                                             backward_passes_per_step=n)
        self.comm = hvd.communicator()
        self.engine = getattr(optimizer, "_ptd_engine_obj", None)
        return model, optimizer

    def clip_and_step(self, optimizer, max_norm):
        """horovod's clipping idiom: reduce, clip, then step without reducing again."""
        optimizer.synchronize()
        self._note_clip(torch.nn.utils.clip_grad_norm_([p for g in optimizer.param_groups for p in g["params"]], max_norm), max_norm)
        with optimizer.skip_synchronize():
            optimizer.step()


class DataParallelStrategy(Strategy):
    """/root/reference/dataparallel.py: one process drives every GPU."""
    name = "dataparallel"
    distributed = False
    shard_batch = False
    reduce_metrics = False
    graph_capable = False       # replica forwards run on host threads across devices
    overlap_optimizer = False   # one reduce at the end of backward (K5): nothing to ride behind
    epoch_csv = "dataparallel.csv"

    def init_process_group(self, args, local_rank, nprocs):
        pass

    def build_model(self, model, args, device, local_rank):
        from .parallel.dp import DataParallel
        if args.gpus:
            gpus = [int(g) for g in args.gpus.split(",")]
        else:
            gpus = list(range(torch.cuda.device_count())) if device.type == "cuda" else []
        model = self.prepare_model(model, args, device)
        if self.set_accum_steps(args) > 1:
            raise ValueError("--accum-steps needs one process per GPU; DataParallel does not support it")
        model = DataParallel(model, device_ids=gpus, output_device=gpus[0] if gpus else None,
                             compute_dtype=self.input_dtype if self.autocast is None else None)
        self.comm = None
        self.engine = model.engine
        optimizer = self.make_optimizer(model, args)
        return model, optimizer


class SlurmStrategy(Strategy):
    """/root/reference/distributed_slurm_main.py (global-rank-0 checkpoint guard instead of every rank, Q11)."""
    name = "distributed_slurm_main"
    epoch_csv = "distributed.csv"


STRATEGIES = {
    "distributed": Strategy,
    "multiprocessing_distributed": Strategy,
    "apex_distributed": ApexStrategy,
    "horovod_distributed": HorovodStrategy,
    "dataparallel": DataParallelStrategy,
    "distributed_slurm_main": SlurmStrategy,
}


def apply_sync_bn(model, args, st, device):
    """``--sync-bn``: every BatchNorm layer becomes a synchronised one (``models.resnet.convert_sync_batchnorm``) before the
    strategy casts and wraps the model."""
    if not getattr(args, "sync_bn", False):
        return model
    if not st.distributed:
        raise ValueError("--sync-bn needs one process per GPU; like torch.nn.SyncBatchNorm it does not support DataParallel")
    kind = st.comm_kind(args, device)
    if args.cuda_graph and kind != "fused":
        raise ValueError("--sync-bn with --comm %s synchronises BatchNorm through torch.distributed, which a CUDA graph cannot "
                         "capture; use --comm fused or drop --cuda-graph" % kind)
    if args.cuda_graph and (args.fused_bn is False or args.channels_last is False):
        raise ValueError("--sync-bn with --no-fused-bn / --no-channels-last synchronises BatchNorm through torch.distributed, "
                         "which a CUDA graph cannot capture; drop --cuda-graph")
    from .models.resnet import convert_sync_batchnorm
    return convert_sync_batchnorm(model)


# ====================================================================== the worker
def main_worker(local_rank: int, nprocs: int, args, strategy: Optional[Strategy] = None):
    """/root/reference/distributed.py:129-225 (shared by every entrypoint)."""
    st = strategy or STRATEGIES[args.entry]()
    best_acc1 = 0.0
    device = pick_device(args, local_rank)
    args.local_rank = local_rank
    st.init_process_group(args, local_rank, nprocs)
    world = st.world() if st.distributed else 1

    model = create_model(args.arch, pretrained=args.pretrained, num_classes=args.num_classes, fused_bn=args.fused_bn)
    model = apply_sync_bn(model, args, st, device)
    # per-process batch: "-b" is the total over the node (reference :146); DataParallel keeps the full batch (:166)
    args.total_batch_size = args.batch_size
    if st.shard_batch:
        args.batch_size = max(1, int(args.batch_size / world))
    model, optimizer = st.build(model, args, device, local_rank)
    criterion = nn.CrossEntropyLoss().to(device)
    bm = getattr(st, "batch_mix", None)
    val_criterion = bm.criterion if bm is not None else criterion     # validation: label smoothing, never mixing
    torch.backends.cudnn.benchmark = True

    train_loader, val_loader, train_sampler, val_sampler = build_loaders(args, args.batch_size, distributed=st.distributed,
                                                                        raw_uint8=st.raw_uint8_loader)
    if args.resume:
        ck = load_checkpoint(args.resume, st.unwrapped(model), optimizer, engine=getattr(st, "engine", None))
        if ck.get("amp") and hasattr(st, "amp"):
            st.amp.load_state_dict(ck["amp"])
        args.start_epoch = ck.get("epoch", args.start_epoch)
        best_acc1 = float(ck.get("best_acc1", 0.0))
        print("=> loaded checkpoint '{}' (epoch {})".format(args.resume, args.start_epoch))
    ema = getattr(st, "model_ema", None)
    if ema is not None and args.resume:
        if ck.get("state_dict_ema") is not None:
            ema.load_state_dict(ck["state_dict_ema"])
        else:
            ema.reset()
            if not st.distributed or st.rank() == 0:
                print("=> no state_dict_ema in checkpoint '{}': the EMA starts from the resumed weights".format(args.resume))

    if args.evaluate:
        validate(val_loader, model, val_criterion, st, device, args)
        if ema is not None:
            validate_ema(ema, val_loader, val_criterion, st, device, args)
        _shutdown(st)
        return

    for epoch in range(args.start_epoch, args.epochs):
        t_epoch = time.time()
        train_sampler.set_epoch(epoch)
        val_sampler.set_epoch(epoch)
        if bm is not None:
            bm.set_epoch(epoch)
        if getattr(st, "batch_augment", None) is not None:
            st.batch_augment.set_epoch(epoch)
        adjust_learning_rate(optimizer, epoch, args)
        train(train_loader, model, criterion, optimizer, epoch, st, device, args)
        acc1 = validate(val_loader, model, val_criterion, st, device, args)
        if ema is not None:
            validate_ema(ema, val_loader, val_criterion, st, device, args)
        is_best = acc1 > best_acc1          # model_best follows the live model's Acc@1
        best_acc1 = max(acc1, best_acc1)
        if st.epoch_csv and st.is_saver(args):
            with open(os.path.join(args.checkpoint_dir, st.epoch_csv), "a+", newline="") as f:
                csv.writer(f).writerow([time.strftime("%Y-%m-%d %H:%M:%S", time.localtime(t_epoch)), time.time() - t_epoch])
        if st.is_saver(args):
            state = {
                "epoch": epoch + 1,
                "arch": args.arch,
                "state_dict": export_state_dict(st.unwrapped(model), getattr(st, "engine", None), optimizer),
                "best_acc1": best_acc1,
                "optimizer": optimizer.state_dict() if args.resume or os.environ.get("PTD_SAVE_OPTIMIZER") else None,
                "amp": st.amp.state_dict() if hasattr(st, "amp") else None,      # loss-scaler state (apex entrypoint)
            }
            if ema is not None:
                state["state_dict_ema"] = export_ema_state_dict(ema)
            save_checkpoint(state, is_best, directory=args.checkpoint_dir)
    _shutdown(st)


def make_model_ema(model, optimizer, args):
    """``--model-ema``: the ModelEma of the unwrapped model, attached to the optimizer (None without the flag)."""
    if not getattr(args, "model_ema", False):
        return None
    from .utils.ema import ModelEma
    return ModelEma(model, decay=args.model_ema_decay, optimizer=optimizer)


def make_batch_mix(args, device, rank: int):
    """``--label-smoothing`` / ``--mixup-alpha`` / ``--cutmix-alpha``: the BatchMix of this rank (None when all three are 0)."""
    eps, mix, cut = (float(getattr(args, k, 0.0) or 0.0) for k in ("label_smoothing", "mixup_alpha", "cutmix_alpha"))
    if not (eps or mix or cut):
        return None
    from .ops.mix import BatchMix
    return BatchMix(mix, cut, eps, num_classes=args.num_classes, seed=args.seed, rank=rank, device=device)


def make_batch_augment(args, device, rank: int):
    """``--auto-augment`` / ``--random-erase``: the BatchAugment of this rank (None when both are off)."""
    policy, p = getattr(args, "auto_augment", None), float(getattr(args, "random_erase", 0.0) or 0.0)
    if policy is None and not p:
        return None
    from .ops.augment import BatchAugment
    return BatchAugment(policy, p, seed=args.seed, rank=rank)


def validate_ema(ema, val_loader, criterion, st, device, args):
    """Validate the averaged weights: ``ema.module`` (DataParallel: on its first device alone, without replicas)."""
    ema.sync_module()
    return validate(val_loader, ema.module, criterion, st, device, args, tag="EMA")


class _DeviceStepTimer:
    """Device-timed seconds per training step: one CUDA event per print interval, read after the metric drain has
    synchronised with the device anyway (no extra stall)."""

    def __init__(self, device):
        self.enabled = device.type == "cuda"
        self.prev = None
        self.prev_i = 0

    def lap(self, i):
        if not self.enabled:
            return 0.0, 0
        ev = torch.cuda.Event(enable_timing=True)
        ev.record()
        ev.synchronize()
        out = (0.0, 0)
        if self.prev is not None and i > self.prev_i:
            n = i - self.prev_i
            out = (self.prev.elapsed_time(ev) / 1e3 / n, n)
        self.prev, self.prev_i = ev, i
        return out


def _test_kill_step(st) -> int:
    """PTD_TEST_KILL_RANK / PTD_TEST_KILL_STEP: failure-injection hook used by the kill-a-rank tests."""
    r = os.environ.get("PTD_TEST_KILL_RANK")
    if r is None or int(r) != (st.rank() if st.distributed else 0):
        return -1
    return int(os.environ.get("PTD_TEST_KILL_STEP", "3"))


def _raise_with_comm_diagnosis(st, err):
    """A peer that never arrives makes the waiting kernel trap after PTD_COMM_TIMEOUT_MS (csrc/common.cuh) and leaves a status
    word in host-mapped memory; the CUDA context is gone after that, so every later call fails with an unrelated-looking
    error.  Turn that into ONE clear message and leave without touching CUDA / the process group again."""
    comm = getattr(st, "comm", None)
    status = 0
    try:
        status = comm.arena.status() if comm is not None and hasattr(comm, "arena") else 0
    except Exception:  # noqa: BLE001
        pass
    if status:
        import sys
        rank = st.rank() if st.distributed else 0
        sys.stderr.write("[ptd] rank %d: a fused collective timed out waiting for a peer (status 0x%08x, timeout %s ms): a peer process "
                         "died or hung. Aborting this rank; the launcher tears the job down.\n  original error: %s\n" %
                         (rank, status, os.environ.get("PTD_COMM_TIMEOUT_MS", "120000"), str(err).splitlines()[0] if str(err) else type(err).__name__))
        sys.stderr.flush()
        os._exit(3)
    raise err


def _shutdown(st):
    comm = getattr(st, "comm", None)
    if comm is not None:
        comm.check()
    if torch.cuda.is_available():
        torch.cuda.synchronize()
    if st.distributed and dist.is_initialized():
        dist.barrier()
        dist.destroy_process_group()


def _log_jsonl(args, rec):
    if args.log_jsonl:
        with open(args.log_jsonl, "a") as f:
            f.write(json.dumps(rec) + "\n")


def train(train_loader, model, criterion, optimizer, epoch, st: Strategy, device, args):
    """/root/reference/distributed.py:228-276"""
    batch_time = AverageMeter("Time", ":6.3f")
    data_time = AverageMeter("Data", ":6.3f")
    losses = AverageMeter("Loss", ":.4e")
    top1 = AverageMeter("Acc@1", ":6.2f")
    top5 = AverageMeter("Acc@5", ":6.2f")
    accum = int(getattr(args, "accum_steps", 1) or 1)
    limit = args.steps_per_epoch
    if accum > 1:
        # whole optimizer steps only: a group of micro-batches never crosses an epoch (or the checkpoint written after it)
        n = len(train_loader) if limit is None else min(len(train_loader), limit)
        limit = n // accum * accum
    pf = st.prefetcher(train_loader, device, args, limit=limit, augment=getattr(st, "batch_augment", None))
    progress = ProgressMeter(len(pf), [batch_time, data_time, losses, top1, top5], prefix="Epoch: [{}]".format(epoch))
    metrics = MetricPipeline(getattr(st, "comm", None), device, (losses, top1, top5), reduce=st.reduce_metrics)
    model.train()
    step = getattr(st, "_train_step", None)
    if step is None or step.model is not model:
        fused = getattr(getattr(st, "comm", None), "backend", "") == "fused"     # library collectives are not captured
        # a captured torch.optim.SGD step bakes the Python-float lr into the graph (the x0.1 decay at epochs 30/60 would be
        # ignored on replay): capture only with an optimizer whose hyper-parameters live on the device
        dev_hyper = hasattr(optimizer, "refresh_hyper")
        if args.cuda_graph and not (st.graph_capable and fused and dev_hyper) and not args.quiet and (not st.distributed or st.rank() == 0):
            print("=> --cuda-graph ignored: %s" % ("entrypoint is not capturable" if not st.graph_capable else
                                                  "library collectives are not captured" if not fused else
                                                  "--optimizer torch keeps lr on the host"))
        step = st._train_step = TrainStep(st, model, criterion, optimizer, metrics,
                                          use_graph=args.cuda_graph and st.graph_capable and fused and dev_hyper)
    step.metrics = metrics
    end = time.time()
    t0 = end
    n_img = n_batches = 0
    comm = getattr(st, "comm", None)
    timer = _DeviceStepTimer(device)
    kill_at = _test_kill_step(st)
    try:
        for i, (images, target) in enumerate(pf):
            data_time.update(time.time() - end)
            step(images, target)
            n_img += images.size(0)
            n_batches += 1
            if not timer.enabled:
                batch_time.update(time.time() - end)      # CPU: the loop is synchronous, host time is step time
            end = time.time()
            if i == kill_at:
                os.kill(os.getpid(), 9)                    # test hook (tests/test_cpu_failure.py): this rank dies mid-epoch
            if i % args.print_freq == 0:
                metrics.drain()
                # The reference's Time meter was valid because .item() synchronised every iteration
                # (/root/reference/distributed.py:262,272).  Here nothing blocks the host (under --cuda-graph a step is one
                # launch), so Time is measured ON THE DEVICE: CUDA events bracket each print interval.
                dt, n = timer.lap(i)
                if n:
                    batch_time.update(dt, n)
                if comm is not None:
                    comm.check()                           # a peer that stopped arriving: fail now, not at shutdown
                if not args.quiet:
                    progress.display(i)
        metrics.drain()
    except RuntimeError as e:
        _raise_with_comm_diagnosis(st, e)
    if device.type == "cuda":
        torch.cuda.synchronize(device)
    rec = {"phase": "train", "epoch": epoch, "rank": st.rank() if st.distributed else 0, "images": n_img,
           "seconds": time.time() - t0, "loss": losses.avg, "acc1": top1.avg, "acc5": top5.avg}
    if accum > 1:
        rec.update(accum_steps=accum, optimizer_steps=n_batches // accum)
    if getattr(args, "clip_grad_norm", None) is not None:
        rec.update(st.clip_record(optimizer))
    _log_jsonl(args, rec)
    return losses.avg


def validate(val_loader, model, criterion, st: Strategy, device, args, tag: Optional[str] = None):
    """/root/reference/distributed.py:279-324 - distributed evaluation: sharded val set + metric all-reduce.
    ``tag="EMA"`` (``--model-ema``): the summary line reads `` * EMA Acc@1 ...`` and the JSONL phase ``val_ema``."""
    batch_time = AverageMeter("Time", ":6.3f")
    losses = AverageMeter("Loss", ":.4e")
    top1 = AverageMeter("Acc@1", ":6.2f")
    top5 = AverageMeter("Acc@5", ":6.2f")
    pf = st.prefetcher(val_loader, device, args, limit=args.val_steps or args.steps_per_epoch)
    progress = ProgressMeter(len(pf), [batch_time, losses, top1, top5], prefix="Test: " if tag is None else "Test %s: " % tag)
    metrics = MetricPipeline(getattr(st, "comm", None), device, (losses, top1, top5), reduce=st.reduce_metrics)
    model.eval()
    with torch.no_grad():
        end = time.time()
        for i, (images, target) in enumerate(pf):
            output = st.forward(model, images)
            loss = criterion(output.float() if output.dtype != torch.float32 else output, target)
            metrics.push(output, target, loss, images.size(0))
            metrics.poll()
            batch_time.update(time.time() - end)
            end = time.time()
            if i % args.print_freq == 0:
                metrics.drain()
                if not args.quiet:
                    progress.display(i)
        metrics.drain()
        # printed by every rank, like the reference (/root/reference/distributed.py:320-321)
        print(" *{tag} Acc@1 {top1.avg:.3f} Acc@5 {top5.avg:.3f}".format(tag="" if tag is None else " " + tag, top1=top1, top5=top5),
              flush=True)
    _log_jsonl(args, {"phase": "val" if tag is None else "val_" + tag.lower(), "rank": st.rank() if st.distributed else 0, "loss": losses.avg, "acc1": top1.avg, "acc5": top5.avg})
    return top1.avg
