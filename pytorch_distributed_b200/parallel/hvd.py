"""A from-scratch ``horovod.torch``-compatible module (the surface used by /root/reference/horovod_distributed.py).

    import pytorch_distributed_b200.parallel.hvd as hvd
    hvd.init(); hvd.local_rank(); hvd.size(); hvd.rank()                         (:125-127,147)
    hvd.broadcast_parameters(model.state_dict(), root_rank=0)                    (:149)
    hvd.broadcast_optimizer_state(optimizer, root_rank=0)                        (:158)
    optimizer = hvd.DistributedOptimizer(optimizer, named_parameters=..., compression=hvd.Compression.fp16)  (:159-164)
    hvd.allreduce(tensor, name='barrier')                                        (:104)

Design (H100-native, not a horovod port):
  * control plane: ``torch.distributed`` (env:// under torchrun, or the self-spawn launcher) - there is no MPI here;
  * per-parameter hooks enqueue into the C++ :class:`FusionQueue` (``csrc/hvd_core.cpp``); a dispatcher thread pops
    closed fusion groups and launches ONE fused cast(fp32->fp16 "compression") + all-reduce + decompress kernel per
    group on a side stream - the fusion buffer IS the symmetric NVLink arena, so there is no copy-in/copy-out;
  * ``optimizer.step()`` first ``synchronize()``s (flush + wait), exactly where horovod waits for its handles.
Deviation (SURVEY Q4): ``allreduce`` really returns the averaged tensor (the reference discards the return value).
"""
from __future__ import annotations

import atexit
import os
import threading
import time
from typing import Dict, Iterable, Optional, Tuple

import torch
import torch.distributed as dist

from ..utils.tensors import is_dense
from .comm import KIND_TWO_SHOT, FusedCommunicator, make_communicator

_state = {"init": False, "comm": None, "device": None, "handles": {}, "next": 1}
_lock = threading.Lock()


# ---------------------------------------------------------------------- basics
def init(comm: Optional[str] = None, device: Optional[str] = None) -> None:
    if _state["init"]:
        return
    use_cuda = torch.cuda.is_available() and (device is None or str(device).startswith("cuda"))
    if not dist.is_initialized():
        if "RANK" in os.environ and "WORLD_SIZE" in os.environ:
            backend = "nccl" if use_cuda else "gloo"
            if use_cuda:
                torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
                dist.init_process_group(backend, device_id=torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0"))))
            else:
                dist.init_process_group(backend)
    _state["device"] = torch.device("cuda", local_rank()) if use_cuda else torch.device("cpu")
    if use_cuda:
        torch.cuda.set_device(_state["device"])
    _state["comm"] = make_communicator(comm or "auto", device=_state["device"])
    _state["init"] = True


def shutdown() -> None:
    _state.update(init=False, comm=None)


def is_initialized() -> bool:
    return _state["init"]


def size() -> int:
    return dist.get_world_size() if dist.is_initialized() else 1


def rank() -> int:
    return dist.get_rank() if dist.is_initialized() else 0


def local_rank() -> int:
    return int(os.environ.get("LOCAL_RANK", rank() % max(1, torch.cuda.device_count() or 1)))


def local_size() -> int:
    return int(os.environ.get("LOCAL_WORLD_SIZE", size()))


def communicator():
    return _state["comm"]


def __getattr__(name):
    if name == "SyncBatchNorm":       # hvd.SyncBatchNorm (lazy: the models import this package's ops)
        from ..models.resnet import SyncBNAct
        return SyncBNAct
    raise AttributeError(name)


def nccl_built() -> bool:
    return False      # the data plane is hand-written peer-memory kernels, not NCCL


def mpi_enabled() -> bool:
    return False


class Compression:
    """Wire formats of the fused all-reduce ("compression" = cast inside the kernel, no extra pass)."""

    class none:  # noqa: N801
        wire = None

    class fp16:  # noqa: N801
        wire = "fp16"

    class bf16:  # noqa: N801
        wire = "bf16"


# reduction ops of horovod's `op=` argument (Adasum needs its own kernel and is not provided)
Average, Sum, Adasum = "average", "sum", "adasum"


def _op_average(op, average: bool) -> bool:
    if op is None:
        return bool(average)
    if op == Average:
        return True
    if op == Sum:
        return False
    raise NotImplementedError("hvd op %r is not supported (available: hvd.Average, hvd.Sum)" % (op,))


# ---------------------------------------------------------------------- tensor collectives
def _wire_for(t: torch.Tensor, compression) -> Optional[str]:
    w = getattr(compression, "wire", None)
    if t.device.type != "cuda":
        return None
    return w


def allreduce_(tensor: torch.Tensor, average: bool = True, name: Optional[str] = None, compression=Compression.none, op=None) -> torch.Tensor:
    average = _op_average(op, average)
    c = _state["comm"]
    if c is None or c.world == 1:
        return tensor
    if tensor.dtype == torch.float32 and tensor.numel() <= 8 and isinstance(c, FusedCommunicator) and tensor.is_contiguous():
        c.reduce_scalars_(tensor, average=average)     # latency path (metrics, "barrier" all-reduces)
    else:
        c.all_reduce_([tensor], average=average, wire=_wire_for(tensor, compression))
    return tensor


def allreduce(tensor: torch.Tensor, average: bool = True, name: Optional[str] = None, compression=Compression.none, op=None) -> torch.Tensor:
    return allreduce_(tensor.clone(), average=average, name=name, compression=compression, op=op)


def allgather(tensor: torch.Tensor, name: Optional[str] = None) -> torch.Tensor:
    """Concatenation of every rank's tensor along dim 0 (first dimensions may differ, like horovod).  Not on any hot path of
    the reference scripts: served by the library collective of the control plane."""
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return tensor.clone()
    sizes = [torch.zeros(1, dtype=torch.int64, device=tensor.device) for _ in range(size())]
    dist.all_gather(sizes, torch.tensor([tensor.size(0)], dtype=torch.int64, device=tensor.device))
    sizes = [int(s.item()) for s in sizes]
    mx = max(sizes)
    pad = tensor if tensor.size(0) == mx else torch.cat([tensor, tensor.new_zeros((mx - tensor.size(0),) + tuple(tensor.shape[1:]))])
    outs = [torch.empty_like(pad) for _ in sizes]
    dist.all_gather(outs, pad.contiguous())
    return torch.cat([o[:n] for o, n in zip(outs, sizes)])


def broadcast_object(obj, root_rank: int = 0, name: Optional[str] = None):
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return obj
    box = [obj]
    dist.broadcast_object_list(box, src=root_rank)
    return box[0]


def barrier() -> None:
    c = _state["comm"]
    if c is not None and c.world > 1:
        c.barrier()


def allreduce_async_(tensor: torch.Tensor, average: bool = True, name: Optional[str] = None) -> int:
    """Stream-ordered: the collective is enqueued immediately; the handle carries an event."""
    allreduce_(tensor, average=average, name=name)
    ev = None
    if tensor.is_cuda:
        ev = torch.cuda.Event()
        ev.record()
    with _lock:
        h = _state["next"]
        _state["next"] += 1
        _state["handles"][h] = (tensor, ev)
    return h


def allreduce_async(tensor, average=True, name=None) -> int:
    return allreduce_async_(tensor.clone(), average=average, name=name)


def poll(handle: int) -> bool:
    t, ev = _state["handles"][handle]
    return True if ev is None else ev.query()


def synchronize(handle: int) -> torch.Tensor:
    t, ev = _state["handles"].pop(handle)
    if ev is not None:
        torch.cuda.current_stream().wait_event(ev)
    return t


def broadcast_(tensor: torch.Tensor, root_rank: int, name: Optional[str] = None) -> torch.Tensor:
    c = _state["comm"]
    if c is not None and c.world > 1:
        if tensor.is_floating_point():
            c.broadcast_([tensor], root=root_rank)
        else:
            dist.broadcast(tensor, src=root_rank)
    return tensor


def broadcast(tensor, root_rank, name=None):
    return broadcast_(tensor.clone(), root_rank, name)


def broadcast_parameters(params, root_rank: int = 0) -> None:
    """Accepts ``model.state_dict()`` or ``model.named_parameters()`` (horovod semantics)."""
    c = _state["comm"]
    if c is None or c.world == 1:
        return
    items = list(params.items()) if isinstance(params, dict) else list(params)
    floats, others = [], []
    for _, t in items:
        if not torch.is_tensor(t):
            continue
        (floats if t.is_floating_point() else others).append(t.data if isinstance(t, torch.nn.Parameter) else t)
    with torch.no_grad():
        c.broadcast_(floats, root=root_rank)
        for t in others:
            dist.broadcast(t, src=root_rank)


def broadcast_optimizer_state(optimizer, root_rank: int = 0) -> None:
    """Scalars of the param groups and every tensor in ``optimizer.state`` follow rank ``root_rank``."""
    c = _state["comm"]
    if c is None or c.world == 1:
        return
    groups = [{k: v for k, v in g.items() if k != "params"} for g in optimizer.param_groups]
    box = [groups]
    dist.broadcast_object_list(box, src=root_rank)
    for g, src in zip(optimizer.param_groups, box[0]):
        g.update(src)
    tensors = []
    for g in optimizer.param_groups:
        for p in g["params"]:
            for v in optimizer.state.get(p, {}).values():
                if torch.is_tensor(v) and v.is_floating_point():
                    tensors.append(v)
    if tensors:
        c.broadcast_(tensors, root=root_rank)


# ---------------------------------------------------------------------- DistributedOptimizer
class _FusionEngine:
    """Hooks -> C++ FusionQueue -> dispatcher thread -> fused all-reduce per fusion group."""

    def __init__(self, named_params: Iterable[Tuple[str, torch.nn.Parameter]], comm, wire: Optional[str],
                 fusion_threshold_mb: float, cycle_time_ms: float, backward_passes_per_step: int = 1):
        from .. import _ext
        self.comm = comm
        self.fused = isinstance(comm, FusedCommunicator)
        self.named = [(n, p) for n, p in named_params if p.requires_grad]
        self.params = [p for _, p in self.named]
        self.index = {id(p): i for i, p in enumerate(self.params)}
        self.wire = wire
        self.passes = backward_passes_per_step
        self._counts = [0] * len(self.params)
        self._handles: Dict[int, int] = {}          # queue handle -> param index
        self._events: Dict[int, object] = {}
        self._plans = {}                            # response cache: tuple(param ids) -> Plan
        self._error = None
        self.enabled = True
        self.queue = None
        self.thread = None
        # Static schedule (default; PTD_HVD_STATIC=0 keeps the queue): group composition only depends on hook order and sizes,
        # so after the first complete step the recorded groups are frozen and the hooks launch them directly - no queue, no
        # dispatcher thread, and the step becomes capturable in a CUDA graph.  Until then requests go through the C++ fusion
        # queue, whose groups close at the cycle budget (so the very first steps overlap with backward as well).
        self._static_wanted = os.environ.get("PTD_HVD_STATIC", "1") == "1"
        self._trace = []            # groups (tuples of parameter indices) launched by the dispatcher during the current step
        self._schedule = None       # frozen trace
        self._group_of: Dict[int, int] = {}
        self._left = []
        self._next_static = 0
        self._fired = 0
        if comm.world > 1 or self.fused:
            C = _ext.lib() if self.fused or _ext.available() else None
            if C is not None:
                # horovod closes a fusion group every HOROVOD_CYCLE_TIME ms; here the tick is a byte budget (same groups on
                # every rank without a negotiation round): cycle_time_ms x PTD_HVD_BYTES_PER_MS (default 2 MiB/ms => 10 MiB)
                per_ms = float(os.environ.get("PTD_HVD_BYTES_PER_MS", 2 << 20))
                self.cycle_bytes = int(os.environ.get("PTD_HVD_CYCLE_BYTES", max(1.0, cycle_time_ms) * per_ms))
                self.queue = C.FusionQueue(int(fusion_threshold_mb * (1 << 20)), float(cycle_time_ms), self.cycle_bytes)
                self._timeline_path = os.environ.get("HOROVOD_TIMELINE", "")
                if self._timeline_path:
                    self.queue.enable_timeline(True)
        self._tuner = _Autotuner(self) if (self.queue is not None and os.environ.get("HOROVOD_AUTOTUNE", "0") == "1") else None
        if self.fused:
            self.stream = comm.side_stream
            self.channel = comm.new_channel()
        if self.queue is not None:
            self.thread = threading.Thread(target=self._dispatch_loop, name="ptd-hvd-cycle", daemon=True)
            self.thread.start()
            atexit.register(self.close)     # the thread must leave the C++ wait before the interpreter finalises
        self._hooks = [p.register_post_accumulate_grad_hook(self._make_hook(i)) for i, p in enumerate(self.params)]

    def _wire_bytes(self, p):
        return p.numel() * (2 if self.wire in ("fp16", "bf16") else p.element_size())

    def _make_hook(self, i):
        def hook(param):
            if not self.enabled or self.comm.world == 1 and not self.fused:
                return
            self._counts[i] += 1
            if self._counts[i] < self.passes:
                return
            self._counts[i] = 0
            if self._schedule is not None:          # static schedule: the last member of a group launches it
                self._fired += 1
                self._left[self._group_of[i]] -= 1
                self._launch_ready_static()
                return
            if self.queue is None:
                return
            ev = None
            if param.is_cuda:
                ev = torch.cuda.Event()
                ev.record()
            with _lock:        # enqueue may close the group and wake the dispatcher: the handle must be registered first
                h = self.queue.enqueue(self.named[i][0], self._wire_bytes(param), i)
                self._handles[h] = i
                self._events[h] = ev
        return hook

    def _launch_group(self, handles):
        with _lock:
            ids = [self._handles.pop(h) for h in handles]
            evs = [self._events.pop(h) for h in handles]
        self._trace.append(tuple(ids))
        self._reduce(ids, evs[-1])                  # events are stream-ordered: the last one covers the group

    def _reduce(self, ids, ready_event):
        """One fused all-reduce (cast -> reduce -> average -> write back) over the gradients of parameters ``ids``."""
        grads = []
        for i in ids:
            p = self.params[i]
            if p.grad is None:                      # unused in this step: contributes zeros, like every other rank's copy
                p.grad = torch.zeros_like(p, memory_format=torch.preserve_format)
            g = p.grad
            if not is_dense(g):
                g = g.contiguous()
                p.grad = g
            grads.append(g)
        if self.fused:
            own = "fp32" if grads[0].dtype == torch.float32 else ("bf16" if grads[0].dtype == torch.bfloat16 else "fp16")
            # "compression" = the wire dtype of the fused kernel; gradients that already are 16-bit travel as they are
            # (casting bf16 to fp16 would only lose range)
            wire = own if own != "fp32" else (self.wire or own)
            if ready_event is not None:
                self.stream.wait_event(ready_event)
            for lo in range(0, len(ids), 256):      # one kernel launch carries at most 256 tensor pointers
                sub_ids, sub = tuple(ids[lo:lo + 256]), grads[lo:lo + 256]
                plan = self._plans.get(sub_ids)     # response cache: the same fusion group recurs every step
                if plan is None:
                    plan = self.comm.make_plan([g.numel() for g in sub], wire)
                    self._plans[sub_ids] = plan
                with torch.cuda.stream(self.stream):
                    self.comm.run(plan, sub, KIND_TWO_SHOT, self.channel, scale=1.0 / self.comm.world, writeback=True)
        else:
            self.comm.all_reduce_(grads, average=True, wire=self.wire)

    # ------------------------------------------------------------------ static schedule
    def _freeze(self, groups):
        self._schedule = [tuple(g) for g in groups]
        self._group_of = {i: k for k, g in enumerate(self._schedule) for i in g}
        self._left = [len(g) for g in self._schedule]
        self._next_static = 0
        self._fired = 0

    def _launch_ready_static(self, force: bool = False):
        while self._next_static < len(self._schedule) and (force or self._left[self._next_static] == 0):
            ev = None
            if self.fused:
                ev = torch.cuda.Event()
                ev.record()                         # gradients of the group are complete on the current (compute) stream
            self._reduce(list(self._schedule[self._next_static]), ev)
            self._next_static += 1

    def _dispatch_loop(self):
        if self.fused:
            torch.cuda.set_device(self.comm.device)
        while True:
            handles = self.queue.next_group(50.0)
            if not handles:
                if self._stop:
                    return
                continue
            try:
                self._launch_group(handles)
            except Exception as e:  # noqa: BLE001 - surfaced by synchronize()
                self._error = e
                self.queue.wake()
            self.queue.mark_done(handles)

    _stop = False

    def synchronize(self):
        """Flush the open fusion group, wait until every request has been launched, join the comm stream."""
        if self._schedule is not None:
            if self._fired:                         # groups whose members did not all fire (unused parameters) go out now, in order
                self._launch_ready_static(force=True)
            self._left = [len(g) for g in self._schedule]
            self._next_static = 0
            self._fired = 0
            if self.fused:
                torch.cuda.current_stream().wait_stream(self.stream)
            return
        if self.queue is None:
            return
        self.queue.flush()
        while not self.queue.wait_idle(1000.0):      # condition variable in C++, GIL released: no polling
            if self._error is not None or self._stop:
                break
        if self._error is not None:
            e, self._error = self._error, None
            raise e
        if self.fused:
            torch.cuda.current_stream().wait_stream(self.stream)
        trace, self._trace = self._trace, []
        if self._tuner is not None and not self._tuner.done:
            self._tuner.step_done()                 # HOROVOD_AUTOTUNE: try the next cycle budget / pick the winner
            return
        if self._static_wanted and trace and sorted(i for g in trace for i in g) == list(range(len(self.params))):
            self._freeze(trace)                     # a complete step (every parameter exactly once): freeze its grouping

    def write_timeline(self):
        """HOROVOD_TIMELINE=<file>: chrome-trace JSON of the fusion queue (one slice per tensor from enqueue to dispatch,
        grouped by fusion group) - the part of horovod's timeline that exists here (there is no negotiation phase)."""
        path = getattr(self, "_timeline_path", "")
        if not path or self.queue is None:
            return
        import json
        recs = self.queue.timeline()
        if not recs:
            return
        evs = [{"name": n, "cat": "fusion", "ph": "X", "ts": t0, "dur": max(t1 - t0, 0.01), "pid": self.comm.rank, "tid": int(g) % 8,
                "args": {"bytes": b, "group": g}} for (n, b, g, t0, t1) in recs]
        base, ext = os.path.splitext(path)
        with open("%s.rank%d%s" % (base, self.comm.rank, ext or ".json"), "w") as f:
            json.dump({"traceEvents": evs, "stats": self.queue.stats()}, f)

    def close(self):
        self._stop = True
        try:
            self.write_timeline()
        except Exception:  # noqa: BLE001
            pass
        if self.queue is not None:
            self.queue.shutdown()
        if self.thread is not None and self.thread.is_alive() and threading.current_thread() is not self.thread:
            self.thread.join(timeout=5.0)
        self.thread = None
        for h in self._hooks:
            h.remove()
        self._hooks = []


class _Autotuner:
    """HOROVOD_AUTOTUNE=1: pick the fusion cycle budget by measurement.

    Horovod tunes fusion threshold and cycle time with Bayesian optimisation over many steps; here the only knob that
    changes the schedule is the byte budget at which a group closes, so a short deterministic sweep is enough: every
    candidate runs ``HOROVOD_AUTOTUNE_STEPS_PER_SAMPLE`` steps (after one settling step) timed with CUDA events, the
    per-candidate means are max-reduced over the ranks (every rank must pick the same winner), the best budget is set
    and - if the static schedule is enabled - the next step's groups are frozen.  All ranks switch candidates at the same
    step counts, so the groups stay identical across ranks throughout.
    """

    def __init__(self, engine, candidates_mb=(2, 4, 8, 16, 32, 64)):
        self.e = engine
        self.cands = [int(c * (1 << 20)) for c in candidates_mb]
        self.per = max(1, int(os.environ.get("HOROVOD_AUTOTUNE_STEPS_PER_SAMPLE", "5")))
        self.idx, self.count, self.done = 0, -1, False
        self.times = [0.0] * len(self.cands)
        self.ev = None
        self.log = os.environ.get("HOROVOD_AUTOTUNE_LOG", "")
        engine.queue.set_cycle_bytes(self.cands[0])

    def _now(self):
        if self.e.fused:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            return ev
        return time.perf_counter()

    def _elapsed_ms(self, a, b):
        if self.e.fused:
            b.synchronize()
            return a.elapsed_time(b)
        return (b - a) * 1e3

    def step_done(self):
        now = self._now()
        if self.count >= 0 and self.ev is not None:        # count == -1: the settling step after a switch is not timed
            self.times[self.idx] += self._elapsed_ms(self.ev, now)
        self.ev = now
        self.count += 1
        if self.count < self.per:
            return
        self.times[self.idx] /= self.per
        self.idx += 1
        self.count, self.ev = -1, None
        if self.idx < len(self.cands):
            self.e.queue.set_cycle_bytes(self.cands[self.idx])
            return
        t = torch.tensor(self.times, dtype=torch.float64, device=self.e.comm.device if self.e.fused else "cpu")
        if dist.is_initialized() and dist.get_world_size() > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        best = int(torch.argmin(t).item())
        self.e.cycle_bytes = self.cands[best]
        self.e.queue.set_cycle_bytes(self.cands[best])
        self.done = True
        if self.e.comm.rank == 0:
            msg = "[hvd autotune] cycle budget MiB -> ms/step: %s; picked %d MiB" % (
                ", ".join("%d: %.3f" % (c >> 20, x) for c, x in zip(self.cands, t.tolist())), self.cands[best] >> 20)
            print(msg, flush=True)
            if self.log:
                with open(self.log, "a") as f:
                    f.write(msg + "\n")


def DistributedOptimizer(optimizer, named_parameters=None, compression=Compression.none, backward_passes_per_step: int = 1,
                         op=None, fusion_threshold_mb: Optional[float] = None, cycle_time_ms: Optional[float] = None):
    """Wrap ``optimizer`` so that ``step()`` first completes the asynchronous gradient all-reduces (horovod semantics).

    Like horovod, this returns an instance of a dynamically created subclass of ``optimizer``'s class sharing its state.
    """
    if not _state["init"]:
        init()
    if not _op_average(op, True):
        raise NotImplementedError("DistributedOptimizer(op=hvd.Sum): gradients are averaged (horovod's default); scale the loss instead")
    comm = _state["comm"]
    if named_parameters is None:
        named_parameters = [("param.%d" % i, p) for i, p in enumerate(p for g in optimizer.param_groups for p in g["params"])]
    named_parameters = list(named_parameters)
    names = [n for n, _ in named_parameters]
    if len(set(names)) != len(names):
        raise ValueError("named_parameters should consist of unique names")
    thr = fusion_threshold_mb if fusion_threshold_mb is not None else float(os.environ.get("HOROVOD_FUSION_THRESHOLD", 64 << 20)) / (1 << 20)
    cyc = cycle_time_ms if cycle_time_ms is not None else float(os.environ.get("HOROVOD_CYCLE_TIME", 5.0))
    wire = getattr(compression, "wire", None)
    if comm.device.type != "cuda":
        wire = None
    engine = _FusionEngine(named_parameters, comm, wire, thr, cyc, backward_passes_per_step)

    base = optimizer.__class__
    skip = [False]                      # inside skip_synchronize(): step() after an explicit synchronize() does not wait again

    class _DistributedOptimizer(base):  # type: ignore[misc,valid-type]
        def __init__(self):             # state is shared with the wrapped instance, not re-created
            pass

        def synchronize(self):
            engine.synchronize()

        def step(self, closure=None):
            if not skip[0]:
                engine.synchronize()
            return base.step(self, closure) if closure is not None else base.step(self)

        def skip_synchronize(self):
            """horovod's ``with optimizer.skip_synchronize(): optimizer.step()`` after ``optimizer.synchronize()`` and gradient
            surgery (clipping): the step does not synchronise a second time, which would count a second step in the autotuner."""
            import contextlib

            @contextlib.contextmanager
            def ctx():
                skip[0] = True
                try:
                    yield
                finally:
                    skip[0] = False
            return ctx()

    wrapped = _DistributedOptimizer.__new__(_DistributedOptimizer)
    wrapped.__dict__ = optimizer.__dict__
    wrapped._ptd_engine_obj = engine
    return wrapped
