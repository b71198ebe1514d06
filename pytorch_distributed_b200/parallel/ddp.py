"""DistributedDataParallel: one process per GPU, gradient buckets reduced during backward by the fused
peer-memory kernel (K1) instead of torch's C++ Reducer + NCCL.

API parity with the reference's use (/root/reference/distributed.py:147-148,223):
``DistributedDataParallel(model, device_ids=[local_rank])``, ``.module``, ``model(images)``, hooks fire inside
``loss.backward()``.  Behaviour parity with torch's Reducer defaults: rank-0 parameters/buffers are broadcast at
construction, float buffers are re-broadcast from rank 0 before every forward (``broadcast_buffers=True``), buckets
are 1 MiB (first) / ``bucket_cap_mb`` in reverse registration order, gradients are averaged.

H100-native design:
  * the wire format is a symmetric arena mapped into every peer (``parallel/comm.py``); bucket ``k`` owns a fixed
    range of it, so there is no flatten/copy-in: K1 reads the autograd-produced gradients through a pointer pack,
    casts (fp32 -> bf16), pre-scales by 1/world and reduces in ONE kernel per bucket on a high-priority side stream;
  * with :class:`~pytorch_distributed_b200.ops.fused_sgd.FusedSGD` the reduced arena is consumed in place by the
    optimizer kernel (no write-back pass into ``p.grad``);
  * small CTA counts (<= 32) + NVLS in-switch reduction keep the SMs for cuDNN while the bucket is in flight.
"""
from __future__ import annotations

import os
import weakref
from contextlib import contextmanager
from typing import List, Optional

import torch
import torch.distributed as dist
import torch.nn as nn

from . import plan as P
from ..utils.tensors import is_dense
from .comm import KIND_ONE_SHOT, KIND_TWO_SHOT, FusedCommunicator, make_communicator

_WIRE_OF = {torch.float32: "fp32", torch.bfloat16: "bf16", torch.float16: "fp16"}
# CTAs of one grad_accumulate / grad_fold launch (the bucket plan's CTAs, each split over several): few enough to leave the
# SMs to the backward kernels the accumulation overlaps, enough to stream the bucket at a good share of HBM bandwidth
ACCUM_CTAS = int(os.environ.get("PTD_ACCUM_CTAS", "64"))


class _FlatState:
    """Flat optimizer-side buffers that share the gradient arena's layout."""

    def __init__(self, engine, master, momentum, model_copy):
        self.engine = engine
        self.master = master
        self.momentum = momentum
        self.model_copy = model_copy


class _Bucket:
    __slots__ = ("index", "param_ids", "plan", "pending", "launched", "elem_off", "region_elems", "one_shot", "views")

    def __init__(self, index, param_ids):
        self.index = index
        self.param_ids = param_ids
        self.plan = None
        self.pending = len(param_ids)
        self.launched = False
        self.elem_off = 0
        self.region_elems = 0
        self.one_shot = False
        self.views = None           # per-parameter views of the arena (gradient_as_bucket_view)


class GradientEngine:
    """Bucketed, overlapped gradient all-reduce over a list of parameters (shared by DDP / apex DDP).

    Everything cross-GPU runs on the communicator's side stream, in the same order on every rank; the compute stream
    only ever waits for it once, at the end of backward.  Per bucket (launched from the post-accumulate-grad hook of
    its last parameter):
      * K1 two-shot (``fused_allreduce_kernel``) or, for latency-bound sizes, K1b one-shot (``oneshot_allreduce_kernel``),
        picked per bucket from its size (``comm.ONE_SHOT_MAX_BYTES``);
      * ``bucket_view=True`` (torch's ``gradient_as_bucket_view``): ``p.grad`` are views of the arena, so an in-place
        accumulating backward leaves nothing to pack - K1 runs barrier -> multimem.ld_reduce/st -> barrier with the
        1/world scale applied to the reduced values;
      * with a bound flat optimizer in overlap mode the SGD update of the bucket's slice is enqueued right behind its
        all-reduce, so only the small tail bucket's all-reduce + update remain after the last gradient;
      * ``fp32_grad_accumulation=True`` (extension): a backward inside ``no_sync()`` adds each ready bucket's gradients
        into a rank-local fp32 accumulator with the arena's element layout (``grad_accumulate``, side stream) and drops
        ``p.grad``; the next synchronising backward folds the sum into each bucket's gradients (``grad_fold``, which also
        clears the accumulator) right before its all-reduce.  Nothing crosses GPUs before that last pass.
    """

    supports_flat_optimizer = True
    supports_overlap_optimizer = True

    def __init__(self, params: List[torch.nn.Parameter], comm, wire_dtype: str = "bf16", bucket_cap_mb: float = 25.0,
                 first_bucket_mb: float = 1.0, max_ctas: Optional[int] = None, check_inf: bool = False, average: bool = True,
                 order: str = "reverse", tail_bucket_mb: Optional[float] = 1.0, bucket_view: bool = False,
                 delay_allreduce: bool = False, scale: Optional[float] = None, fp32_grad_accumulation: bool = False):
        self.comm = comm
        self.world = comm.world
        self.fused = isinstance(comm, FusedCommunicator)
        self.params = [p for p in params if p.requires_grad]
        self.wire = wire_dtype
        self.check_inf = check_inf
        self.average = average
        self.scale = scale if scale is not None else ((1.0 / self.world) if average else 1.0)
        self.writeback = True           # flipped off when a flat FusedSGD consumes the arena directly / with bucket views
        self.enabled = True             # no_sync()
        self.fp32_accum = bool(fp32_grad_accumulation)
        self._accumulating = False      # the running backward is a no_sync pass that adds into the fp32 accumulator
        self.accum_pending = False      # the accumulator holds passes that no synchronising backward has folded yet
        self.delay_allreduce = delay_allreduce
        self.bucket_view = bool(bucket_view) and self.fused
        self._flat: Optional[_FlatState] = None
        self._overlap_opt = None        # FusedSGD in overlap mode: applies its update per bucket, behind the all-reduce
        self._callback_queued = False
        self._pending_finish = []       # TorchCommunicator async handles
        self._keepalive = []            # tensors a side-stream kernel still reads (released after the join)
        self._grads_ready_event = None
        self._next_bucket = 0
        esz = P.WIRE_BYTES[wire_dtype]
        if bucket_view and self.fused:
            bad = [p.dtype for p in self.params if _WIRE_OF.get(p.dtype) != wire_dtype]
            if bad:
                raise ValueError("gradient_as_bucket_view needs gradients in the wire dtype (%s); found %s - pass "
                                 "wire_dtype=... or cast the model" % (wire_dtype, sorted({str(d) for d in bad})))
        ids = list(range(len(self.params)))
        if order == "reverse":
            ids = ids[::-1]             # gradients become ready roughly in reverse registration order
        numels = [self.params[i].numel() for i in ids]
        max_t = 256
        tail = int(tail_bucket_mb * (1 << 20)) if tail_bucket_mb else None
        groups = P.compute_buckets(numels, esz, int(bucket_cap_mb * (1 << 20)), int(first_bucket_mb * (1 << 20)), max_t, tail)
        self.buckets = [_Bucket(k, [ids[j] for j in g]) for k, g in enumerate(groups)]
        self.bucket_of = {}
        for b in self.buckets:
            for pid in b.param_ids:
                self.bucket_of[pid] = b
        self.param_elem_off = [0] * len(self.params)
        if self.fused:
            from .comm import _VIEW_NAME, ONE_SHOT_MAX_BYTES
            self.stream = comm.side_stream
            self.channel = comm.new_channel()
            # one contiguous arena range for all buckets => the optimizer can treat it as a single flat tensor
            layouts = []
            # the last bucket runs after the last gradient with nothing left to hide behind: spread it over many CTAs
            # (32 KB each instead of 256 KB) so that its pack / reduce phases are short
            per_cta = [256 << 10] * len(self.buckets)
            if tail and len(self.buckets) > 1:
                per_cta[-1] = 32 << 10
            for k, b in enumerate(self.buckets):
                ns = [self.params[i].numel() for i in b.param_ids]
                offs, total = P.tensor_layout(ns)
                b.one_shot = self.world > 1 and total * esz <= ONE_SHOT_MAX_BYTES
                if b.one_shot:
                    per_cta[k] = 16 << 10      # latency-bound: many small CTA ranges, all requests in flight at once
                pc = per_cta[k]
                grid = P.choose_grid(total, esz, min(max_ctas or comm.max_ctas, comm.max_blocks), pc)
                layouts.append((ns, offs, total, P.build_layout(ns, self.world, grid, offs, total).region_elems))
            self.total_elems = sum(l[3] for l in layouts)
            self.arena_off = comm.alloc(self.total_elems * esz)
            cur = 0
            for b, (ns, offs, total, region), pc in zip(self.buckets, layouts, per_cta):
                b.elem_off, b.region_elems = cur, region
                # one-shot: the pack goes to a private double-buffered staging area, the reduced values land in the
                # bucket's slot of the gradient arena (result_off_bytes at launch)
                data_off = comm.alloc(2 * region * esz) if b.one_shot else self.arena_off + cur * esz
                b.plan = comm.make_plan(ns, wire_dtype, max_ctas=max_ctas, double_buffer=False, offsets=offs, total=total,
                                        data_off_bytes=data_off, bytes_per_cta=pc)
                assert b.plan.layout.region_elems == region
                for pid, o in zip(b.param_ids, offs):
                    self.param_elem_off[pid] = cur + o
                cur += region
            self._arena_flat = comm.arena.view(self.arena_off, self.total_elems, _VIEW_NAME[wire_dtype], 0)
            if self.bucket_view:
                self.writeback = False
                for b in self.buckets:
                    b.views = [self._arena_flat[self.param_elem_off[pid]:self.param_elem_off[pid] + self.params[pid].numel()]
                               .as_strided(self.params[pid].size(), self.params[pid].stride()) for pid in b.param_ids]
        else:
            self.stream = None
            self.total_elems = 0
        self._acc = None
        if self.fp32_accum:
            if self.fused:
                self._acc = torch.zeros(self.total_elems, dtype=torch.float32, device=comm.device)
            else:               # library collectives: the same sum with torch ops, parameters back to back
                offs = [0]
                for p in self.params:
                    offs.append(offs[-1] + p.numel())
                self._acc = torch.zeros(offs[-1], dtype=torch.float32, device=self.params[0].device)
                self._acc_views = [self._acc[o:o + p.numel()].view(p.shape) for o, p in zip(offs, self.params)]
        ref = weakref.ref(self)
        self._hooks = []
        for pid, p in enumerate(self.params):
            p._ptd_engine = ref
            p._ptd_index = pid
            self._hooks.append(p.register_post_accumulate_grad_hook(self._make_hook(pid)))

    # ------------------------------------------------------------------ flat optimizer binding
    def grad_arena(self) -> torch.Tensor:
        return self._arena_flat

    def bind_flat_optimizer(self, optimizer, params) -> Optional[_FlatState]:
        if not self.fused or self._flat is not None:
            return None
        if [id(p) for p in params] != [id(p) for p in self.params]:
            return None
        dtypes = {p.dtype for p in self.params}
        if len(dtypes) != 1:
            return None
        dt = dtypes.pop()
        dev = self.comm.device
        n = self.total_elems
        master = torch.zeros(n, dtype=torch.float32, device=dev)
        momentum = torch.zeros(n, dtype=torch.float32, device=dev)
        model_copy = None if dt == torch.float32 else torch.zeros(n, dtype=dt, device=dev)
        holder = master if model_copy is None else model_copy
        with torch.no_grad():
            for pid, p in enumerate(self.params):
                off, cnt = self.param_elem_off[pid], p.numel()
                if not is_dense(p):
                    return None
                view = holder[off:off + cnt].as_strided(p.size(), p.stride())
                view.copy_(p.data)
                if model_copy is not None:
                    init = getattr(p, "_ptd_master_init", None)     # fp32 values stashed by amp.cast_model
                    master[off:off + cnt].as_strided(p.size(), p.stride()).copy_(p.data.float() if init is None else init)
                    if init is not None:
                        del p._ptd_master_init
                p.data = view
                mview = momentum[off:off + cnt].as_strided(p.size(), p.stride())
                old = optimizer.state[p].get("momentum_buffer") if p in optimizer.state else None
                if old is not None:          # bound after a resume / after eager steps: keep the accumulated momentum
                    mview.copy_(old.to(mview.dtype))
                optimizer.state[p]["momentum_buffer"] = mview
        self._flat = _FlatState(self, master, momentum, model_copy)
        if not getattr(self, "bucket_view", False):      # (shared with the single-process DataParallel engine)
            self.writeback = False
        return self._flat

    def set_overlap_optimizer(self, optimizer) -> None:
        """``optimizer._apply_slice(elem_off, n)`` is enqueued on the side stream right behind each bucket's all-reduce."""
        self._overlap_opt = optimizer

    def master_params(self):
        """fp32 views of the master weights (== the parameters themselves unless a low-precision copy is in use)."""
        if self._flat is None or self._flat.model_copy is None:
            return [p.data for p in self.params]
        return [self._flat.master[self.param_elem_off[i]:self.param_elem_off[i] + p.numel()].as_strided(p.size(), p.stride())
                for i, p in enumerate(self.params)]

    # ------------------------------------------------------------------ backward-time machinery
    def _make_hook(self, pid):
        def hook(param):
            if not self.enabled and not self.fp32_accum:
                return
            if not self._callback_queued:
                torch.autograd.Variable._execution_engine.queue_callback(self._finalize)
                self._callback_queued = True
                self._accumulating = not self.enabled
            b = self.bucket_of[pid]
            b.pending -= 1
            if b.pending == 0 and not self.delay_allreduce:
                self._launch_ready()
        return hook

    def _launch_ready(self):
        while self._next_bucket < len(self.buckets) and self.buckets[self._next_bucket].pending == 0:
            self._launch(self.buckets[self._next_bucket])
            self._next_bucket += 1

    def _bucket_grads(self, b):
        grads = []
        for k, pid in enumerate(b.param_ids):
            p = self.params[pid]
            if p.grad is None:      # parameter unused in this iteration: contributes zeros
                if b.views is not None:
                    b.views[k].zero_()
                    p.grad = b.views[k]
                else:
                    p.grad = torch.zeros_like(p, memory_format=torch.preserve_format)
            g = p.grad
            if not is_dense(g):
                g = g.contiguous()
                p.grad = g
            grads.append(g)
        return grads

    def _accumulate(self, b, grads, fold: bool):
        """``grad_accumulate`` (acc += g) or ``grad_fold`` (g = round(acc + g), acc = 0) over one bucket, on the current stream."""
        if self.fused:
            from .. import _ext
            _ext.note_launch()
            fn = _ext.lib().grad_fold if fold else _ext.lib().grad_accumulate
            pl = b.plan
            fn(grads, pl.seg_begin, pl.segs, pl.grid, max(1, ACCUM_CTAS // pl.grid), self._acc, b.elem_off, b.region_elems)
            return
        with torch.no_grad():
            for pid, g in zip(b.param_ids, grads):
                acc = self._acc_views[pid]
                if fold:
                    g.copy_((acc + g.float()).to(g.dtype))
                    acc.zero_()
                else:
                    acc.add_(g.float())

    def _launch(self, b):
        grads = self._bucket_grads(b)
        if self._accumulating:
            if self.fused:
                ev = torch.cuda.Event()
                ev.record()
                self.stream.wait_event(ev)
                with torch.cuda.stream(self.stream):
                    self._accumulate(b, grads, fold=False)
                self._keepalive.append(grads)       # read on the side stream: released after the end-of-backward join
            else:
                self._accumulate(b, grads, fold=False)
            b.launched = True
            return
        fold = self.accum_pending
        if self.fused:
            # bucket views + in-place accumulation: every gradient already sits in its arena slot => nothing to pack
            prepacked = (b.views is not None and not b.one_shot
                         and all(g.data_ptr() == v.data_ptr() for g, v in zip(grads, b.views)))
            opt = self._overlap_opt
            if opt is not None and b.index == 0:
                opt._prepare_overlap()          # hyper-parameters to the device, on the compute stream, before the fork
            ev = torch.cuda.Event()
            ev.record()
            self.stream.wait_event(ev)
            with torch.cuda.stream(self.stream):
                if fold:
                    self._accumulate(b, grads, fold=True)
                esz = P.WIRE_BYTES[self.wire]
                self.comm.run(b.plan, grads, KIND_ONE_SHOT if b.one_shot else KIND_TWO_SHOT, self.channel, scale=self.scale,
                              writeback=self.writeback, check_inf=self.check_inf, prepacked=prepacked,
                              result_off_bytes=(self.arena_off + b.elem_off * esz) if b.one_shot else -1)
                if opt is not None:
                    opt._apply_slice(b.elem_off, b.region_elems)
            if b.views is not None:
                if not prepacked:
                    # the autograd-produced gradients are still being read by the pack pass on the side stream: re-pointing
                    # p.grad drops their last reference, and the allocator would hand the memory to the next backward kernel
                    # on the compute stream at once - keep them alive until the end-of-backward join
                    self._keepalive.append(grads)
                for pid, v in zip(b.param_ids, b.views):    # torch semantics: after the reduction p.grad IS the bucket view
                    self.params[pid].grad = v
        else:
            if fold:
                self._accumulate(b, grads, fold=True)
            fin = self.comm.all_reduce_(grads, average=self.average, wire=self.wire, async_op=True)
            if fin is not None:
                self._pending_finish.append(fin)
        b.launched = True

    def _finalize(self):
        """End of backward: flush stragglers, then make the compute stream wait for the comm stream."""
        self._callback_queued = False
        if self._next_bucket < len(self.buckets):
            for b in self.buckets[self._next_bucket:]:
                b.pending = 0
            self._launch_ready()
        if self.fused:
            ev = torch.cuda.Event()
            ev.record(self.stream)
            self._grads_ready_event = ev
            torch.cuda.current_stream().wait_event(ev)
            self._keepalive.clear()
        else:
            for fin in self._pending_finish:
                fin()
            self._pending_finish.clear()
        for b in self.buckets:
            b.pending = len(b.param_ids)
            b.launched = False
        self._next_bucket = 0
        if self._accumulating:
            # the pass lives in the accumulator now: a later backward must not add it again through p.grad
            for p in self.params:
                p.grad = None
            self._accumulating = False
            self.accum_pending = True
        else:
            self.accum_pending = False

    def wait_for_gradients(self):
        if self._grads_ready_event is not None and not torch.cuda.is_current_stream_capturing():
            torch.cuda.current_stream().wait_event(self._grads_ready_event)

    def reduce_now(self):
        """Synchronously reduce whatever is in ``p.grad`` (used after ``no_sync`` accumulation or by tests)."""
        for b in self.buckets:
            b.pending = 0
        self._next_bucket = 0
        self._finalize()

    def zero_grads(self) -> bool:
        """Bucket views only: clear every gradient with ONE memset of the arena (instead of one fill per parameter) and keep
        ``p.grad`` pointing at the views, so the next backward accumulates in place.  Returns False when not applicable."""
        if not self.bucket_view:
            return False
        self._arena_flat.zero_()
        for b in self.buckets:
            for pid, v in zip(b.param_ids, b.views):
                self.params[pid].grad = v
        return True

    def remove_hooks(self):
        for h in self._hooks:
            h.remove()
        self._hooks = []


def _float_buffers(module):
    return [b for b in module.buffers() if b.is_floating_point()]


def sync_module_states(module: nn.Module, comm, root: int = 0) -> None:
    """Make every rank start from rank ``root``'s parameters and buffers (torch DDP ctor semantics)."""
    if comm.world == 1:
        return
    with torch.no_grad():
        tensors = [p.data for p in module.parameters()] + _float_buffers(module)
        comm.broadcast_(tensors, root=root)
        # fp32 values stashed by amp.cast_model become the master weights: they must be rank `root`'s as well, or every
        # rank would run root's low-precision model over its OWN masters and diverge after the first step
        inits = [p._ptd_master_init for p in module.parameters() if getattr(p, "_ptd_master_init", None) is not None]
        if inits:
            comm.broadcast_(inits, root=root)
        ints = [b for b in module.buffers() if not b.is_floating_point()]
        if ints and dist.is_initialized():
            for b in ints:
                dist.broadcast(b, src=root, group=comm.group)


class DistributedDataParallel(nn.Module):
    """``torch.nn.parallel.DistributedDataParallel`` surface over :class:`GradientEngine`.

    Constructor arguments with torch's meaning: ``device_ids`` (checked against the module's device), ``broadcast_buffers``,
    ``process_group``, ``bucket_cap_mb``, ``gradient_as_bucket_view`` (``p.grad`` become views of the symmetric arena: no
    write-back pass, and no pack pass either when the gradients are accumulated in place - ``zero_grad(set_to_none=False)``
    or ``engine.zero_grads()``).  ``fp32_grad_accumulation`` (extension): backwards inside ``no_sync()`` sum into an fp32
    buffer instead of ``p.grad`` (which they leave None); the next backward outside it folds the sum in and reduces it.
    ``find_unused_parameters`` is accepted and always effectively on: a bucket whose
    parameters did not all receive a gradient is flushed at the end of backward with zeros for the missing ones, no
    graph traversal needed.  ``output_device`` / ``dim`` other than the module's device / 0 are rejected (single-device
    module replicas only, like the reference's use).
    """

    def __init__(self, module: nn.Module, device_ids=None, output_device=None, dim=0, broadcast_buffers: bool = True,
                 process_group=None, bucket_cap_mb: float = 25.0, find_unused_parameters: bool = False,
                 gradient_as_bucket_view: bool = False, comm="auto", wire_dtype: Optional[str] = None, max_ctas: Optional[int] = None,
                 check_inf: bool = False, tail_bucket_mb: Optional[float] = 1.0, deferred_buffer_broadcast: Optional[bool] = None,
                 fp32_grad_accumulation: bool = False):
        super().__init__()
        self.module = module
        params = [p for p in module.parameters() if p.requires_grad]
        if not params:
            raise RuntimeError("DistributedDataParallel is not needed when a module doesn't have any parameter that requires a gradient.")
        self.device = params[0].device
        if device_ids is not None and self.device.type == "cuda":
            if len(device_ids) != 1:
                raise NotImplementedError("one device per process: device_ids must hold exactly one device (got %r)" % (device_ids,))
            d = device_ids[0]
            d = d.index if isinstance(d, torch.device) else int(d)
            if d != self.device.index:
                raise ValueError("device_ids %r does not match the module's device %s" % (device_ids, self.device))
        if dim != 0:
            raise NotImplementedError("DistributedDataParallel(dim=%r): only dim=0 is supported" % (dim,))
        if output_device is not None and self.device.type == "cuda":
            od = output_device.index if isinstance(output_device, torch.device) else int(output_device)
            if od != self.device.index:
                raise NotImplementedError("output_device must be the module's device (%s)" % (self.device,))
        self.broadcast_buffers = broadcast_buffers
        self.find_unused_parameters = find_unused_parameters
        if isinstance(comm, str):
            comm = make_communicator(comm, group=process_group, device=self.device)
        self.comm = comm
        from ..utils.dist_ops import register_for_sync_batchnorm
        register_for_sync_batchnorm(module, comm)
        if wire_dtype is None:
            if gradient_as_bucket_view and self.device.type == "cuda":
                wire_dtype = _WIRE_OF.get(params[0].dtype, "bf16")       # bucket views carry the gradients' own dtype
            else:
                wire_dtype = "bf16" if self.device.type == "cuda" else "fp32"
        sync_module_states(module, comm, root=0)
        self.engine = GradientEngine(params, comm, wire_dtype=wire_dtype, bucket_cap_mb=bucket_cap_mb, max_ctas=max_ctas,
                                     check_inf=check_inf, tail_bucket_mb=tail_bucket_mb, bucket_view=gradient_as_bucket_view,
                                     fp32_grad_accumulation=fp32_grad_accumulation)
        self._buffers_f = _float_buffers(module)
        # torch re-broadcasts rank 0's buffers BEFORE every forward, on the compute stream: a cross-GPU barrier at the top of
        # each step.  Deferred mode broadcasts rank 0's buffers right AFTER the forward that updated them, on the side stream
        # (it hides behind backward); the next forward therefore starts from rank 0's values exactly as with torch's order.
        if deferred_buffer_broadcast is None:
            deferred_buffer_broadcast = os.environ.get("PTD_DEFERRED_BCAST", "1") == "1"
        self._deferred = bool(deferred_buffer_broadcast) and isinstance(comm, FusedCommunicator)
        self._buffers_synced = False
        self._bcast_event = None

    def _broadcast_buffers_now(self):
        with torch.no_grad():
            self.comm.broadcast_(self._buffers_f, root=0)

    def forward(self, *inputs, **kwargs):
        sync = self.broadcast_buffers and self.comm.world > 1 and bool(self._buffers_f)
        capturing = self.device.type == "cuda" and torch.cuda.is_current_stream_capturing()
        if self._bcast_event is not None and not capturing:
            torch.cuda.current_stream().wait_event(self._bcast_event)      # the deferred broadcast of the previous forward
            self._bcast_event = None
        if not (sync and torch.is_grad_enabled()):
            return self.module(*inputs, **kwargs)
        if not self._deferred:
            self._broadcast_buffers_now()
            return self.module(*inputs, **kwargs)
        if not self._buffers_synced:                # very first training forward: establish rank 0's buffers everywhere
            self._broadcast_buffers_now()
            self._buffers_synced = True
        out = self.module(*inputs, **kwargs)
        side = self.comm.side_stream
        ev = torch.cuda.Event()
        ev.record()
        side.wait_event(ev)
        with torch.cuda.stream(side):
            self._broadcast_buffers_now()
            if not capturing:                       # inside a graph the end-of-backward join orders the next step
                done = torch.cuda.Event()
                done.record(side)
                self._bcast_event = done
        return out

    @contextmanager
    def no_sync(self):
        old = self.engine.enabled
        self.engine.enabled = False
        try:
            yield
        finally:
            self.engine.enabled = old

    def state_dict(self, *args, **kwargs):  # keys carry the "module." prefix exactly like torch DDP
        return super().state_dict(*args, **kwargs)
