"""Single-process multi-GPU data parallelism - the ``nn.DataParallel`` of /root/reference/dataparallel.py:138.

Call path parity (torch: scatter -> replicate -> parallel_apply -> gather, backward reduce-add onto GPU0):
    model = DataParallel(model, device_ids=gpus, output_device=gpus[0]);  output = model(images);  loss.backward()

H100-native redesign:
  * **persistent replicas** - ``replicate()``'s per-iteration Python module cloning is gone; each device owns a
    long-lived replica, only the *values* move;
  * **K2' broadcast** - one kernel on the root packs parameters + float buffers into its arena and multicasts them
    through NVSwitch (``multimem.st``; peer stores without NVLS) into every device's arena: root egress is N bytes,
    not (W-1)·N; replicas unpack locally;
  * **K5 gather-reduce** - after backward every device packs its gradients (cast to the wire dtype) into its arena,
    then the ROOT pulls the sum with ``multimem.ld_reduce`` (in-switch reduction; plain peer loads without NVLS) and
    either writes ``p.grad`` or leaves the flat result for :class:`FusedSGD`;
  * scatter uses the copy engines (SMs stay free), gather of the logits is one peer-load kernel on the root;
  * cross-device ordering is CUDA events only - one process, no flags, no host blocking;
  * **graphed replicas** - one Python process cannot enqueue 8 x ~900 kernels per step fast enough (that, not the
    interconnect, is why the reference's DataParallel is 3.5x slower than DDP): after two eager steps every replica's
    forward and backward are captured as CUDA graphs on its own device (``torch.cuda.make_graphed_callables``), so a step
    costs the host 2 graph launches per device plus the handful of engine kernels (``PTD_DP_GRAPH=0`` disables).
BN semantics follow torch (SURVEY Q14): only the root replica's running statistics persist.
"""
from __future__ import annotations

import copy
import os
import weakref
from concurrent.futures import ThreadPoolExecutor
from typing import List, Optional

import torch
import torch.nn as nn

from . import plan as P
from .comm import _VIEW_NAME, KIND_PACK, KIND_PUSH, KIND_REDUCE, KIND_UNPACK, Plan
from ..utils.tensors import is_dense
from .ddp import _FlatState


class LocalCommunicator:
    """Symmetric arenas of all local devices inside ONE process (VMM + optional multicast, see csrc/symm.cpp)."""

    backend = "fused-local"

    def __init__(self, devices: List[int], arena_bytes: int = 512 << 20, allow_nvls: bool = True):
        from .. import _ext
        self._C = _ext.lib()
        self._ext = _ext
        self.devices = list(devices)
        self.world = len(devices)
        self.rank = 0
        self.device = torch.device("cuda", devices[0])
        # the single-process kernels (pack / push / reduce-to-caller / unpack) carry no cross-GPU flags, so they are not bound by
        # the flag table (MAX_BLOCKS): two CTAs per SM keep enough multimem requests in flight to approach the link rate
        sms = torch.cuda.get_device_properties(devices[0]).multi_processor_count
        self.max_blocks = 2 * sms
        self.max_ctas = 2 * sms
        self.arena = self._C.SymmArena.create_local(self.devices, arena_bytes, allow_nvls)
        self.nvls = bool(self.arena.has_multicast)
        self.header_bytes = P.round_up(self._C.SIGNAL_PAD_BYTES, 128 << 10)
        self._bump = self.header_bytes

    def device_of(self, rank_slot: int = 0) -> torch.device:
        return torch.device("cuda", self.devices[rank_slot])

    def alloc(self, nbytes: int, align: int = 4096) -> int:
        off = P.round_up(self._bump, align)
        if off + nbytes > self.arena.bytes:
            raise RuntimeError("local symmetric arena exhausted; raise arena_bytes")
        self._bump = off + nbytes
        return off

    def check(self) -> None:
        pass

    def run(self, plan: Plan, tensors, kind: int, rank_slot: int, scale: float = 1.0, writeback: bool = True) -> None:
        """``tensors``: a list of tensors, or ``[pack]`` with a pointer pack from ``_C.pack_pointers`` (persistent lists)."""
        with torch.cuda.device(self.devices[rank_slot]):
            self._ext.note_launch()
            self.arena.launch_plan(0, rank_slot, kind, P.WIRE_CODES[plan.wire], self.nvls, plan.grid, tensors,
                                   plan.seg_begin.data_ptr(), plan.segs.data_ptr(), plan.data_off_bytes, plan.block_elems,
                                   plan.calls.data_ptr(), 0, float(scale), bool(writeback), 0)


class _TensorSet:
    """A list of same-role tensors on every device + per-device plans over one shared arena range."""

    def __init__(self, comm: LocalCommunicator, per_device: List[List[torch.Tensor]], wire: str, max_tensors: int = 256):
        self.comm = comm
        self.wire = wire
        self.per_device = per_device
        numels = [t.numel() for t in per_device[0]]
        esz = P.WIRE_BYTES[wire]
        groups = P.compute_buckets(numels, esz, 64 << 20, None, max_tensors) if numels else []
        self.groups = groups
        layouts = []
        for g in groups:
            ns = [numels[i] for i in g]
            offs, total = P.tensor_layout(ns)
            grid = P.choose_grid(total, esz, comm.max_ctas, 128 << 10)
            layouts.append((ns, offs, total, grid, P.build_layout(ns, comm.world, grid, offs, total).region_elems))
        self.total_elems = sum(l[4] for l in layouts)
        self.arena_off = comm.alloc(max(self.total_elems, 8) * esz)
        self.elem_off = [0] * len(numels)
        self.plans = []     # plans[group][device_slot]
        cur = 0
        for g, (ns, offs, total, grid, region) in zip(groups, layouts):
            row = [Plan(comm, ns, wire, grid, False, offsets=offs, total=total, data_off_bytes=self.arena_off + cur * esz, rank_slot=r,
                        bytes_per_cta=128 << 10) for r in range(comm.world)]
            self.plans.append(row)
            for i, o in zip(g, offs):
                self.elem_off[i] = cur + o
            cur += region

    def launch(self, kind: int, slot: int, scale: float = 1.0, writeback: bool = True, tensors=None, packs=None):
        """``packs``: per-group pointer packs from :meth:`make_packs` (skips the per-launch tensor-list marshalling)."""
        if packs is not None:
            for row, pk in zip(self.plans, packs):
                self.comm.run(row[slot], [pk], kind, slot, scale=scale, writeback=writeback)
            return
        ts = self.per_device[slot] if tensors is None else tensors
        for g, row in zip(self.groups, self.plans):
            self.comm.run(row[slot], [ts[i] for i in g], kind, slot, scale=scale, writeback=writeback)

    def make_packs(self, tensors):
        """Pointer packs (one per group) of a tensor list whose storage does not move."""
        C = self.comm._C
        return [C.pack_pointers([tensors[i] for i in g]) for g in self.groups]

    def flat(self, slot: int = 0) -> torch.Tensor:
        return self.comm.arena.view(self.arena_off, self.total_elems, _VIEW_NAME[self.wire], slot)


class _Gather(torch.autograd.Function):
    """Concatenate replica outputs on the root (one peer-load kernel); backward scatters the gradient slices."""

    @staticmethod
    def forward(ctx, engine, *outputs):
        ctx.engine = engine
        ctx.sizes = [o.size(0) for o in outputs]
        ctx.devices = [o.device for o in outputs]
        root = engine.root_device
        total = sum(ctx.sizes)
        out = torch.empty((total,) + tuple(outputs[0].shape[1:]), dtype=outputs[0].dtype, device=root)
        root_stream = torch.cuda.current_stream(root)
        srcs, dsts, off = [], [], 0
        for o, n in zip(outputs, ctx.sizes):
            if o.device != root:
                ev = torch.cuda.Event()
                with torch.cuda.device(o.device):
                    ev.record(torch.cuda.current_stream(o.device))
                root_stream.wait_event(ev)
            srcs.append(o.detach().contiguous())
            dsts.append(out[off:off + n])
            off += n
        engine.C.p2p_copy_multi(srcs, dsts, root.index)
        ctx.keep = srcs
        return out

    @staticmethod
    def backward(ctx, grad):
        engine = ctx.engine
        engine._arm_reduce()
        grads, off = [], 0
        for n, dev in zip(ctx.sizes, ctx.devices):
            g = grad[off:off + n]
            grads.append(g if dev == grad.device else g.to(dev, non_blocking=True))
            off += n
        return (None,) + tuple(grads)


class _ReplicaGraph:
    """Forward and backward of ONE replica as two CUDA graphs on its device, with static input / output / gradient buffers.

    Unlike ``torch.cuda.make_graphed_callables`` the parameter gradients never re-enter autograd: the backward graph leaves
    them in ``static_grads`` (fixed addresses), which the K5 pack reads directly - no per-parameter AccumulateGrad, no
    per-parameter Python at all in the steady state (8 replicas x 161 parameters of ResNet-50 cost the host milliseconds per
    step that way).
    """

    def __init__(self, module, params, sample, device, autocast_state):
        import contextlib
        self.device = device
        self.fresh = False
        with torch.cuda.device(device):
            def ctx():
                return (torch.autocast("cuda", dtype=autocast_state[1], cache_enabled=False) if autocast_state[0]
                        else contextlib.nullcontext())
            saved = [b.detach().clone() for b in module.buffers()]     # warm-up + capture run BatchNorm updates: undone below
            self.static_x = sample.detach().clone()
            self.token = torch.zeros((), device=self.static_x.device, requires_grad=True)   # ties the output into autograd
            stream = torch.cuda.Stream(device=device)                  # capture stream on THIS device
            stream.wait_stream(torch.cuda.current_stream(device))
            with torch.cuda.stream(stream):
                for _ in range(3):                                     # cuDNN autotuning, lazy workspaces
                    with ctx():
                        out = module(self.static_x)
                    g = torch.autograd.grad(out, params, torch.zeros_like(out), allow_unused=True)
                    del out, g
            stream.synchronize()
            pool = torch.cuda.graph_pool_handle()
            self.g_fwd = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.g_fwd, pool=pool, stream=stream):
                with ctx():
                    self.static_out = module(self.static_x)
            self.static_gout = torch.zeros_like(self.static_out)
            self.g_bwd = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.g_bwd, pool=pool, stream=stream):
                grads = torch.autograd.grad(self.static_out, params, self.static_gout, allow_unused=True)
            self.static_grads = [g if g is not None else torch.zeros_like(p) for g, p in zip(grads, params)]
            torch.cuda.current_stream(device).wait_stream(stream)
            with torch.no_grad():
                for b, old in zip(module.buffers(), saved):
                    b.copy_(old)
            self.shape, self.dtype = self.static_x.shape, self.static_x.dtype


class _Replay(torch.autograd.Function):
    @staticmethod
    def forward(ctx, rep, x, token):
        ctx.rep = rep
        with torch.cuda.device(rep.device):
            rep.static_x.copy_(x)
            rep.g_fwd.replay()
        return rep.static_out.detach()

    @staticmethod
    def backward(ctx, gout):
        rep = ctx.rep
        with torch.cuda.device(rep.device):
            rep.static_gout.copy_(gout)
            rep.g_bwd.replay()
        rep.fresh = True               # static_grads now hold this step's gradients of the replica
        return None, None, None


class _ArmReduce(torch.autograd.Function):
    """Identity whose backward arms the end-of-backward gradient hand-over (single-device engine: there is no gather node)."""

    @staticmethod
    def forward(ctx, engine, x):
        ctx.engine = engine
        return x.view_as(x)

    @staticmethod
    def backward(ctx, grad):
        ctx.engine._arm_reduce()
        return None, grad


class DataParallelEngine:
    supports_flat_optimizer = True

    def __init__(self, module: nn.Module, device_ids: List[int], wire_dtype: Optional[str] = None, arena_bytes: int = 768 << 20):
        from .. import _ext
        self.C = _ext.lib()
        self.devices = list(device_ids)
        self.world = len(self.devices)
        self.root_device = torch.device("cuda", self.devices[0])
        self.comm = LocalCommunicator(self.devices, arena_bytes)
        self.fused = True
        self.modules = [module]
        for d in self.devices[1:]:
            with torch.cuda.device(d):
                self.modules.append(copy.deepcopy(module).to(torch.device("cuda", d)))
        self.params = [p for p in module.parameters() if p.requires_grad]
        pdt = {p.dtype for p in self.params}
        self.param_dtype = pdt.pop() if len(pdt) == 1 else torch.float32
        wire_p = {torch.float32: "fp32", torch.bfloat16: "bf16", torch.float16: "fp16"}[self.param_dtype]
        self.wire = wire_dtype or ("bf16" if self.param_dtype != torch.float16 else "fp16")
        # value sets: [parameters + float buffers] for the broadcast, gradients for the reduce
        self.bcast = _TensorSet(self.comm, [self._values(m) for m in self.modules], wire_p)
        self.rparams = [[p for p in m.parameters() if p.requires_grad] for m in self.modules]
        self.grads = _TensorSet(self.comm, [[p for p in ps] for ps in self.rparams], self.wire)
        self.param_elem_off = self.grads.elem_off
        self.total_elems = self.grads.total_elems
        self._arena_flat = self.grads.flat(0)
        self.writeback = True
        self._flat: Optional[_FlatState] = None
        self._armed = False
        self._grads_ready_event = None
        self.graphs = None              # per replica _ReplicaGraph (DataParallel(graph_replicas=True))
        self._grad_packs = None         # pointer packs of the replicas' static gradient buffers
        self._value_cache = {}          # module index -> (first data_ptr, tensor list, pointer packs)
        self.pool = ThreadPoolExecutor(max_workers=max(1, self.world - 1), thread_name_prefix="ptd-dp")
        ref = weakref.ref(self)
        for pid, p in enumerate(self.params):
            p._ptd_engine = ref
            p._ptd_index = pid

    # ---- flat optimizer protocol (same contract as GradientEngine)
    def grad_arena(self):
        return self._arena_flat

    def wait_for_gradients(self):
        if self._grads_ready_event is not None:
            torch.cuda.current_stream(self.root_device).wait_event(self._grads_ready_event)

    bind_flat_optimizer = None  # assigned below (shared implementation)
    master_params = None

    @staticmethod
    def _values(m):
        return [p.data for p in m.parameters()] + [b for b in m.buffers() if b.is_floating_point()]

    def _value_packs(self, r):
        """Pointer packs of replica ``r``'s parameters + float buffers.  Walking the module tree and marshalling 267 tensors
        per replica per step is host time a single process does not have; the lists only change when a flat optimizer
        re-points ``p.data`` (detected through the first parameter's address)."""
        m = self.modules[r]
        first = next(m.parameters()).data_ptr()
        ent = self._value_cache.get(r)
        if ent is None or ent[0] != first:
            vals = self._values(m)
            ent = (first, vals, self.bcast.make_packs(vals))
            self._value_cache[r] = ent
        return ent[2]

    # ---- K2': root -> all replicas
    def broadcast_values(self):
        if self.world == 1:
            return
        root_stream = torch.cuda.current_stream(self.root_device)
        # replicas must be done reading their previous values before the arena is overwritten
        for r in range(1, self.world):
            ev = torch.cuda.Event()
            with torch.cuda.device(self.devices[r]):
                ev.record(torch.cuda.current_stream())
            root_stream.wait_event(ev)
        self.bcast.launch(KIND_PUSH, 0, packs=self._value_packs(0))
        ev = torch.cuda.Event()
        ev.record(root_stream)
        for r in range(1, self.world):
            with torch.cuda.device(self.devices[r]):
                torch.cuda.current_stream().wait_event(ev)
                self.bcast.launch(KIND_UNPACK, r, packs=self._value_packs(r))

    # ---- K5: all replicas -> root
    def _arm_reduce(self):
        if not self._armed:
            self._armed = True
            torch.autograd.Variable._execution_engine.queue_callback(self._reduce)

    def _reduce(self):
        self._armed = False
        root_stream = torch.cuda.current_stream(self.root_device)
        graphed = self.graphs is not None and all(g.fresh for g in self.graphs)
        for r in range(self.world):
            ps = self.rparams[r]
            with torch.cuda.device(self.devices[r]):
                if graphed:             # the backward graph left the gradients in static buffers: prebuilt pointer pack
                    self.graphs[r].fresh = False
                    self.grads.launch(KIND_PACK, r, scale=1.0, packs=self._grad_packs[r])
                else:
                    grads = []
                    for p in ps:
                        if p.grad is None:
                            p.grad = torch.zeros_like(p, memory_format=torch.preserve_format)
                        grads.append(p.grad if is_dense(p.grad) else p.grad.contiguous())
                    self.grads.launch(KIND_PACK, r, scale=1.0, tensors=grads)
                if r > 0:
                    ev = torch.cuda.Event()
                    ev.record(torch.cuda.current_stream())
                    root_stream.wait_event(ev)
        with torch.cuda.device(self.root_device):
            if graphed and self.writeback:
                for p, g in zip(self.rparams[0], self.graphs[0].static_grads):     # the reduced values are unpacked into these
                    p.grad = g
            root_grads = self.graphs[0].static_grads if graphed else [p.grad for p in self.rparams[0]]
            if self.world > 1:          # world == 1: the pack above already left this device's gradients in the arena
                if graphed:
                    self.grads.launch(KIND_REDUCE, 0, writeback=self.writeback, packs=self._grad_packs[0])
                else:
                    self.grads.launch(KIND_REDUCE, 0, writeback=self.writeback, tensors=root_grads)
            ev = torch.cuda.Event()
            ev.record(root_stream)
        self._grads_ready_event = ev
        # replicas may not overwrite their arenas (next pack) before the root has pulled them
        for r in range(1, self.world):
            with torch.cuda.device(self.devices[r]):
                torch.cuda.current_stream().wait_event(ev)
                if not graphed:
                    for p in self.rparams[r]:
                        p.grad = None


def _bind_flat_optimizer(self, optimizer, params):
    from .ddp import GradientEngine
    return GradientEngine.bind_flat_optimizer(self, optimizer, params)


def _master_params(self):
    from .ddp import GradientEngine
    return GradientEngine.master_params(self)


DataParallelEngine.bind_flat_optimizer = _bind_flat_optimizer
DataParallelEngine.master_params = _master_params


class DataParallel(nn.Module):
    def __init__(self, module: nn.Module, device_ids=None, output_device=None, dim: int = 0, compute_dtype=None,
                 wire_dtype: Optional[str] = None, graph_replicas: Optional[bool] = None, graph_warmup: int = 2):
        super().__init__()
        if graph_replicas is None:
            graph_replicas = os.environ.get("PTD_DP_GRAPH", "1") == "1"
        self.graph_replicas = bool(graph_replicas)
        self.graph_warmup = graph_warmup
        self._train_calls = 0
        self._graphed = None            # per replica: (graphed callable, eager forward, input shape, input dtype)
        self.graph_launches_per_step = 0
        if dim != 0:
            raise NotImplementedError("only dim=0 scatter/gather is supported")
        self.module = module
        self.dim = dim
        if not torch.cuda.is_available():
            self.device_ids = []
            self.engine = None
            return
        if device_ids is None:
            device_ids = list(range(torch.cuda.device_count()))
        self.device_ids = [d.index if isinstance(d, torch.device) else int(d) for d in device_ids]
        self.output_device = self.device_ids[0] if output_device is None else (
            output_device.index if isinstance(output_device, torch.device) else int(output_device))
        if self.output_device != self.device_ids[0]:
            raise NotImplementedError("output_device must be device_ids[0]")
        root = torch.device("cuda", self.device_ids[0])
        if next(module.parameters()).device != root:
            raise RuntimeError("module must have its parameters and buffers on device %s (device_ids[0])" % root)
        self.engine = DataParallelEngine(module, self.device_ids, wire_dtype=wire_dtype)

    def _replica_forward(self, r, x, grad_enabled, autocast_state):
        dev = self.engine.devices[r]
        m = self.engine.modules[r]
        graphs = self.engine.graphs
        if graphs is not None and grad_enabled and m.training and x.shape == graphs[r].shape and x.dtype == graphs[r].dtype:
            # the captured graphs replay one shape in training mode; everything else (eval, ragged last batch) runs eagerly
            return _Replay.apply(graphs[r], x, graphs[r].token)
        with torch.cuda.device(dev), torch.set_grad_enabled(grad_enabled):
            if autocast_state[0]:
                with torch.autocast("cuda", dtype=autocast_state[1]):
                    return m(x)
            return m(x)

    def _graph_replicas(self, inputs, autocast_state):
        """Capture forward + backward of every replica on its device (see :class:`_ReplicaGraph`)."""
        eng = self.engine
        from .. import _ext
        for d in eng.devices:
            torch.cuda.synchronize(d)
        n0 = _ext.launches
        eng.graphs = [_ReplicaGraph(m, eng.rparams[r], inputs[r], eng.devices[r], autocast_state) for r, m in enumerate(eng.modules)]
        eng._grad_packs = [eng.grads.make_packs(g.static_grads) for g in eng.graphs]
        for d in eng.devices:
            torch.cuda.synchronize(d)
        # 3 warm-ups + 1 capture ran every native kernel of forward + backward once per replica
        self.graph_launches_per_step = (_ext.launches - n0) // 4
        _ext.launches = n0
        self._graphed = eng.graphs

    def forward(self, x):
        eng = self.engine
        if eng is None or eng.world == 0:
            return self.module(x)
        if eng.world == 1:
            # one device: no scatter / broadcast / gather, but a flat optimizer still reads the gradient ARENA, so backward
            # must end with the pack that fills it (without it the optimizer would step on stale memory)
            out = self.module(x)
            if torch.is_grad_enabled() and out.requires_grad:
                out = _ArmReduce.apply(eng, out)
            return out
        for m in eng.modules[1:]:
            if m.training != self.module.training:       # (walking ~160 submodules of 7 replicas every step is host time)
                m.train(self.module.training)
        eng.broadcast_values()
        # scatter (copy engines): chunk on dim 0 like torch.nn.parallel.scatter
        chunks = x.chunk(eng.world, dim=0)
        n = len(chunks)
        root_stream = torch.cuda.current_stream(eng.root_device)
        ev_in = torch.cuda.Event()
        ev_in.record(root_stream)
        inputs = [chunks[0]]
        for r in range(1, n):
            with torch.cuda.device(eng.devices[r]):
                torch.cuda.current_stream().wait_event(ev_in)
                inputs.append(chunks[r].to(torch.device("cuda", eng.devices[r]), non_blocking=True))
        ge = torch.is_grad_enabled()
        ac = (torch.is_autocast_enabled("cuda"), torch.get_autocast_dtype("cuda"))
        if ge and self.module.training and n == eng.world:
            self._train_calls += 1
            if self.graph_replicas and self._graphed is None and self._train_calls > self.graph_warmup:
                self._graph_replicas(inputs, ac)
        if self._graphed is not None and ge and self.module.training:
            from .. import _ext
            _ext.note_launch(self.graph_launches_per_step)
        # replica threads in both modes: launching a ~450-node CUDA graph costs the host ~2 ms and cudaGraphLaunch releases the
        # GIL, so the per-device launches proceed in parallel (backward: autograd's per-device threads do the same)
        futs = [eng.pool.submit(self._replica_forward, r, inputs[r], ge, ac) for r in range(1, n)]
        outs = [self._replica_forward(0, inputs[0], ge, ac)]
        outs += [f.result() for f in futs]
        return _Gather.apply(eng, *outs)
