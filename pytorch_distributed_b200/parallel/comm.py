"""Communicators: the data plane behind every parallel engine.

``FusedCommunicator``  - the product: symmetric arena over NVLink/NVSwitch + the hand-written kernels in
                         ``csrc/collectives.cu`` (NVLS multimem when the fabric offers it, plain P2P otherwise).
                         ``torch.distributed`` is used for rendezvous only (exchange of memory handles).
``TorchCommunicator``  - library all-reduce/broadcast through ``torch.distributed`` (NCCL on GPUs = the A/B baseline,
                         gloo on CPU = the test backend).  Same interface, so engines do not care.

Replaces, for the reference: ``dist.init_process_group('nccl')`` + the implicit NCCL communicator
(/root/reference/distributed.py:132), ``dist.all_reduce`` / ``dist.barrier`` (:105-109,256) and the broadcasts
hidden in the DDP constructor (:147).
"""
from __future__ import annotations

import os
import threading
import uuid
from typing import List, Optional, Sequence

import numpy as np
import torch
import torch.distributed as dist

from . import plan as P

KIND_TWO_SHOT, KIND_ONE_SHOT, KIND_BCAST, KIND_PACK, KIND_REDUCE, KIND_PUSH, KIND_UNPACK = range(7)
FLAG_PREPACKED = 1        # csrc/collectives.cu kPrepacked: gradients already live in the arena (bucket views)
# payloads up to this size take the one-shot kernel (one barrier, W x the traffic); tools/comm_bench.py measures the crossover
ONE_SHOT_MAX_BYTES = int(os.environ.get("PTD_ONESHOT_MAX_BYTES", str(512 << 10)))
_DT = {torch.float32: "fp32", torch.bfloat16: "bf16", torch.float16: "fp16"}
_TORCH_DT = {"fp32": torch.float32, "bf16": torch.bfloat16, "fp16": torch.float16}
_VIEW_NAME = {"fp32": "float32", "bf16": "bfloat16", "fp16": "float16"}


class Plan:
    """Device-resident segment tables + the arena range of one fused collective."""

    def __init__(self, comm: "FusedCommunicator", numels: Sequence[int], wire: str, max_ctas: int, double_buffer: bool,
                 offsets=None, total=None, data_off_bytes: Optional[int] = None, rank_slot: int = 0, bytes_per_cta: int = 256 << 10):
        self.comm = comm
        self.wire = wire
        esz = P.WIRE_BYTES[wire]
        if total is None:
            offs, total = P.tensor_layout(numels)
        else:
            offs = list(offsets)
        if total * esz >= (64 << 20) and "PTD_MAX_CTAS" not in os.environ:
            max_ctas = max(max_ctas, 64)        # >= 64 MB messages: 64 CTAs keep enough multimem requests in flight
        grid = P.choose_grid(total, esz, min(max_ctas, comm.max_blocks), bytes_per_cta)
        self.layout = P.build_layout(numels, comm.world, grid, offs, total)
        self.grid = grid
        self.block_elems = self.layout.block_elems
        self.region_bytes = self.layout.region_elems * esz
        self.double_buffer = double_buffer
        dev = comm.device_of(rank_slot)
        self.seg_begin = torch.from_numpy(self.layout.seg_begin.copy()).to(dev)
        segs = self.layout.segs
        raw = np.frombuffer(segs.tobytes(), dtype=np.uint8).copy() if len(segs) else np.zeros(24, dtype=np.uint8)
        self.segs = torch.from_numpy(raw).to(dev)
        self.calls = torch.zeros(max(grid, 1), dtype=torch.int32, device=dev)
        if data_off_bytes is None:
            # double_buffer: [staging 0 | staging 1 | result] - the third region receives the one-shot kernel's reduced values
            data_off_bytes = comm.alloc(self.region_bytes * (3 if double_buffer else 1))
        self.data_off_bytes = data_off_bytes
        self.rank_slot = rank_slot

    def arena_tensor(self, rank_slot: Optional[int] = None) -> torch.Tensor:
        """The plan's (first) region of the local arena as a flat tensor of the wire dtype."""
        r = self.rank_slot if rank_slot is None else rank_slot
        return self.comm.arena.view(self.data_off_bytes, self.layout.region_elems, _VIEW_NAME[self.wire], r)


class FusedCommunicator:
    backend = "fused"

    def __init__(self, group=None, device: Optional[torch.device] = None, arena_bytes: Optional[int] = None, timeout_ms: int = 120000,
                 allow_nvls: Optional[bool] = None, max_ctas: int = 32):
        from .. import _ext
        self._C = _ext.lib()
        self._ext = _ext
        self.group = group
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        if self.world > self._C.MAX_WORLD:
            raise RuntimeError("world size %d exceeds the fused communicator limit %d" % (self.world, self._C.MAX_WORLD))
        self.device = torch.device(device if device is not None else "cuda:%d" % torch.cuda.current_device())
        if arena_bytes is None:       # 1 GiB covers ResNet-152-sized models (gradient arena + double-buffered fp32 weight broadcast)
            arena_bytes = int(os.environ.get("PTD_ARENA_MB", "1024")) << 20
        timeout_ms = int(os.environ.get("PTD_COMM_TIMEOUT_MS", timeout_ms))
        self.max_blocks = self._C.MAX_BLOCKS
        self.max_ctas = min(int(os.environ.get("PTD_MAX_CTAS", max_ctas)), self.max_blocks)   # CTAs per collective (<= 64): sweepable
        self.header_bytes = P.round_up(self._C.SIGNAL_PAD_BYTES, 128 << 10)
        self._bump = self.header_bytes
        self._next_channel = 0
        self._plans = {}
        self._side_stream = None
        self._lock = threading.RLock()      # plans / arena offsets may be requested from the hvd dispatcher thread too
        if allow_nvls is None:
            allow_nvls = os.environ.get("PTD_NVLS", "1") != "0"
        self.symm_backend = "native"
        torch.cuda.set_device(self.device)
        self.arena = self._rendezvous(arena_bytes, allow_nvls)
        self.arena.set_timeout_ms(timeout_ms)
        self.nvls = bool(self.arena.has_multicast)
        # found_inf word lives inside the (symmetric) header, right after the SignalPad struct
        self.found_inf_off = P.round_up(self._C.SIGNAL_PAD_BYTES, 64)
        assert self.found_inf_off + 64 <= self.header_bytes
        self.found_inf = self.arena.view(self.found_inf_off, 1, "int32", 0)
        self._ll_in = torch.zeros(8, dtype=torch.float32, device=self.device)
        self.ll_channel = self.new_channel()
        self.misc_channel = self.new_channel()
        self.bcast_channel = self.new_channel()

    # ------------------------------------------------------------------ setup
    def device_of(self, rank_slot: int = 0) -> torch.device:
        return self.device

    @property
    def side_stream(self) -> "torch.cuda.Stream":
        """THE communication stream of this communicator (high priority): gradient buckets, the deferred BN-buffer
        broadcast and the metric all-reduce are all enqueued here, in the same order on every rank, so none of their
        cross-GPU waits sits on the compute stream."""
        if self._side_stream is None:
            self._side_stream = torch.cuda.Stream(device=self.device, priority=-1)
        return self._side_stream

    def _gather_obj(self, obj):
        out = [None] * self.world
        dist.all_gather_object(out, obj, group=self.group)
        return out

    def _rendezvous(self, arena_bytes: int, allow_nvls: bool):
        C = self._C
        dev = self.device.index if self.device.index is not None else torch.cuda.current_device()
        mode = os.environ.get("PTD_SYMM", "native")
        if self.world == 1:
            return C.SymmArena(dev, 0, 1, arena_bytes)
        err = None
        arena = None
        if mode != "torch":
            try:
                arena = C.SymmArena(dev, self.rank, self.world, arena_bytes)
            except Exception as e:  # noqa: BLE001
                err = repr(e)
        errs = self._gather_obj(err)
        if any(e is not None for e in errs) or mode == "torch":
            if mode != "torch" and self.rank == 0:
                print("[ptd] native VMM arena failed (%s); falling back to torch symmetric memory" % [e for e in errs if e][:1])
            return self._rendezvous_torch(arena_bytes, allow_nvls)
        token = self._gather_obj(uuid.uuid4().hex if self.rank == 0 else None)[0]
        name = lambda r: "ptd-%s-%d" % (token, r)  # noqa: E731
        arena.open_socket(name(self.rank))
        dist.barrier(group=self.group)
        fd = arena.export_fd()
        for p in range(self.world):
            if p != self.rank:
                arena.send_fd(name(p), fd, 0)
        for _ in range(self.world - 1):
            tag, src, pfd = arena.recv_fd()
            assert tag == 0, "unexpected descriptor tag %d" % tag
            arena.map_peer(src, pfd)
        os.close(fd)
        dist.barrier(group=self.group)
        # ---- NVLS multicast (optional)
        want = bool(arena.multicast_candidate) and allow_nvls
        if all(self._gather_obj(want)):
            mfd, e = -1, None
            if self.rank == 0:
                try:
                    mfd = arena.mc_create()
                except Exception as ex:  # noqa: BLE001
                    e = repr(ex)
            ok = self._gather_obj(e)[0] is None
            if ok:
                if self.rank == 0:
                    for p in range(1, self.world):
                        arena.send_fd(name(p), mfd, 1)
                    os.close(mfd)
                else:
                    tag, src, pfd = arena.recv_fd()
                    assert tag == 1
                    arena.mc_import(pfd)
                e = None
                try:
                    arena.mc_add_device()
                except Exception as ex:  # noqa: BLE001
                    e = repr(ex)
                ok = all(x is None for x in self._gather_obj(e))
            if ok:
                try:
                    arena.mc_bind_and_map()
                except Exception as ex:  # noqa: BLE001
                    e = repr(ex)
                ok = all(x is None for x in self._gather_obj(e))
            if not ok:
                arena.disable_multicast("multicast setup failed: %s" % (e,))
        else:
            arena.disable_multicast("multicast not supported or disabled")
        dist.barrier(group=self.group)
        return arena

    def _rendezvous_torch(self, arena_bytes: int, allow_nvls: bool):
        import torch.distributed._symmetric_memory as symm_mem
        self.symm_backend = "torch"
        grp = self.group if self.group is not None else dist.group.WORLD
        buf = symm_mem.empty(arena_bytes, dtype=torch.uint8, device=self.device)
        hdl = symm_mem.rendezvous(buf, grp.group_name)
        buf.zero_()
        torch.cuda.synchronize()
        dist.barrier(group=self.group)
        self._torch_symm = (buf, hdl)
        mc = int(getattr(hdl, "multicast_ptr", 0) or 0) if allow_nvls else 0
        return self._C.SymmArena.from_pointers(self.rank, self.world, [int(p) for p in hdl.buffer_ptrs], mc, arena_bytes,
                                               self.device.index or 0)

    # ------------------------------------------------------------------ resources
    def alloc(self, nbytes: int, align: int = 4096) -> int:
        with self._lock:
            off = P.round_up(self._bump, align)
            if off + nbytes > self.arena.bytes:
                raise RuntimeError("symmetric arena exhausted: need %d more bytes (capacity %d); raise PTD_ARENA_MB / arena_bytes" %
                                   (off + nbytes - self.arena.bytes, self.arena.bytes))
            self._bump = off + nbytes
            return off

    def new_channel(self) -> int:
        ch = self._next_channel
        if ch >= self._C.MAX_CHANNELS:
            raise RuntimeError("out of signal channels")
        self._next_channel += 1
        return ch

    def make_plan(self, numels: Sequence[int], wire: str = "bf16", max_ctas: Optional[int] = None, double_buffer: bool = False,
                  **kw) -> Plan:
        if "bytes_per_cta" not in kw:
            nbytes = sum(int(n) for n in numels) * P.WIRE_BYTES[wire]
            if double_buffer and nbytes <= (4 << 20):
                # latency-bound payloads (one-shot all-reduce, small broadcasts such as the BN buffers' 106 tiny tensors):
                # many small CTA ranges => short per-CTA segment loops and more requests in flight
                kw["bytes_per_cta"] = 16 << 10
        return Plan(self, numels, wire, max_ctas or self.max_ctas, double_buffer, **kw)

    def check(self) -> None:
        st = self.arena.status()
        if st:
            raise RuntimeError("fused collective timed out waiting for a peer (status 0x%08x, rank %d of %d): a peer process died "
                               "or hung" % (st, self.rank, self.world))

    # ------------------------------------------------------------------ launches
    def run(self, plan: Plan, tensors: List[torch.Tensor], kind: int, channel: int, scale: float = 1.0, writeback: bool = True,
            root: int = 0, check_inf: bool = False, nvls: Optional[bool] = None, rank_slot: int = 0, prepacked: bool = False,
            result_off_bytes: int = -1) -> None:
        use_nvls = self.nvls if nvls is None else (nvls and self.nvls)
        if len(tensors) > self._C.MAX_PTRS:
            raise RuntimeError("too many tensors for one plan launch")
        self._ext.note_launch()
        self.arena.launch_plan(channel, rank_slot, kind, P.WIRE_CODES[plan.wire], use_nvls, plan.grid, tensors,
                               plan.seg_begin.data_ptr(), plan.segs.data_ptr(), plan.data_off_bytes, plan.block_elems,
                               plan.calls.data_ptr(), self.found_inf.data_ptr() if check_inf else 0, float(scale), bool(writeback),
                               int(root), FLAG_PREPACKED if prepacked else 0, int(result_off_bytes))

    def _cached_plan(self, key, tensors, wire, double_buffer, max_ctas=None):
        with self._lock:
            pl = self._plans.get(key)
            if pl is None:
                pl = self.make_plan([t.numel() for t in tensors], wire, max_ctas=max_ctas, double_buffer=double_buffer)
                self._plans[key] = pl
            return pl

    @staticmethod
    def _sig(tensors):
        return tuple((t.numel(), t.dtype) for t in tensors)

    def all_reduce_(self, tensors: Sequence[torch.Tensor], average: bool = True, wire: Optional[str] = None) -> None:
        """In-place fused all-reduce of a tensor list (sum or mean) on the current stream."""
        tensors = list(tensors)
        if not tensors:
            return
        if wire is None:
            wire = "fp32" if all(t.dtype == torch.float32 for t in tensors) else _DT[tensors[0].dtype]
        nbytes = sum(t.numel() for t in tensors) * P.WIRE_BYTES[wire]
        one_shot = nbytes <= ONE_SHOT_MAX_BYTES
        key = ("ar", one_shot, wire, self._sig(tensors))
        pl = self._cached_plan(key, tensors, wire, double_buffer=one_shot)
        scale = 1.0 / self.world if average else 1.0
        self.run(pl, tensors, KIND_ONE_SHOT if one_shot else KIND_TWO_SHOT, self.misc_channel, scale=scale, writeback=True)

    def broadcast_(self, tensors: Sequence[torch.Tensor], root: int = 0, wire: Optional[str] = None) -> None:
        tensors = list(tensors)
        if not tensors or self.world == 1:
            return
        if wire is None:
            wire = "fp32" if any(t.dtype == torch.float32 for t in tensors) else _DT[tensors[0].dtype]
        for i in range(0, len(tensors), self._C.MAX_PTRS):
            chunk = tensors[i:i + self._C.MAX_PTRS]
            key = ("bc", wire, self._sig(chunk))
            pl = self._cached_plan(key, chunk, wire, double_buffer=True)
            self.run(pl, chunk, KIND_BCAST, self.bcast_channel, root=root)

    def barrier(self) -> None:
        self._ext.note_launch()
        self.arena.launch_barrier(self.misc_channel)

    def metrics(self, logits: torch.Tensor, target: torch.Tensor, loss: Optional[torch.Tensor], out: torch.Tensor) -> torch.Tensor:
        """out[0:3] = mean over ranks of (loss, acc1 %, acc5 %) - one kernel, includes the top-k counting."""
        self._ext.note_launch()
        self.arena.launch_metrics(self.ll_channel, logits, target, loss, out)
        return out

    def reduce_scalars_(self, t: torch.Tensor, average: bool = True) -> torch.Tensor:
        """Low-latency all-reduce of <= 8 floats (LL protocol: flag travels with the payload)."""
        if self.world == 1:
            return t
        flat = t.reshape(-1)
        n = flat.numel()
        assert n <= 8 and flat.dtype == torch.float32
        self._ll_in[:n].copy_(flat)
        self._ext.note_launch()
        self.arena.launch_ll_allreduce(self.ll_channel, self._ll_in[:n], flat, 1.0 / self.world if average else 1.0)
        return t


class TorchCommunicator:
    """Library collectives through torch.distributed (NCCL baseline / gloo for CPU tests)."""

    def __init__(self, group=None, device: Optional[torch.device] = None):
        self.group = group
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.device = torch.device(device) if device is not None else torch.device("cpu")
        self.backend = dist.get_backend(group) if dist.is_initialized() else "none"
        self.nvls = False

    def check(self) -> None:
        pass

    def all_reduce_(self, tensors, average: bool = True, wire: Optional[str] = None, async_op: bool = False):
        tensors = list(tensors)
        if not tensors or self.world == 1:
            return None
        wdt = _TORCH_DT[wire] if wire else tensors[0].dtype
        if self.device.type == "cpu" and wdt != torch.float32:
            wdt = torch.float32  # gloo: keep the test backend exact
        flat = torch.cat([t.reshape(-1).to(wdt) for t in tensors])
        if average:
            flat.div_(self.world)
        work = dist.all_reduce(flat, group=self.group, async_op=True)

        def finish():
            work.wait()
            off = 0
            for t in tensors:
                n = t.numel()
                t.copy_(flat[off:off + n].view_as(t))
                off += n
        if async_op:
            return finish
        finish()
        return None

    def broadcast_(self, tensors, root: int = 0, wire: Optional[str] = None) -> None:
        tensors = list(tensors)
        if not tensors or self.world == 1:
            return
        by_dtype = {}
        for t in tensors:
            by_dtype.setdefault(t.dtype, []).append(t)
        for dt, ts in by_dtype.items():
            flat = torch.cat([t.reshape(-1) for t in ts])
            dist.broadcast(flat, src=dist.get_global_rank(self.group, root) if self.group is not None else root, group=self.group)
            off = 0
            for t in ts:
                n = t.numel()
                t.copy_(flat[off:off + n].view_as(t))
                off += n

    def barrier(self) -> None:
        if self.world > 1:
            dist.barrier(group=self.group)

    def metrics(self, logits, target, loss, out):
        from ..utils.meters import accuracy
        acc1, acc5 = accuracy(logits, target, topk=(1, 5))
        out[0] = loss.detach().float() if loss is not None else 0.0
        out[1] = acc1[0]
        out[2] = acc5[0]
        out[3] = 0
        if self.world > 1:
            dist.all_reduce(out[:3], group=self.group)
            out[:3] /= self.world
        return out

    def reduce_scalars_(self, t, average: bool = True):
        if self.world > 1:
            dist.all_reduce(t, group=self.group)
            if average:
                t /= self.world
        return t


def make_communicator(kind: str = "auto", group=None, device=None, **kw):
    """kind: auto | fused | nccl | gloo.  ``auto`` = fused on CUDA, library collectives on CPU."""
    device = torch.device(device) if device is not None else torch.device("cuda" if torch.cuda.is_available() else "cpu")
    if kind == "auto":
        kind = "fused" if device.type == "cuda" else "gloo"
    if kind == "fused":
        if device.type != "cuda":
            raise RuntimeError("--comm fused needs CUDA devices")
        return FusedCommunicator(group=group, device=device, **kw)
    return TorchCommunicator(group=group, device=device)
