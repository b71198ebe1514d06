"""FusedSGD: SGD with momentum / weight decay as hand-written sm_90a kernels (``csrc/optim.cu``).

Drop-in for ``torch.optim.SGD`` as used at /root/reference/distributed.py:153-156 and, together with
:mod:`..parallel.amp`, for apex's patched optimizer + ``amp_C`` kernels (/root/reference/apex_distributed.py:211-216,330).

Three execution modes, picked automatically:
  * **flat / arena** - the parameters belong to one of our data-parallel engines: the reduced gradients are read
    directly from the symmetric wire arena (no write-back into ``p.grad``), master weights / momentum / model copy are
    flat buffers with the arena's layout, and the whole step is ONE streaming kernel.
  * **multi-tensor** - CUDA parameters without an engine: chunked multi-tensor-apply kernel over ``p.grad``.
  * **reference** - CPU tensors: plain PyTorch math (also the numerical oracle for the tests).

``enable_larc`` (what ``apex.parallel.LARC`` calls) adds layer-wise adaptive rates to all three modes: a norm pass and an
update pass per flat step, per bucket in overlap mode, or per group in multi-tensor mode (``csrc/optim.cu``).

``attach_ema`` (what :class:`~pytorch_distributed_b200.utils.ema.ModelEma` calls) folds an exponential moving average of
the fp32 masters into the update kernels of every mode (one more fp32 read and write per element), and averages the
model's float buffers with one ``ema_multi`` launch at the end of each step.  The decay sits in hyper slots 6 and 7.

``clip_grad_norm`` / ``set_clip_grad_norm`` (``--clip-grad-norm``) clip the unscaled, reduced gradient to a global L2 norm, as
``torch.nn.utils.clip_grad_norm_`` right before the step: a norm pass over every gradient of the step, then one CTA that
writes a clipped copy of each group's hyper tensor (slot 4, the gradient multiplier, times the clip coefficient), which the
unchanged update kernels take in place of ``hyper``.  ``max_norm`` sits in hyper slot 8.  While clipping is on, the
per-bucket update of overlap mode stays off: no bucket may be updated before the last gradient is known.
"""
from __future__ import annotations

import math
from types import SimpleNamespace
from typing import Optional

import torch
from torch.optim import Optimizer


_FP32_STATE = ("momentum_buffer", "master")     # per-parameter state that stays fp32 whatever the parameter's dtype


def sgd_reference_step(p, g, buf, lr, momentum, weight_decay, dampening, nesterov, first):
    """torch.optim.SGD semantics on plain tensors (fp32 math)."""
    g = g.float()
    if weight_decay != 0:
        g = g.add(p.float(), alpha=weight_decay)
    if momentum != 0:
        if first:
            buf.copy_(g)
        else:
            buf.mul_(momentum).add_(g, alpha=1 - dampening)
        g = g.add(buf, alpha=momentum) if nesterov else buf
    p.add_(g.to(p.dtype), alpha=-lr)


def larc_reference_grad(p, g, lr, weight_decay, trust_coefficient, clip, eps):
    """apex.parallel.LARC on one tensor in fp32: the gradient the wrapped SGD step (run with weight_decay = 0) sees, and
    ``(pn, gn, f)``.  Where a norm is zero the gradient is left as is, without weight decay, and f is reported as 1."""
    p, g = p.float(), g.float()
    pn, gn = torch.linalg.vector_norm(p), torch.linalg.vector_norm(g)
    if pn == 0 or gn == 0:
        return g, (float(pn), float(gn), 1.0)
    f = trust_coefficient * pn / (gn + pn * weight_decay + eps)
    if clip:
        f = torch.clamp(f / lr, max=1.0)
    return (g + weight_decay * p) * f, (float(pn), float(gn), float(f))


class FusedSGD(Optimizer):
    def __init__(self, params, lr=0.1, momentum=0.0, dampening=0.0, weight_decay=0.0, nesterov=False, flat: Optional[bool] = None,
                 overlap_backward: bool = False, clip_grad_norm: Optional[float] = None):
        if nesterov and (momentum <= 0 or dampening != 0):
            raise ValueError("Nesterov momentum requires a momentum and zero dampening")
        defaults = dict(lr=lr, momentum=momentum, dampening=dampening, weight_decay=weight_decay, nesterov=nesterov)
        super().__init__(params, defaults)
        self._steps = 0
        self._flat = None           # _FlatState when bound to an engine
        self._hyper = {}            # group index -> (device tensor, cached python tuple)
        self._amp = None            # LossScaler (set by amp.initialize)
        self._want_flat = flat
        # overlap_backward: in flat mode the update of each gradient bucket is enqueued on the communication stream right
        # behind that bucket's all-reduce (inside loss.backward()), so after the last gradient only the small tail bucket
        # remains; step() then only joins.  Contract: exactly one backward per step() and no gradient surgery between them
        # (the reference loop, /root/reference/distributed.py:267-269).  Inactive under a loss scaler (an overflow found in
        # a later bucket must be able to cancel the whole step).
        self._overlap = bool(overlap_backward)
        self._ov_active = False
        self._ov_applied = 0
        self._ov_first = False
        self._bind_refused = False  # an engine was found but declined (mixed dtypes, other parameter list): do not retry
        self._larc = None           # (trust_coefficient, clip, eps) in LARC mode (enable_larc)
        self._larc_stats = None     # [n_params, 3] fp32 {pn, gn, f} of the last applied step
        self._larc_tab = None       # flat mode: chunk table of the arena layout (built once)
        self._ema = None            # ModelEma updated inside the step (attach_ema)
        self._ema_flat = None       # flat mode: its parameter averages in the arena layout
        self._clip = None           # max_norm of global-norm gradient clipping (set_clip_grad_norm)
        self._clip_state = None     # norm, clipped-step count, clipped hyper copies, partials (made by the first clipped step)
        self.set_clip_grad_norm(clip_grad_norm)
        self._try_bind()

    # ------------------------------------------------------------------ engine binding (flat mode)
    def _try_bind(self):
        if self._want_flat is False or len(self.param_groups) != 1:
            return
        params = [p for p in self.param_groups[0]["params"] if p.requires_grad]
        if not params or not all(p.is_cuda for p in params):
            return
        engines = {getattr(p, "_ptd_engine", None) for p in params}
        if len(engines) != 1:
            return
        ref = engines.pop()
        eng = ref() if ref is not None else None
        if eng is None or not getattr(eng, "supports_flat_optimizer", False):
            return
        self._flat = eng.bind_flat_optimizer(self, params)
        if self._flat is None:
            self._bind_refused = True
            return
        if self._ema is not None:
            self._ema_to_flat()
        if self._overlap and getattr(eng, "supports_overlap_optimizer", False):
            eng.set_overlap_optimizer(self)

    # ------------------------------------------------------------------ overlap mode (called by the gradient engine)
    def _prepare_overlap(self) -> None:
        """First bucket of a backward pass, on the compute stream: decide whether this step is applied bucket by bucket
        and push the hyper-parameters to the device before the side stream forks off."""
        if self._ov_active and self._ov_applied:
            raise RuntimeError("FusedSGD(overlap_backward=True): a second backward pass started before step() - the update of the "
                               "previous pass has already been applied bucket by bucket; accumulate gradients with the "
                               "engine's fp32_grad_accumulation=True and no_sync() (--accum-steps), which keeps the per-bucket "
                               "update, or use overlap_backward=False (--no-overlap-optimizer)")
        self._ov_applied = 0
        self._ov_active = self._flat is not None and self._amp is None and self._clip is None
        if self._ov_active:
            self._ov_first = self._steps == 0
            self._hyper_tensor(0, self.param_groups[0], self._flat.master.device)

    @torch.no_grad()
    def _apply_slice(self, off: int, n: int) -> None:
        """SGD update of flat elements [off, off + n) - the bucket whose all-reduce was just enqueued on this stream."""
        if not self._ov_active:
            return
        fs = self._flat
        from .. import _ext
        if self._larc is not None:
            self._larc_flat(self._hyper[0][0], None, self._ov_first, self._larc_table().ranges[(off, n)])
            self._ov_applied += n
            return
        _ext.note_launch()
        copy = fs.model_copy[off:off + n] if fs.model_copy is not None else None
        ema = self._ema_flat[off:off + n] if self._ema_flat is not None else None
        _ext.lib().fused_sgd_flat(fs.engine.grad_arena()[off:off + n], fs.master[off:off + n], fs.momentum[off:off + n], copy,
                                  self._hyper[0][0], None, bool(self.param_groups[0]["nesterov"]), self._ov_first, ema=ema)
        self._ov_applied += n

    # ------------------------------------------------------------------ LARC (apex.parallel.LARC semantics)
    def enable_larc(self, trust_coefficient: float = 0.02, clip: bool = True, eps: float = 1e-8) -> None:
        """Layer-wise adaptive rates on top of every step (what wrapping this optimizer in ``apex.parallel.LARC`` does)."""
        if not (trust_coefficient > 0 and eps >= 0):
            raise ValueError("LARC needs trust_coefficient > 0 and eps >= 0")
        self._larc = (float(trust_coefficient), bool(clip), float(eps))

    def larc_stats(self) -> Optional[torch.Tensor]:
        """``[n_params, 3]`` fp32 ``(||p||, ||g||, f)`` per parameter in ``param_groups`` order, as of the last applied LARC step
        (f = 1 where a norm is zero; rows of parameters without a gradient stay as they were).  None before the first one."""
        return self._larc_stats

    def _larc_rows(self):
        return {id(p): i for i, p in enumerate(p for g in self.param_groups for p in g["params"])}

    def _larc_stats_on(self, device):
        n = sum(len(g["params"]) for g in self.param_groups)
        old = self._larc_stats
        if old is None or old.size(0) != n:
            # first LARC step, or add_param_group since: rows keep param_groups order, the existing ones keep their values
            self._larc_stats = torch.zeros(n, 3, dtype=torch.float32, device=device)
            if old is not None:
                k = min(n, old.size(0))
                self._larc_stats[:k].copy_(old[:k])
        return self._larc_stats

    def _larc_table(self):
        """Chunk table of the flat layout: tensors in arena order with their first chunk, and the chunk range of every
        gradient bucket.  The layout never changes after binding, so this is built once and kept on the device."""
        if self._larc_tab is not None:
            return self._larc_tab
        from types import SimpleNamespace
        from .. import _ext
        chunk = _ext.lib().LARC_CHUNK
        eng = self._flat.engine
        rows = self._larc_rows()
        order = sorted(range(len(eng.params)), key=lambda i: eng.param_elem_off[i])
        info, chunk_tensor, spans = [], [], []
        for t, pid in enumerate(order):
            p, off = eng.params[pid], eng.param_elem_off[pid]
            assert not spans or off >= spans[-1][1], "flat LARC: parameters overlap in the arena"
            info.append((off, p.numel(), len(chunk_tensor), rows[id(p)]))
            spans.append((off, off + p.numel(), len(chunk_tensor)))
            chunk_tensor += [t] * (-(-p.numel() // chunk))
        assert not spans or spans[-1][1] <= self._flat.master.numel()
        ranges = {}
        for b in getattr(eng, "buckets", []):
            lo, hi = b.elem_off, b.elem_off + b.region_elems
            inside = [s for s in spans if lo <= s[0] < hi]
            # buckets hold whole tensors (plan.compute_buckets): a tensor's norm never spans two per-bucket launches
            assert all(s[1] <= hi for s in inside), "flat LARC: a gradient bucket splits a tensor"
            first = inside[0][2] if inside else 0
            last = inside[-1][2] + -(-(inside[-1][1] - inside[-1][0]) // chunk) if inside else 0
            ranges[(b.elem_off, b.region_elems)] = (first, last)
        dev = self._flat.master.device
        self._larc_tab = SimpleNamespace(
            chunk_tensor=torch.tensor(chunk_tensor, dtype=torch.int32, device=dev),
            info=torch.tensor(info, dtype=torch.int64, device=dev).reshape(-1, 4),
            partials=torch.zeros(max(2 * len(chunk_tensor), 2), dtype=torch.float32, device=dev),
            chunks=len(chunk_tensor), ranges=ranges)
        return self._larc_tab

    def _larc_flat(self, hyper, found_inf, first, chunk_range=None):
        fs = self._flat
        tab = self._larc_table()
        lo, hi = chunk_range if chunk_range is not None else (0, tab.chunks)
        trust, clip, eps = self._larc
        from .. import _ext
        _ext.note_launch(2)
        _ext.lib().larc_sgd_flat(fs.engine.grad_arena(), fs.master, fs.momentum, fs.model_copy, hyper, found_inf,
                                 bool(self.param_groups[0]["nesterov"]), first, tab.chunk_tensor, tab.info, lo, hi, tab.partials,
                                 self._larc_stats_on(fs.master.device), trust, eps, clip, ema=self._ema_flat)

    # ------------------------------------------------------------------ exponential moving average (ModelEma)
    def attach_ema(self, ema) -> None:
        """Update ``ema`` (a :class:`~pytorch_distributed_b200.utils.ema.ModelEma` over this optimizer's model) inside every
        applied step: its parameter averages in the update kernels, its float buffers right after them."""
        self._ema = ema
        if self._flat is not None:
            self._ema_to_flat()
        self.refresh_hyper()

    def _ema_to_flat(self):
        """Move the parameter averages into one fp32 buffer with the arena layout (the flat kernels stream it next to the
        masters); the average's tensors become views of it.  The padding between tensors follows the masters."""
        fs, ema = self._flat, self._ema
        eng = fs.engine
        flat = fs.master.clone()
        with torch.no_grad():
            for pid, p in enumerate(eng.params):
                off, cnt = eng.param_elem_off[pid], p.numel()
                view = flat[off:off + cnt].as_strided(p.size(), p.stride())
                view.copy_(ema.shadow_of(p))
                ema.set_shadow_of(p, view)
        self._ema_flat = flat

    def _ema_multi_lists(self, params):
        return [self._ema.shadow_of(p) for p in params] if self._ema is not None else []

    def _ema_buffers(self, hyper, found_inf, pairs=None):
        """Average the model's float buffers (BatchNorm running statistics) with the decay in ``hyper[6:8]``; skipped
        with the step when ``found_inf`` is set."""
        if self._ema is None:
            return
        live, shadow = pairs if pairs is not None else self._ema.buffer_pairs()
        if not live:
            return
        from .. import _ext
        _ext.note_launch()
        _ext.lib().ema_multi(live, shadow, hyper[6:8], found_inf)

    # ------------------------------------------------------------------ global-norm gradient clipping (clip_grad_norm_)
    def set_clip_grad_norm(self, max_norm: Optional[float]) -> None:
        """Clip the unscaled gradient of every following step to the global L2 norm ``max_norm`` (None: no clipping).  A step
        captured in a CUDA graph follows a new value on replay; turning clipping on or off takes a new capture."""
        if max_norm is not None:
            max_norm = float(max_norm)
            if not (max_norm > 0 and math.isfinite(max_norm)):
                raise ValueError("clip_grad_norm needs a positive finite max_norm, got %r" % (max_norm,))
        self._clip = max_norm
        self.refresh_hyper()

    def grad_norm(self) -> Optional[torch.Tensor]:
        """fp32 scalar tensor: the global norm of the unscaled gradient before clipping, as of the last applied clipped step
        (what ``clip_grad_norm_`` returns); None before the first clipped step."""
        return self._clip_state.total if self._clip_state is not None else None

    def clipped_steps(self) -> Optional[torch.Tensor]:
        """int32 tensor of one element: the number of applied steps whose clip coefficient was below 1; None before the
        first clipped step."""
        return self._clip_state.count if self._clip_state is not None else None

    def _clip_on(self, device):
        if self._clip_state is None:
            self._clip_state = SimpleNamespace(total=torch.zeros((), dtype=torch.float32, device=device),
                                               count=torch.zeros(1, dtype=torch.int32, device=device), hyper={}, partials=None)
        return self._clip_state

    def _clipped_copy(self, gi, hyper):
        cs = self._clip_on(hyper.device)
        t = cs.hyper.get(gi)
        if t is None or t.numel() != hyper.numel():
            t = cs.hyper[gi] = torch.zeros_like(hyper)
        return t

    def _clip_flat(self, hyper, found_inf):
        """Norm pass over the arena's parameter ranges and finalize; returns the clipped copy of ``hyper``."""
        fs, tab = self._flat, self._larc_table()
        cs = self._clip_on(hyper.device)
        clipped = self._clipped_copy(0, hyper)
        from .. import _ext
        _ext.note_launch(2)
        _ext.lib().grad_sumsq_flat(fs.engine.grad_arena(), tab.chunk_tensor, tab.info, tab.partials, hyper, found_inf)
        _ext.lib().clip_finalize(tab.partials, tab.chunks, [hyper], [clipped], found_inf, cs.total, cs.count)
        return clipped

    @staticmethod
    def _kernel_group(params) -> bool:
        return params[0].is_cuda and all(p.dtype in (torch.float32, torch.bfloat16, torch.float16) for p in params)

    def _clip_multi(self, amp):
        """Multi-tensor and PyTorch modes: the clipping of this step, over every group.  Returns ``{group index: clipped
        hyper}`` on the kernel path, the clip coefficient (a 0-d tensor) on the PyTorch path, None when nothing is clipped."""
        groups = [(gi, [p for p in g["params"] if p.grad is not None]) for gi, g in enumerate(self.param_groups)]
        groups = [(gi, ps) for gi, ps in groups if ps]
        if not groups:
            return None
        kinds = {self._kernel_group(ps) for _, ps in groups}
        if len(kinds) != 1:
            raise NotImplementedError("clip_grad_norm: the parameter groups mix the CUDA kernels and the PyTorch path")
        if kinds.pop():
            from .. import _ext
            C = _ext.lib()
            dev = groups[0][1][0].device
            cs = self._clip_on(dev)
            need = sum(-(-p.numel() // C.LARC_CHUNK) for _, ps in groups for p in ps)
            if cs.partials is None or cs.partials.numel() < need:
                cs.partials = torch.zeros(max(need, 1), dtype=torch.float32, device=dev)
            fi = amp.found_inf if amp is not None else None
            hypers, off = [], 0
            for gi, ps in groups:
                hyper = self._hyper_tensor(gi, self.param_groups[gi], dev)
                if amp is not None:
                    amp.attach_hyper(hyper)
                hypers.append(hyper)
                _ext.note_launch()
                off = C.grad_sumsq_multi([p.grad for p in ps], hyper, fi, cs.partials, off)
            clipped = [self._clipped_copy(gi, h) for (gi, _), h in zip(groups, hypers)]
            _ext.note_launch()
            C.clip_finalize(cs.partials, off, hypers, clipped, fi, cs.total, cs.count)
            return {gi: c for (gi, _), c in zip(groups, clipped)}
        if amp is not None and amp.host_found_inf():
            return None
        gmul = amp.host_inv_scale() if amp is not None else 1.0
        grads = [p.grad if gmul == 1.0 else p.grad.float() * gmul for _, ps in groups for p in ps]
        # torch.nn.utils.clip_grad_norm_'s arithmetic (L2, foreach) on the unscaled gradients, which stay unwritten in p.grad
        total = torch.nn.utils.get_total_norm(grads, 2.0)
        coef = torch.clamp(self._clip / (total + 1e-6), max=1.0)
        cs = self._clip_on(total.device)
        cs.total.copy_(total)
        cs.count.add_((coef < 1).to(cs.count.dtype))
        return coef

    @property
    def is_flat(self) -> bool:
        return self._flat is not None

    # ------------------------------------------------------------------ hyper-parameters on the device
    def _hyper_tensor(self, gi: int, group, device):
        gmul = 1.0
        vals = (float(group["lr"]), float(group["momentum"]), float(group["weight_decay"]), float(group["dampening"]))
        dw = self._ema.decay_pair() if self._ema is not None else (0.0, 0.0)      # slots 6, 7: EMA decay d and fp32(1 - d)
        clip = self._clip if self._clip is not None else 0.0                       # slot 8: max_norm of gradient clipping
        ent = self._hyper.get(gi)
        if ent is None:
            # slot 5 (momentum_pending): under dynamic loss scaling the momentum is initialised by the first step that is
            # actually applied; the loss scaler clears the slot after it (csrc/optim.cu)
            pending = 1.0 if self._steps == 0 else 0.0
            t = torch.tensor(list(vals) + [gmul, pending] + list(dw) + [clip], dtype=torch.float32, device=device)
            self._hyper[gi] = [t, vals, dw, clip]
            return t
        if ent[1] != vals:
            # only lr..dampening and the EMA slots are host-owned; slot 4 (gradient multiplier) belongs to the loss scaler kernel
            ent[0][:4].copy_(torch.tensor(vals, dtype=torch.float32), non_blocking=True)
            ent[1] = vals
        if ent[2] != dw:
            ent[0][6:8].copy_(torch.tensor(dw, dtype=torch.float32), non_blocking=True)
            ent[2] = dw
        if ent[3] != clip:
            ent[0][8:9].fill_(clip)
            ent[3] = clip
        return ent[0]

    def refresh_hyper(self) -> None:
        """Push changed lr/momentum/weight-decay/max_norm to the device copies (needed when ``step`` is replayed from a CUDA graph)."""
        for gi, ent in self._hyper.items():
            self._hyper_tensor(gi, self.param_groups[gi], ent[0].device)

    # ------------------------------------------------------------------ step
    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        first = self._steps == 0
        amp = self._amp
        self._check_no_pending_accumulation()
        if self._flat is None and not self._bind_refused:
            # the engine may have been created after this optimizer (apex order: amp -> DDP), and a resumed optimizer
            # has _steps > 0 before its first step: bind whenever still unbound (existing momentum is carried over)
            self._try_bind()
        if self._flat is not None:
            fs = self._flat
            fs.engine.wait_for_gradients()
            group = self.param_groups[0]
            if self._ov_active and self._ov_applied == fs.master.numel():
                self._ov_applied = 0       # every bucket was updated behind its all-reduce during backward: only the buffers
                self._ema_buffers(self._hyper[0][0], None)
                self._steps += 1
                return loss
            if self._ov_applied:
                raise RuntimeError("FusedSGD(overlap_backward=True): only %d of %d elements were updated during backward" %
                                   (self._ov_applied, fs.master.numel()))
            hyper = self._hyper_tensor(0, group, fs.master.device)
            if amp is not None:
                amp.attach_hyper(hyper)
            from .. import _ext
            step_hyper = self._clip_flat(hyper, amp.found_inf if amp is not None else None) if self._clip is not None else hyper
            if self._larc is not None:
                self._larc_flat(step_hyper, amp.found_inf if amp is not None else None, first)
            else:
                _ext.note_launch()
                _ext.lib().fused_sgd_flat(fs.engine.grad_arena(), fs.master, fs.momentum, fs.model_copy, step_hyper,
                                          amp.found_inf if amp is not None else None, bool(group["nesterov"]), first,
                                          ema=self._ema_flat)
            self._ema_buffers(hyper, amp.found_inf if amp is not None else None)
            if amp is not None:
                amp.update()
        else:
            clipped = self._clip_multi(amp) if self._clip is not None else None
            for gi, group in enumerate(self.param_groups):
                self._step_group(gi, group, first, amp, clipped)
            self._ema_buffers_multi(amp)
            if amp is not None:
                amp.update()
        self._steps += 1
        return loss

    def _check_no_pending_accumulation(self):
        """An engine with fp32_grad_accumulation keeps no_sync passes in its accumulator until a synchronising backward
        folds them in: a step before that would apply the previous step's gradients (flat) or none at all."""
        if self._flat is not None:
            engines = (self._flat.engine,)
        else:
            refs = {getattr(p, "_ptd_engine", None) for g in self.param_groups for p in g["params"]}
            engines = [ref() for ref in refs if ref is not None]
        for eng in engines:
            if eng is not None and getattr(eng, "accum_pending", False):
                raise RuntimeError("FusedSGD.step(): the gradient engine holds accumulated no_sync() passes that no synchronising "
                                   "backward has reduced yet - run the last micro-batch's backward outside no_sync() first")

    def _step_group(self, gi, group, first, amp, clipped=None):
        """``clipped``: what ``_clip_multi`` returned for this step (clipped hyper copies, or the PyTorch path's coefficient)."""
        params = [p for p in group["params"] if p.grad is not None]
        if not params:
            return
        bufs = []
        for p in params:
            st = self.state[p]
            if "momentum_buffer" not in st:
                st["momentum_buffer"] = torch.zeros_like(p, dtype=torch.float32, memory_format=torch.preserve_format)
                st["_fresh"] = True
            bufs.append(st["momentum_buffer"])
        if self._kernel_group(params):
            from .. import _ext
            C = _ext.lib()
            hyper = self._hyper_tensor(gi, group, params[0].device)
            if amp is not None:
                amp.attach_hyper(hyper)
            if clipped is not None:
                hyper = clipped[gi]
            fresh = [p for p in params if self.state[p].pop("_fresh", False)]

            def master_of(p):
                """fp32 tensor the kernel updates for a low-precision parameter (multi-tensor mode of a bf16 / fp16 model without
                a flat engine, e.g. under hvd.DistributedOptimizer); the parameter itself is refreshed from it as the model copy."""
                st = self.state[p]
                if "master" not in st:
                    init = getattr(p, "_ptd_master_init", None)         # fp32 values stashed by amp.cast_model
                    st["master"] = (init if init is not None else p.detach().float()).clone(memory_format=torch.preserve_format)
                    if init is not None:
                        del p._ptd_master_init
                return st["master"]

            if self._larc is not None:
                # one call: every norm of the group is formed before any update; `fresh` travels as a per-tensor first flag
                rows = self._larc_rows()
                trust, clip, eps = self._larc
                fresh_ids = {id(p) for p in fresh}
                _ext.note_launch(2)
                C.larc_sgd_multi([p.grad for p in params], [p if p.dtype == torch.float32 else master_of(p) for p in params],
                                 [self.state[p]["momentum_buffer"] for p in params],
                                 [None if p.dtype == torch.float32 else p.data for p in params], hyper,
                                 amp.found_inf if amp is not None else None, bool(group["nesterov"]),
                                 [id(p) in fresh_ids for p in params], [rows[id(p)] for p in params],
                                 self._larc_stats_on(params[0].device), trust, eps, clip, ema=self._ema_multi_lists(params))
                return
            fs = set(fresh) if (fresh and len(fresh) != len(params)) else None      # rare: first gradient later than the others
            for first_flag, sub in ((True, fresh), (False, [p for p in params if p not in fs])) if fs is not None else ((bool(fresh), params),):
                full = [p for p in sub if p.dtype == torch.float32]
                low = [p for p in sub if p.dtype != torch.float32]
                if full:
                    C.fused_sgd_multi([p.grad for p in full], full, [self.state[p]["momentum_buffer"] for p in full], [], hyper,
                                      amp.found_inf if amp is not None else None, bool(group["nesterov"]), first_flag,
                                      ema=self._ema_multi_lists(full))
                if low:
                    C.fused_sgd_multi([p.grad for p in low], [master_of(p) for p in low], [self.state[p]["momentum_buffer"] for p in low],
                                      [p.data for p in low], hyper, amp.found_inf if amp is not None else None, bool(group["nesterov"]),
                                      first_flag, ema=self._ema_multi_lists(low))
        else:
            if amp is not None and amp.host_found_inf():
                return
            gmul = amp.host_inv_scale() if amp is not None else 1.0
            rows = self._larc_rows() if self._larc is not None else None
            for p, buf in zip(params, bufs):
                fresh = self.state[p].pop("_fresh", False)
                g = p.grad if gmul == 1.0 else p.grad.float() * gmul
                if clipped is not None:
                    g = g * clipped
                st = self.state[p]
                if p.dtype != torch.float32 and "master" not in st:
                    st["master"] = p.detach().float().clone()
                master = p if p.dtype == torch.float32 else st["master"]
                wd = group["weight_decay"]
                if rows is not None:
                    trust, clip, eps = self._larc
                    g, stats = larc_reference_grad(master, g, group["lr"], wd, trust, clip, eps)
                    self._larc_stats_on(p.device)[rows[id(p)]] = torch.tensor(stats)
                    wd = 0.0
                sgd_reference_step(master, g, buf, group["lr"], group["momentum"], wd, group["dampening"], group["nesterov"], fresh)
                if master is not p:
                    p.copy_(master)
                if self._ema is not None:
                    from ..utils.ema import ema_reference_
                    ema_reference_(self._ema.shadow_of(p), master, *self._ema.decay_pair())

    def _ema_buffers_multi(self, amp):
        """Buffer average after a multi-tensor or CPU step (the CPU path skips an overflowed step on the host)."""
        if self._ema is None:
            return
        live, shadow = self._ema.buffer_pairs()
        if not live:
            return
        if live[0].is_cuda:
            dev = live[0].device
            self._ema_buffers(self._hyper_tensor(0, self.param_groups[0], dev), amp.found_inf if amp is not None else None,
                              (live, shadow))
        elif amp is None or not amp.host_found_inf():
            from ..utils.ema import ema_reference_
            for b, e in zip(live, shadow):
                ema_reference_(e, b, *self._ema.decay_pair())

    def zero_grad(self, set_to_none: bool = True):
        super().zero_grad(set_to_none=set_to_none)

    def load_state_dict(self, state_dict):
        """Standard ``Optimizer.load_state_dict``; in flat mode the loaded momentum is copied INTO the flat buffer
        (the kernel reads that buffer, not the per-parameter tensors) and the state entries are re-pointed at its views."""
        # torch casts loaded state to the parameter's dtype, but momentum and masters are fp32 whatever the model copy is (the
        # kernels require it): put the saved fp32 values back, for every order of binding (bound now, bound later through
        # bind_flat_optimizer, or never: multi-tensor / CPU)
        saved_ids = [i for g in state_dict["param_groups"] for i in g["params"]]
        own = [p for g in self.param_groups for p in g["params"]]
        saved = {id(p): {k: v for k, v in state_dict["state"].get(i, {}).items() if k in _FP32_STATE and torch.is_tensor(v)}
                 for p, i in zip(own, saved_ids)}
        super().load_state_dict(state_dict)
        for p in own:
            for k, v in saved[id(p)].items():
                self.state[p][k] = v.to(device=p.device, dtype=torch.float32)
        loaded = False
        if self._flat is not None:
            eng = self._flat.engine
            with torch.no_grad():
                for i, p in enumerate(eng.params):
                    buf = self.state.get(p, {}).get("momentum_buffer")
                    off, cnt = eng.param_elem_off[i], p.numel()
                    view = self._flat.momentum[off:off + cnt].as_strided(p.size(), p.stride())
                    if buf is not None and buf.data_ptr() != view.data_ptr():
                        view.copy_(buf.to(view.dtype))
                        loaded = True
                    self.state[p]["momentum_buffer"] = view
        else:
            loaded = any("momentum_buffer" in st for st in self.state.values())
        if loaded:
            self._steps = max(self._steps, 1)      # do not re-initialise the momentum on the next step
            for ent in self._hyper.values():
                ent[0][5].fill_(0.0)
