"""``ModelEma``: an exponential moving average of a model's weights (timm ``ModelEmaV2`` / torchvision ``--model-ema``).

After every applied optimizer step, for each parameter with ``p`` its fp32 master value after the update, and for each
floating-point buffer (BatchNorm running statistics) with ``p`` its current value::

    e <- fmaf(d, e, w * p)          fp32, d = decay, w = fp32(1 - d)

so ``d = 0`` gives ``e == p`` and ``d = 1`` leaves ``e`` unchanged, bit for bit.  Integer buffers (``num_batches_tracked``)
are copied from the live model whenever the average is read.

With a :class:`~pytorch_distributed_b200.ops.fused_sgd.FusedSGD` (also through ``apex.parallel.LARC``, horovod's
``DistributedOptimizer`` or amp) the average is updated inside the optimizer's own kernels, in the same pass that
writes the masters (``csrc/optim.cu``): it follows every mode of the step (flat, per bucket behind the all-reduce,
multi-tensor, LARC, CPU), skips the steps the loss scaler skips, lives in a CUDA graph with the step, and ``update()``
has nothing left to do.  With any other optimizer ``update()`` is one ``ema_multi`` launch (torch math on the CPU),
to be called after each ``optimizer.step()``.

The averages are kept in fp32.  ``module`` is a separate evaluation copy of the model (same dtypes and memory format as
the live model, no tensor shared with it); ``sync_module()`` writes the averages into it before it is evaluated.
"""
from __future__ import annotations

import copy
from collections import OrderedDict

import numpy as np
import torch


def _unwrap(model):
    return model.module if hasattr(model, "module") and isinstance(model.module, torch.nn.Module) else model


def _fused(optimizer):
    """The FusedSGD behind ``optimizer`` (LARC and horovod's wrapper forward to it), or None."""
    return optimizer if optimizer is not None and hasattr(optimizer, "attach_ema") else None


def decay_pair(decay: float):
    """``(d, w)`` as the kernels read them: ``d`` rounded to fp32 and ``w = fp32(1 - d)``."""
    d = np.float32(decay)
    return float(d), float(np.float32(1.0 - float(d)))


def _eval_copy(live: torch.nn.Module) -> torch.nn.Module:
    """Deep copy of ``live`` that shares no tensor, communicator or hook with it."""
    memo = {}
    for m in live.modules():
        sync = getattr(m, "_sync", None)        # synchronised BN: the copy finds its own context (eval never synchronises)
        if sync is not None:
            memo[id(sync)] = None
    module = copy.deepcopy(live, memo)
    inner_fwd = module.__dict__.get("forward")
    if inner_fwd is not None:
        # amp's forward wrapper closes over the live model: wrap the copy's own forward the same way
        del module.forward
        amp_args = getattr(inner_fwd, "_ptd_amp", None)
        if amp_args is None:
            raise RuntimeError("ModelEma: the model's forward is replaced by an unknown wrapper that a copy cannot re-create")
        from ..parallel.amp import _wrap_forward
        _wrap_forward(module, *amp_args)
    for m in module.modules():
        for name, b in list(m._buffers.items()):
            if b is not None:
                m._buffers[name] = b.clone(memory_format=torch.preserve_format)      # a buffer view must not keep its base
    for p in module.parameters():
        p.requires_grad_(False)
    module.eval()
    return module


def _master_value(p, optimizer):
    """fp32 value of the master weight of live parameter ``p``: the flat engine's master, the multi-tensor optimizer's
    master, the fp32 values amp.cast_model stashed for an optimizer that has not bound yet, or ``p`` itself."""
    ref = getattr(p, "_ptd_engine", None)
    eng = ref() if ref is not None else None
    if eng is not None and getattr(eng, "_flat", None) is not None:
        idx = {id(q): i for i, q in enumerate(eng.params)}
        if id(p) in idx:
            return eng.master_params()[idx[id(p)]]
    if optimizer is not None:
        m = optimizer.state.get(p, {}).get("master") if hasattr(optimizer, "state") else None
        if m is not None:
            return m
    init = getattr(p, "_ptd_master_init", None)
    return init if init is not None else p.detach()


class ModelEma:
    def __init__(self, model: torch.nn.Module, decay: float = 0.9999, optimizer=None):
        self._check(decay)
        self._decay = float(decay)
        self.live = _unwrap(model)
        self._wrapper = model if model is not self.live else None
        self.module = _eval_copy(self.live)
        self._opt = optimizer
        self._fused = _fused(optimizer)
        names = {id(p): n for n, p in self.live.named_parameters()}
        self.param_names = list(names.values())
        self.buffer_names = [n for n, b in self.live.named_buffers() if b.is_floating_point()]
        self.shadow = OrderedDict()
        with torch.no_grad():
            for n, p in self.live.named_parameters():
                self.shadow[n] = _master_value(p, optimizer).detach().to(torch.float32).clone(memory_format=torch.preserve_format)
            for n, b in self.live.named_buffers():
                if b.is_floating_point():
                    self.shadow[n] = b.detach().to(torch.float32).clone(memory_format=torch.preserve_format)
        self._param_of = {id(p): n for n, p in self.live.named_parameters()}
        dev = next(iter(self.shadow.values())).device if self.shadow else torch.device("cpu")
        self._dw = torch.tensor(decay_pair(self._decay), dtype=torch.float32, device=dev)
        self._flag = torch.zeros(1, dtype=torch.int32, device=dev)     # multi_tensor_scale's non-finite flag (unused here)
        if self._fused is not None:
            self._fused.attach_ema(self)

    @torch.no_grad()
    def reset(self) -> None:
        """Start the average again from the live model's current fp32 masters and buffers (e.g. after loading weights)."""
        params = dict(self.live.named_parameters())
        bufs = dict(self.live.named_buffers())
        for n, e in self.shadow.items():
            e.copy_(_master_value(params[n], self._opt) if n in params else bufs[n])

    @staticmethod
    def _check(decay):
        if not (0.0 <= float(decay) <= 1.0):
            raise ValueError("ModelEma decay must lie in [0, 1], got %r" % (decay,))

    # ------------------------------------------------------------------ decay
    @property
    def decay(self) -> float:
        return self._decay

    @decay.setter
    def decay(self, value: float) -> None:
        self._check(value)
        self._decay = float(value)
        self._dw.copy_(torch.tensor(decay_pair(self._decay), dtype=torch.float32))
        if self._fused is not None:
            self._fused.refresh_hyper()

    def decay_pair(self):
        return decay_pair(self._decay)

    # ------------------------------------------------------------------ what the optimizer reads
    def shadow_of(self, p) -> torch.Tensor:
        """fp32 average of live parameter ``p``."""
        return self.shadow[self._param_of[id(p)]]

    def set_shadow_of(self, p, t: torch.Tensor) -> None:
        self.shadow[self._param_of[id(p)]] = t

    def buffer_pairs(self):
        """(live float buffers, their fp32 averages), in ``named_buffers`` order.  Under our DistributedDataParallel every
        rank must average rank 0's buffers: the deferred broadcast has already joined when the step runs, the immediate one
        (library collectives) only comes before the next forward, so it is run here once more (the next forward's
        broadcast then finds the same values)."""
        ddp = self._wrapper
        if (ddp is not None and getattr(ddp, "broadcast_buffers", False) and hasattr(ddp, "_broadcast_buffers_now")
                and not getattr(ddp, "_deferred", True) and ddp.comm.world > 1 and ddp._buffers_f):
            ddp._broadcast_buffers_now()
        live = dict(self.live.named_buffers())
        return [live[n] for n in self.buffer_names], [self.shadow[n] for n in self.buffer_names]

    # ------------------------------------------------------------------ update
    @torch.no_grad()
    def update(self) -> None:
        """One EMA step over every parameter and float buffer.  A no-op when a FusedSGD does it inside its step."""
        if self._fused is not None:
            return
        if getattr(self._opt, "_amp_last_skipped", False):     # amp skipped the stock optimizer's step on overflow
            return
        live = dict(self.live.named_parameters())
        src = [live[n].detach() for n in self.param_names]
        dst = [self.shadow[n] for n in self.param_names]
        bsrc, bdst = self.buffer_pairs()
        src, dst = src + bsrc, dst + bdst
        if not dst:
            return
        if dst[0].is_cuda:
            from .. import _ext
            _ext.note_launch()
            _ext.lib().ema_multi(src, dst, self._dw, None)
        else:
            d, w = self.decay_pair()
            for s, e in zip(src, dst):
                ema_reference_(e, s, d, w)

    @torch.no_grad()
    def sync_module(self) -> None:
        """Write the averages into ``module`` (in the module's dtypes) and copy the live integer buffers."""
        own = self.module.state_dict(keep_vars=True)
        src, dst = [], []
        for n, e in self.shadow.items():
            t = own[n]
            t = t.data if isinstance(t, torch.nn.Parameter) else t
            if t.stride() != e.stride():
                raise RuntimeError("ModelEma: %s has strides %s in the copy and %s in the average" % (n, t.stride(), e.stride()))
            src.append(e)
            dst.append(t)
        if dst and dst[0].is_cuda:
            from .. import _ext
            _ext.note_launch()
            _ext.lib().multi_tensor_scale(src, dst, 1.0, self._flag)
        else:
            for s, t in zip(src, dst):
                t.copy_(s)
        live = dict(self.live.named_buffers())
        for n, b in self.module.named_buffers():
            if not b.is_floating_point() and n in live:
                b.copy_(live[n])

    # ------------------------------------------------------------------ checkpoints
    def state_dict(self):
        """fp32 averages under the unwrapped model's ``state_dict`` keys (integer buffers: the live values)."""
        out = OrderedDict()
        for k, v in self.live.state_dict().items():
            if k in self.shadow:
                out[k] = self.shadow[k].detach().clone()
            else:
                out[k] = v.detach().clone() if torch.is_tensor(v) else v
        return out

    @torch.no_grad()
    def load_state_dict(self, state_dict) -> None:
        sd = state_dict
        if sd and all(k.startswith("module.") for k in sd):
            sd = {k[len("module."):]: v for k, v in sd.items()}
        missing = [k for k in self.shadow if k not in sd]
        if missing:
            raise KeyError("ModelEma.load_state_dict: missing %s" % (missing[:4],))
        for k, e in self.shadow.items():
            e.copy_(sd[k].to(device=e.device, dtype=torch.float32).reshape(e.shape))


def ema_reference_(e: torch.Tensor, p: torch.Tensor, d: float, w: float) -> None:
    """``e <- fmaf(d, e, w * p)`` on the CPU: ``w * p`` rounded to fp32, then ``d * e`` (exact in fp64) plus it, rounded
    once more to fp32 (a double rounding, unlike the kernels' single one: within one fp32 ulp of them)."""
    wp = (torch.tensor(w, dtype=torch.float32) * p.to(torch.float32)).double()
    e.copy_((torch.tensor(d, dtype=torch.float64) * e.double() + wp).to(torch.float32))
