"""Mixed precision with dynamic loss scaling - the apex.amp surface the reference uses.

Reference call sites (/root/reference/apex_distributed.py):
  :216  ``model, optimizer = amp.initialize(model, optimizer)``         (no opt_level => "O1")
  :328  ``with amp.scale_loss(loss, optimizer) as scaled_loss: scaled_loss.backward()``
  :330  ``optimizer.step()``                                            (skipped by amp on overflow)

Semantics kept from apex: O0 fp32 / O1 autocast with fp32 weights / O2 half model + fp32 master weights /
O3 pure half; dynamic scale starts at 2**16, halves on overflow (and the step is skipped), doubles after 2000 clean
steps.  H100-native execution: the scale, the growth tracker and the overflow flag live on the device; the
unscale, the overflow test and the skipped step are folded into the fused optimizer kernel (``csrc/optim.cu``), and
under a data-parallel engine the non-finite test runs on the *reduced* gradients inside the all-reduce kernel, so
every rank takes the same decision without any extra collective or host synchronisation.
"""
from __future__ import annotations

import contextlib
from typing import Optional

import torch
import torch.nn as nn


class LossScaler:
    def __init__(self, device, loss_scale="dynamic", init_scale: float = 2.0 ** 16, growth_factor: float = 2.0,
                 backoff_factor: float = 0.5, growth_interval: int = 2000):
        self.device = torch.device(device)
        self.dynamic = loss_scale == "dynamic"
        s = init_scale if self.dynamic else float(loss_scale)
        self.scale = torch.full((1,), float(s), dtype=torch.float32, device=self.device)
        self.tracker = torch.zeros(1, dtype=torch.int32, device=self.device)
        self.found_inf = torch.zeros(1, dtype=torch.int32, device=self.device)
        self.growth_factor, self.backoff_factor, self.growth_interval = growth_factor, backoff_factor, growth_interval
        self._hyper = None            # hyper tensor attached last (the one amp_update_scale refreshes)
        self._hypers = []             # every hyper tensor ever attached (one per FusedSGD param group)
        self.skipped_steps_host = 0   # only maintained on the host-synchronising (stock optimizer) path

    # ---- device-side protocol used by FusedSGD
    def rebind_found_inf(self, t: torch.Tensor) -> None:
        """Use a flag word owned by someone else (the communicator's symmetric header)."""
        t.copy_(self.found_inf)
        self.found_inf = t

    def attach_hyper(self, hyper: torch.Tensor) -> None:
        if self._hyper is not hyper:
            self._hyper = hyper
            hyper[4:5].copy_(1.0 / self.scale)
        if not any(h is hyper for h in self._hypers):
            self._hypers.append(hyper)

    def update(self) -> None:
        """Post-step: run the scale state machine, refresh 1/scale for the optimizer, clear the overflow flag."""
        if self.device.type == "cuda":
            from .. import _ext
            hyper = self._hyper if self._hyper is not None else torch.empty(0, device=self.device)
            # every param group has its own hyper tensor; amp_update_scale refreshes the last attached one, the others get
            # the same treatment here: momentum_pending (slot 5) stays set only if this step was skipped, and 1/scale (slot 4)
            others = [h for h in self._hypers if h is not hyper or not self.dynamic]
            for h in others:
                if h.numel() >= 6:
                    h[5:6].mul_(self.found_inf)
            if self.dynamic:
                _ext.note_launch()
                _ext.lib().amp_update_scale(self.scale, self.tracker, self.found_inf, self.growth_factor, self.backoff_factor,
                                            self.growth_interval, hyper)
                for h in others:
                    h[4:5].copy_(hyper[4:5])
            else:
                self.found_inf.zero_()
        else:
            bad = bool(self.found_inf.item())
            if self.dynamic:
                if bad:
                    self.scale.mul_(self.backoff_factor).clamp_(min=1.0)
                    self.tracker.zero_()
                else:
                    self.tracker.add_(1)
                    if int(self.tracker.item()) >= self.growth_interval:
                        self.scale.mul_(self.growth_factor)
                        self.tracker.zero_()
            self.found_inf.zero_()
            for h in self._hypers:
                h[4:5].copy_(1.0 / self.scale)

    # ---- host-synchronising helpers (CPU path and stock torch optimizers)
    def host_found_inf(self) -> bool:
        return bool(self.found_inf.item())

    def host_inv_scale(self) -> float:
        return 1.0 / float(self.scale.item())

    def loss_scale(self) -> float:
        return float(self.scale.item())

    def state_dict(self):
        return {"loss_scale": float(self.scale.item()), "unskipped": int(self.tracker.item())}

    def load_state_dict(self, sd):
        self.scale.fill_(float(sd["loss_scale"]))
        self.tracker.fill_(int(sd.get("unskipped", 0)))


class _AmpState:
    def __init__(self):
        self.scaler: Optional[LossScaler] = None
        self.opt_level = "O0"
        self.half_dtype = torch.float16
        self.enabled = False


_amp_state = _AmpState()


def _is_bn(m: nn.Module) -> bool:
    return isinstance(m, nn.modules.batchnorm._BatchNorm)


def cast_model(model: nn.Module, dtype: torch.dtype, keep_batchnorm_fp32: bool = True) -> nn.Module:
    """Cast parameters in place (same Parameter objects => existing optimizers stay valid); running statistics and
    integer buffers stay as they are.  The fp32 values are stashed so fp32 master weights lose nothing."""
    from ..models.resnet import BNAct
    for m in model.modules():
        native_bn = isinstance(m, BNAct)
        if _is_bn(m) and keep_batchnorm_fp32 and not native_bn:
            continue
        for p in m.parameters(recurse=False):
            if p.is_floating_point() and p.dtype != dtype:
                p._ptd_master_init = p.data.clone()
                p.data = p.data.to(dtype)
        if not _is_bn(m):
            for name, b in list(m._buffers.items()):
                if b is not None and b.is_floating_point():
                    m._buffers[name] = b.to(dtype)
    return model


def _wrap_forward(model: nn.Module, autocast_dtype: Optional[torch.dtype], input_dtype: Optional[torch.dtype]):
    inner = model.forward

    def forward(*args, **kwargs):
        if input_dtype is not None:
            args = tuple(a.to(input_dtype) if torch.is_tensor(a) and a.is_floating_point() else a for a in args)
        if autocast_dtype is not None:
            dev = next(model.parameters()).device.type
            with torch.autocast(device_type=dev, dtype=autocast_dtype):
                return inner(*args, **kwargs)
        return inner(*args, **kwargs)

    forward._ptd_amp = (autocast_dtype, input_dtype)        # lets a copy of the model (ModelEma) be wrapped the same way
    model.forward = forward
    return model


def initialize(models, optimizers=None, enabled: bool = True, opt_level: str = "O1", cast_model_type=None,
               keep_batchnorm_fp32=None, master_weights=None, loss_scale=None, half_dtype: torch.dtype = torch.float16,
               verbosity: int = 1, **scaler_kw):
    """apex.amp.initialize equivalent.  Returns ``(models, optimizers)`` with the same container shapes."""
    single_model = not isinstance(models, (list, tuple))
    model_list = [models] if single_model else list(models)
    single_opt = optimizers is not None and not isinstance(optimizers, (list, tuple))
    opt_list = [] if optimizers is None else ([optimizers] if single_opt else list(optimizers))
    if opt_level not in ("O0", "O1", "O2", "O3"):
        raise RuntimeError("Unexpected optimization level %r (options are 'O0', 'O1', 'O2', 'O3')" % (opt_level,))
    st = _amp_state
    st.enabled = enabled and opt_level != "O0"
    st.opt_level = opt_level
    st.half_dtype = half_dtype
    if not enabled:
        return (models, optimizers) if optimizers is not None else models
    device = next(model_list[0].parameters()).device
    if loss_scale is None:
        loss_scale = "dynamic" if opt_level in ("O1", "O2") else 1.0
    if half_dtype == torch.bfloat16 and loss_scale == "dynamic" and opt_level != "O0":
        loss_scale = 1.0  # bf16 has fp32's exponent range: no scaling needed
    st.scaler = LossScaler(device, loss_scale, **scaler_kw)
    if verbosity and (not torch.distributed.is_initialized() or torch.distributed.get_rank() == 0):
        print("Selected optimization level %s: %s, loss_scale=%s" % (opt_level, str(half_dtype).replace("torch.", ""), loss_scale))
    for m in model_list:
        if opt_level == "O1":
            _wrap_forward(m, half_dtype, None)
        elif opt_level in ("O2", "O3"):
            keep = (opt_level == "O2") if keep_batchnorm_fp32 is None else bool(keep_batchnorm_fp32)
            cast_model(m, half_dtype, keep_batchnorm_fp32=keep)
            _wrap_forward(m, None, half_dtype)
    for o in opt_list:
        o._amp = st.scaler
        if not hasattr(o, "is_flat"):
            _patch_stock_optimizer(o, st.scaler)
    if optimizers is None:
        return models
    return models, optimizers


def _patch_stock_optimizer(opt, scaler: LossScaler):
    """torch.optim.* under amp: skip the step when the last unscale found non-finite gradients."""
    inner = opt.step

    def step(*a, **kw):
        skip = bool(getattr(opt, "_amp_skip", False))
        opt._amp_last_skipped = skip            # read by ModelEma.update(): a skipped step is not averaged either
        if skip:
            opt._amp_skip = False
            return None
        return inner(*a, **kw)

    opt.step = step


def _grads_of(opt):
    return [p.grad for g in opt.param_groups for p in g["params"] if p.grad is not None]


@contextlib.contextmanager
def scale_loss(loss, optimizers, loss_id: int = 0, model=None, delay_unscale: bool = False):
    """``with amp.scale_loss(loss, optimizer) as scaled_loss: scaled_loss.backward()``"""
    st = _amp_state
    if not st.enabled or st.scaler is None:
        yield loss
        return
    scaler = st.scaler
    yield loss.float() * scaler.scale.to(loss.device)
    if delay_unscale:
        return
    opts = optimizers if isinstance(optimizers, (list, tuple)) else [optimizers]
    for opt in opts:
        if hasattr(opt, "is_flat"):          # FusedSGD: unscale + skip happen inside the optimizer kernel
            eng_checks = opt.is_flat and getattr(opt._flat.engine, "check_inf", False)
            if not eng_checks:
                grads = _grads_of(opt)
                if grads and grads[0].is_cuda:
                    from .. import _ext
                    _ext.lib().multi_tensor_scale(grads, grads, 1.0, scaler.found_inf)
                elif grads:
                    bad = any(not torch.isfinite(g).all() for g in grads)
                    if bad:
                        scaler.found_inf.fill_(1)
            continue
        # stock optimizer: explicit unscale pass + host-side decision (one sync, like apex)
        grads = _grads_of(opt)
        inv = scaler.host_inv_scale()
        if grads and grads[0].is_cuda:
            from .. import _ext
            _ext.lib().multi_tensor_scale(grads, grads, inv, scaler.found_inf)
        else:
            for g in grads:
                if not torch.isfinite(g).all():
                    scaler.found_inf.fill_(1)
                g.mul_(inv)
        if scaler.host_found_inf():
            opt._amp_skip = True
            scaler.skipped_steps_host += 1
        scaler.update()


def master_params(optimizer):
    """Iterator over the fp32 master weights owned by ``optimizer`` (apex.amp.master_params)."""
    if getattr(optimizer, "is_flat", False):
        yield from optimizer._flat.engine.master_params()
        return
    for g in optimizer.param_groups:
        for p in g["params"]:
            st = optimizer.state.get(p, {})
            yield st.get("master", p)


def state_dict():
    s = _amp_state.scaler
    return {"loss_scaler0": s.state_dict()} if s is not None else {}


def load_state_dict(sd):
    if _amp_state.scaler is not None and "loss_scaler0" in sd:
        _amp_state.scaler.load_state_dict(sd["loss_scaler0"])


def current_scaler() -> Optional[LossScaler]:
    return _amp_state.scaler if _amp_state.enabled else None
