"""``apex.parallel.LARC``: layer-wise adaptive rate control around an SGD optimizer.

Per parameter ``p`` with gradient ``g`` (after loss-scale unscaling), ``wd`` = the group's weight decay, ``lr`` = its lr::

    pn, gn = ||p||, ||g||
    if pn != 0 and gn != 0:
        f = trust_coefficient * pn / (gn + pn * wd + eps)
        if clip: f = min(f / lr, 1)
        g = (g + wd * p) * f          # where a norm is zero, g is left as is and gets no weight decay
    then the wrapped optimizer steps with weight_decay = 0

Wrapping a :class:`~pytorch_distributed_b200.ops.fused_sgd.FusedSGD` switches it into its LARC mode: the norms and the
update run in the fused sm_90a kernels (flat arena, per-bucket overlap, multi-tensor), on the device, CUDA-graph
capturable, with loss-scale unscaling and overflow skipping folded in as for plain SGD.  Any other optimizer gets the
algorithm above as a Python loop, as apex runs it.

Everything else is delegated to the wrapped optimizer, so the wrapper can stand wherever the optimizer stood: attribute
reads and writes it does not own (``_amp``, ``is_flat``, ``refresh_hyper``, ...) go to ``optim``.
"""
from __future__ import annotations

import torch


class LARC:
    # `step` stays on the wrapper: amp patches `opt.step` of the object it is given, and that patch must wrap LARC's step,
    # not the inner optimizer's (which LARC's step calls)
    _OWN = frozenset(("optim", "__dict__", "step"))
    _HYPER = ("trust_coefficient", "clip", "eps")

    def __init__(self, optimizer, trust_coefficient: float = 0.02, clip: bool = True, eps: float = 1e-8):
        object.__setattr__(self, "optim", optimizer)
        object.__setattr__(self, "trust_coefficient", trust_coefficient)
        object.__setattr__(self, "clip", clip)
        object.__setattr__(self, "eps", eps)
        self._push_hyper()

    def _push_hyper(self):
        """The fused optimizer takes the LARC settings as launch arguments: hand it every change (a step already captured
        in a CUDA graph keeps the values it was captured with)."""
        if hasattr(self.optim, "enable_larc"):
            self.optim.enable_larc(self.trust_coefficient, self.clip, self.eps)

    # ---- delegation
    def __getattr__(self, name):
        optim = self.__dict__.get("optim")
        if optim is None:
            raise AttributeError(name)
        return getattr(optim, name)

    def __setattr__(self, name, value):
        if name in self._OWN:
            object.__setattr__(self, name, value)
        elif name in self._HYPER:
            old = self.__dict__.get(name)
            object.__setattr__(self, name, value)
            try:
                self._push_hyper()
            except ValueError:
                object.__setattr__(self, name, old)
                raise
        else:
            setattr(self.optim, name, value)

    def __getstate__(self):
        return self.optim.__getstate__()

    def __setstate__(self, state):
        self.optim.__setstate__(state)

    def __repr__(self):
        return "LARC(trust_coefficient=%r, clip=%r, eps=%r)\n%r" % (self.trust_coefficient, self.clip, self.eps, self.optim)

    @property
    def state(self):
        return self.optim.state

    @property
    def param_groups(self):
        return self.optim.param_groups

    @param_groups.setter
    def param_groups(self, value):
        self.optim.param_groups = value

    def state_dict(self):
        return self.optim.state_dict()

    def load_state_dict(self, state_dict):
        self.optim.load_state_dict(state_dict)

    def zero_grad(self, *args, **kwargs):
        self.optim.zero_grad(*args, **kwargs)

    def add_param_group(self, param_group):
        self.optim.add_param_group(param_group)

    # ---- the step
    def step(self, closure=None):
        if hasattr(self.optim, "enable_larc"):
            return self.optim.step(closure) if closure is not None else self.optim.step()
        weight_decays = []
        try:
            with torch.no_grad():
                for group in self.optim.param_groups:
                    weight_decay = group.get("weight_decay", 0)
                    weight_decays.append(weight_decay)
                    group["weight_decay"] = 0
                    for p in group["params"]:
                        if p.grad is None:
                            continue
                        param_norm = torch.norm(p.data)
                        grad_norm = torch.norm(p.grad.data)
                        if param_norm != 0 and grad_norm != 0:
                            adaptive_lr = self.trust_coefficient * param_norm / (grad_norm + param_norm * weight_decay + self.eps)
                            if self.clip:
                                adaptive_lr = min(adaptive_lr / group["lr"], 1)
                            p.grad.data += weight_decay * p.data
                            p.grad.data *= adaptive_lr
            return self.optim.step(closure) if closure is not None else self.optim.step()
        finally:
            for group, weight_decay in zip(self.optim.param_groups, weight_decays):
                group["weight_decay"] = weight_decay
