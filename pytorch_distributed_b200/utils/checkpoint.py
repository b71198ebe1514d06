"""Checkpoint layout of the reference, plus an optional resume path.

Reference: ``save_checkpoint`` /root/reference/distributed.py:327-330 and its call site :218-225 - files
``checkpoint.pth.tar`` / ``model_best.pth.tar`` in the working directory, keys ``epoch`` (= epoch + 1), ``arch``,
``state_dict`` (the *unwrapped* module), ``best_acc1``.  The state dict written here is always fp32, whatever
precision the arenas / model copy run in.  ``--resume`` (SURVEY Q10) is an additive extension; optimizer and
loss-scaler state ride along under extra keys that a reference-style reader simply ignores, and so does
``state_dict_ema`` (``--model-ema``: the fp32 weight averages under the unwrapped module's keys).
"""
from __future__ import annotations

import os
import shutil

import torch


def export_state_dict(module: torch.nn.Module, engine=None, optimizer=None):
    """fp32 ``state_dict`` of the unwrapped module; master weights replace low-precision model copies (flat engines keep them
    in the engine, the multi-tensor optimizer path in ``optimizer.state[p]["master"]``)."""
    sd = module.state_dict()
    masters = {}
    if optimizer is not None:
        for name, p in module.named_parameters():
            m = optimizer.state.get(p, {}).get("master") if hasattr(optimizer, "state") else None
            if m is not None:
                masters[name] = m
    if engine is not None and hasattr(engine, "master_params"):
        idx = {id(p): i for i, p in enumerate(engine.params)}
        mp = engine.master_params()
        for name, p in module.named_parameters():
            if id(p) in idx:
                masters[name] = mp[idx[id(p)]]
    out = type(sd)()
    for k, v in sd.items():
        v = masters.get(k, v)
        if torch.is_tensor(v):
            v = v.detach()
            if v.is_floating_point() and v.dtype != torch.float32:
                v = v.float()
            v = v.cpu().contiguous().clone()
        out[k] = v
    return out


def export_ema_state_dict(ema):
    """``state_dict_ema``: fp32 CPU copy of :meth:`ModelEma.state_dict` (loads into a fresh model of the architecture)."""
    sd = ema.state_dict()
    return type(sd)((k, v.detach().cpu().contiguous() if torch.is_tensor(v) else v) for k, v in sd.items())


def save_checkpoint(state, is_best: bool, filename: str = "checkpoint.pth.tar", directory: str = ".") -> str:
    path = os.path.join(directory, filename)
    torch.save(state, path)
    if is_best:
        shutil.copyfile(path, os.path.join(directory, "model_best.pth.tar"))
    return path


def load_checkpoint(path: str, module: torch.nn.Module, optimizer=None, map_location="cpu", engine=None):
    ckpt = torch.load(path, map_location=map_location, weights_only=False)
    sd = ckpt["state_dict"]
    if all(k.startswith("module.") for k in sd):
        sd = {k[len("module."):]: v for k, v in sd.items()}
    with torch.no_grad():
        own = module.state_dict()
        for k, v in sd.items():
            if k in own:
                own[k].copy_(v.to(own[k].dtype))
        # low-precision model copies are derived from fp32 master weights: the masters must get the checkpoint too,
        # otherwise the next optimizer step would regenerate the model from stale masters
        # masters that do not exist yet (optimizer binds lazily at its first step) are seeded from the stash left by
        # amp.cast_model: point it at the checkpoint's fp32 values, otherwise the first step would discard the checkpoint
        for name, p in module.named_parameters():
            if getattr(p, "_ptd_master_init", None) is not None and name in sd:
                p._ptd_master_init = sd[name].detach().to(device=p.device, dtype=torch.float32).reshape(p.shape).clone()
        if engine is not None and hasattr(engine, "master_params"):
            idx = {id(p): i for i, p in enumerate(engine.params)}
            masters = engine.master_params()
            for name, p in module.named_parameters():
                if id(p) in idx and name in sd:
                    masters[idx[id(p)]].copy_(sd[name].to(device=masters[idx[id(p)]].device, dtype=torch.float32))
    if optimizer is not None and "optimizer" in ckpt:
        try:
            optimizer.load_state_dict(ckpt["optimizer"])
        except Exception as e:  # noqa: BLE001
            print("=> optimizer state not restored (%s)" % (e,))
    return ckpt
