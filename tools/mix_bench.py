"""CUDA-event times of the MixUp / CutMix batch kernel and of the soft-target cross-entropy against the torch-op paths they
replace, at the ResNet-50 training shapes of one GPU: a 256 x 3 x 224 x 224 bf16 channels_last batch and [256, 1000] bf16
logits.  Prints one JSON line with the card, its power limit and SM clock, the times, and for ``mix_batch`` the bytes per
second against 3.35 TB/s (H100 SXM HBM3, data sheet) using the 154 MB lower bound (read the batch once, write it once).

    python tools/mix_bench.py [--iters 200]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

PEAK_BW = 3.35e12


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        return [s.strip() for s in q.split(",")]
    except Exception:  # noqa: BLE001
        return [torch.cuda.get_device_name(0), "unknown", "unknown", "unknown"]


def time_us(fn, iters):
    for _ in range(10):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) * 1e3 / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "mix_bench needs a GPU"
    from pytorch_distributed_b200 import _ext
    from pytorch_distributed_b200.ops.mix import CUTMIX, MIXUP, cutmix_box, lam_pair
    C = _ext.lib()
    dev = torch.device("cuda", 0)
    B, H, W, K = 256, 224, 224, 1000
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.randn(B, 3, H, W, device=dev, generator=g).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, K, (B,), device=dev, generator=g)
    out, yb, dom = torch.empty_like(x), torch.empty_like(y), torch.empty_like(y)
    lam = 0.7
    la, lb = lam_pair(lam)
    box, lam_c = cutmix_box(lam, 100, 120, H, W)
    lca, lcb = lam_pair(lam_c)
    prm_mix = torch.tensor([MIXUP, la, lb, 0, 0, 0, 0, 0], device=dev)
    prm_cut = torch.tensor([CUTMIX, lca, lcb, *box, 0], device=dev)
    x1, y1, x2, y2 = box
    bytes_lb = 2 * x.numel() * x.element_size()

    def torch_mixup():
        return x.roll(1, 0).mul_(1.0 - lam).add_(x.mul(lam))

    def torch_cutmix():
        o = x.clone()
        o[..., y1:y2, x1:x2] = x.roll(1, 0)[..., y1:y2, x1:x2]
        return o

    res = {}
    for name, prm, ref in (("mixup", prm_mix, torch_mixup), ("cutmix", prm_cut, torch_cutmix)):
        t = time_us(lambda: C.mix_batch(x, out, y, yb, dom, prm), a.iters)
        tr = time_us(ref, a.iters)
        res[name] = {"mix_batch_us": t, "torch_ops_us": tr, "speedup": tr / t, "bytes_lower_bound": bytes_lb,
                     "gb_per_s": bytes_lb / (t * 1e-6) / 1e9, "share_of_3.35TBps": bytes_lb / (t * 1e-6) / PEAK_BW}
    res["cutmix"]["box"] = box

    # cross-entropy: fused forward + backward against .float() + one-hot mixing + F.cross_entropy + backward
    z = (torch.randn(B, K, device=dev, generator=g) * 3).to(torch.bfloat16)
    eps = 0.1
    gone = torch.ones((), device=dev)

    def fused():
        loss, _, lse = C.soft_ce_fwd(z, y, yb, prm_mix, eps)
        return C.soft_ce_bwd(z, y, yb, prm_mix, lse, gone, eps)

    zr = z.detach().requires_grad_()

    def current():
        q = F.one_hot(yb, K).float().mul_(lb).add_(F.one_hot(y, K).float().mul(la))
        loss = F.cross_entropy(zr.float(), q, label_smoothing=eps)
        (d,) = torch.autograd.grad(loss, zr)
        return d

    res["soft_ce"] = {"shape": [B, K], "fused_fwd_bwd_us": time_us(fused, a.iters), "torch_fwd_bwd_us": time_us(current, a.iters)}
    res["soft_ce"]["speedup"] = res["soft_ce"]["torch_fwd_bwd_us"] / res["soft_ce"]["fused_fwd_bwd_us"]
    name, power, sm, sm_max = card()
    print(json.dumps({"card": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max, "iters": a.iters, **res}), flush=True)


if __name__ == "__main__":
    main()
