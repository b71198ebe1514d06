"""CUDA-event time of one pass of ``grad_accumulate`` and of ``grad_fold`` (csrc/collectives.cu) over the real ResNet-50
bucket plan: the fused engine at world 1 with the command line's buckets (8 MiB cap, 1 MiB first and tail buckets, bf16
wire), bf16 gradients, one launch per bucket.  Prints one JSON line with the card, its power limit, the times, the bytes a
pass must move (accumulate: 2 B read of the gradient + 4 B read and 4 B write of the fp32 sum per element; fold: 2 B more
for the gradient written back) and their share of 3.35 TB/s (H100 SXM HBM3, data sheet), for a few CTA budgets.

    python tools/accum_bench.py [--iters 200]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

PEAK_BW = 3.35e12


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in q.split(",")]
        return name, power
    except Exception:  # noqa: BLE001
        return torch.cuda.get_device_name(0), "unknown"


def time_ms(fn, iters):
    for _ in range(10):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "accum_bench needs a GPU"
    from pytorch_distributed_b200.models import create_model
    from pytorch_distributed_b200.parallel import ddp
    from pytorch_distributed_b200.parallel.comm import FusedCommunicator
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    model = create_model("resnet50").to(dev).to(torch.bfloat16).to(memory_format=torch.channels_last)
    params = list(model.parameters())
    assert sum(p.numel() for p in params) == 25_557_032
    eng = ddp.GradientEngine(params, FusedCommunicator(device=dev), wire_dtype="bf16", bucket_cap_mb=8.0,
                             fp32_grad_accumulation=True)
    g = torch.Generator(device=dev).manual_seed(0)
    grads = [(torch.randn(p.shape, device=dev, generator=g) * 1e-3).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
             if p.dim() == 4 else (torch.randn(p.shape, device=dev, generator=g) * 1e-3).to(torch.bfloat16) for p in params]
    per_bucket = [[grads[i] for i in b.param_ids] for b in eng.buckets]

    def one_pass(fold):
        def run():
            for b, gs in zip(eng.buckets, per_bucket):
                eng._accumulate(b, gs, fold)
        return run

    elems = sum(p.numel() for p in params)
    b_acc, b_fold = elems * 10, elems * 12
    rows = []
    default = ddp.ACCUM_CTAS
    for ctas in sorted({32, default, 128, 264}):
        ddp.ACCUM_CTAS = ctas
        t_acc = time_ms(one_pass(False), a.iters)
        t_fold = time_ms(one_pass(True), a.iters)
        rows.append({"accum_ctas": ctas, "grad_accumulate_us": round(t_acc * 1e3, 1), "grad_fold_us": round(t_fold * 1e3, 1),
                     "grad_accumulate_share_of_3.35TBps": round(b_acc / (t_acc * 1e-3) / PEAK_BW, 3),
                     "grad_fold_share_of_3.35TBps": round(b_fold / (t_fold * 1e-3) / PEAK_BW, 3)})
    ddp.ACCUM_CTAS = default
    name, power = card()
    print(json.dumps({"card": name, "power_limit": power, "elements": elems, "buckets": len(eng.buckets),
                      "plan_ctas": [b.plan.grid for b in eng.buckets], "default_accum_ctas": default, "iters": a.iters,
                      "grad_accumulate_bytes": b_acc, "grad_fold_bytes": b_fold, "runs": rows}))


if __name__ == "__main__":
    main()
