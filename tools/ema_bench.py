"""CUDA-event time of the fused SGD step with the EMA epilogue (``fused_sgd_flat(..., ema=...)``) against the plain step,
and of the standalone ``ema_multi`` pass over the same elements, at the ResNet-50 flat size: 25,557,032 parameters in the
engine's 64-element aligned layout, bf16 gradient arena, fp32 masters / momentum / average, bf16 model copy.  Prints one
JSON line with the card, its power limit, the times, the bytes each call must move and their share of 3.35 TB/s
(H100 SXM HBM3, data sheet).

    python tools/ema_bench.py [--iters 200]
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
    assert torch.cuda.is_available(), "ema_bench needs a GPU"
    from pytorch_distributed_b200 import _ext
    from pytorch_distributed_b200.models import create_model
    from pytorch_distributed_b200.parallel import plan as P
    C = _ext.lib()
    dev = torch.device("cuda", 0)
    shapes = [p.shape for p in create_model("resnet50").parameters()]
    numels = [s.numel() for s in shapes]
    assert sum(numels) == 25_557_032
    offs, n = P.tensor_layout(numels)
    g = torch.Generator(device=dev).manual_seed(0)
    grad = (torch.randn(n, device=dev, generator=g) * 1e-3).to(torch.bfloat16)
    master = torch.randn(n, device=dev, generator=g) * 0.05
    mom = torch.zeros(n, device=dev)
    copy = master.to(torch.bfloat16)
    ema = master.clone()
    hyper = torch.tensor([1e-4, 0.9, 1e-4, 0.0, 1.0, 0.0, 0.9999, 1e-4], dtype=torch.float32, device=dev)  # tiny lr: values stay put
    src = [master[o:o + k].view(s) for o, k, s in zip(offs, numels, shapes)]
    dst = [ema[o:o + k].view(s) for o, k, s in zip(offs, numels, shapes)]

    def sgd():
        C.fused_sgd_flat(grad, master, mom, copy, hyper, None, False, False)

    def sgd_ema():
        C.fused_sgd_flat(grad, master, mom, copy, hyper, None, False, False, ema=ema)

    def standalone():
        C.ema_multi(src, dst, hyper[6:8], None)

    runs = {"sgd": [], "sgd_ema": [], "ema_multi": []}
    for _ in range(3):                       # alternate the three, three rounds each
        runs["sgd"].append(time_ms(sgd, a.iters))
        runs["sgd_ema"].append(time_ms(sgd_ema, a.iters))
        runs["ema_multi"].append(time_ms(standalone, a.iters))
    med = {k: sorted(v)[1] for k, v in runs.items()}
    elems = sum(numels)
    # bytes of the parameters themselves (the alignment padding the flat kernel also streams is left out of all three):
    # SGD 2 R grad + 4 R/W master + 4 R/W momentum + 2 W copy; the epilogue adds 4 R + 4 W of the average; the standalone
    # pass reads the master and reads and writes the average
    b = {"sgd": elems * 20, "sgd_ema": elems * 28, "ema_multi": elems * 12}
    name, power = card()
    out = {"card": name, "power_limit": power, "elements": elems, "iters": a.iters,
           "epilogue_overhead_ms": round(med["sgd_ema"] - med["sgd"], 4)}
    for k in runs:
        out[k + "_ms"] = round(med[k], 4)
        out[k + "_ms_runs"] = [round(t, 4) for t in runs[k]]
        out[k + "_bytes"] = b[k]
        out[k + "_GBps"] = round(b[k] / (med[k] * 1e-3) / 1e9, 1)
        out[k + "_share_of_3.35TBps"] = round(b[k] / (med[k] * 1e-3) / PEAK_BW, 3)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
