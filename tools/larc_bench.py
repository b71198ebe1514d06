"""CUDA-event time of the LARC optimizer step (norm pass + update, ``larc_sgd_flat``) against the plain fused SGD step
(``fused_sgd_flat``) at the ResNet-50 flat size: 25,557,032 parameters in the engine's 64-element aligned layout, bf16
gradient arena, fp32 masters and momentum, bf16 model copy.  Prints one JSON line with the card, its power limit, the
times, the bytes each step must move and their share of 3.35 TB/s (H100 SXM HBM3, data sheet).

    python tools/larc_bench.py [--iters 200]
"""
import argparse
import json
import math
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
    assert torch.cuda.is_available(), "larc_bench needs a GPU"
    from pytorch_distributed_b200 import _ext
    from pytorch_distributed_b200.models import create_model
    from pytorch_distributed_b200.parallel import plan as P
    C = _ext.lib()
    dev = torch.device("cuda", 0)
    numels = [p.numel() for p in create_model("resnet50").parameters()]
    assert sum(numels) == 25_557_032
    offs, n = P.tensor_layout(numels)
    chunk = C.LARC_CHUNK
    info, ct = [], []
    for i, (o, k) in enumerate(zip(offs, numels)):
        info.append((o, k, len(ct), i))
        ct += [i] * math.ceil(k / chunk)
    g = torch.Generator(device=dev).manual_seed(0)
    grad = (torch.randn(n, device=dev, generator=g) * 1e-3).to(torch.bfloat16)
    master = torch.randn(n, device=dev, generator=g) * 0.05
    mom = torch.zeros(n, device=dev)
    copy = master.to(torch.bfloat16)
    hyper = torch.tensor([1e-4, 0.9, 1e-4, 0.0, 1.0, 0.0, 0, 0], dtype=torch.float32, device=dev)   # tiny lr: values stay put
    chunk_tensor = torch.tensor(ct, dtype=torch.int32, device=dev)
    info_t = torch.tensor(info, dtype=torch.int64, device=dev)
    partials = torch.zeros(2 * len(ct), device=dev)
    stats = torch.zeros(len(numels), 3, device=dev)

    def sgd():
        C.fused_sgd_flat(grad, master, mom, copy, hyper, None, False, False)

    def larc():
        C.larc_sgd_flat(grad, master, mom, copy, hyper, None, False, False, chunk_tensor, info_t, 0, len(ct), partials, stats, 0.02,
                        1e-8, True)

    t_sgd = time_ms(sgd, a.iters)
    t_larc = time_ms(larc, a.iters)
    t_sgd2 = time_ms(sgd, a.iters)              # alternate: the SGD figure before and after
    elems = sum(numels)
    # bytes each step needs for the parameters themselves (the 64-element alignment padding, which fused_sgd_flat also
    # streams, is left out of both so the two shares compare): SGD 2 R grad + 4 R/W master + 4 R/W momentum + 2 W copy;
    # LARC adds the norm pass (2 R grad + 4 R master) and the chunk partials (8 B written, 8 B read per chunk)
    b_sgd = elems * 20
    b_larc = elems * (6 + 20) + len(ct) * 8 * 2
    name, power = card()
    t_s = min(t_sgd, t_sgd2)
    print(json.dumps({
        "card": name, "power_limit": power, "elements": elems, "chunks": len(ct), "iters": a.iters,
        "fused_sgd_flat_ms": round(t_s, 4), "fused_sgd_flat_ms_runs": [round(t_sgd, 4), round(t_sgd2, 4)],
        "larc_sgd_flat_ms": round(t_larc, 4), "larc_overhead_ms": round(t_larc - t_s, 4),
        "fused_sgd_flat_bytes": b_sgd, "larc_sgd_flat_bytes": b_larc,
        "fused_sgd_flat_share_of_3.35TBps": round(b_sgd / (t_s * 1e-3) / PEAK_BW, 3),
        "larc_sgd_flat_share_of_3.35TBps": round(b_larc / (t_larc * 1e-3) / PEAK_BW, 3),
    }))


if __name__ == "__main__":
    main()
