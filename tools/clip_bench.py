"""CUDA-event time of global-norm gradient clipping (``grad_sumsq_flat`` + ``clip_finalize``) at the ResNet-50 flat size:
25,557,032 parameters in the engine's 64-element aligned layout, bf16 gradient arena.  Also times the plain fused SGD
update (``fused_sgd_flat``) for scale.  Prints one JSON line with the card, its power limit, the times, the bytes the norm
pass must move and their share of 3.35 TB/s (H100 SXM HBM3, data sheet).

    python tools/clip_bench.py [--iters 200]
"""
import argparse
import json
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import torch  # noqa: E402

from larc_bench import PEAK_BW, card, time_ms  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "clip_bench needs a GPU"
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
    hyper = torch.tensor([1e-4, 0.9, 1e-4, 0.0, 1.0, 0.0, 0, 0, 1.0], dtype=torch.float32, device=dev)   # tiny lr: values stay put
    clipped = torch.zeros_like(hyper)
    chunk_tensor = torch.tensor(ct, dtype=torch.int32, device=dev)
    info_t = torch.tensor(info, dtype=torch.int64, device=dev)
    partials = torch.zeros(2 * len(ct), device=dev)
    total, count = torch.zeros((), device=dev), torch.zeros(1, dtype=torch.int32, device=dev)

    def norm():
        C.grad_sumsq_flat(grad, chunk_tensor, info_t, partials, hyper, None)

    def finalize():
        C.clip_finalize(partials, len(ct), [hyper], [clipped], None, total, count)

    def sgd():
        C.fused_sgd_flat(grad, master, mom, copy, clipped, None, False, False)

    t_norm = time_ms(norm, a.iters)
    t_fin = time_ms(finalize, a.iters)
    t_sgd = time_ms(sgd, a.iters)
    t_norm2 = time_ms(norm, a.iters)            # alternate: the norm figure before and after
    elems = sum(numels)
    b_norm = elems * 2 + len(ct) * 4            # bf16 gradient read once, one fp32 partial written per chunk
    t_n = min(t_norm, t_norm2)
    name, power = card()
    print(json.dumps({
        "card": name, "power_limit": power, "elements": elems, "chunks": len(ct), "iters": a.iters,
        "grad_sumsq_flat_ms": round(t_n, 4), "grad_sumsq_flat_ms_runs": [round(t_norm, 4), round(t_norm2, 4)],
        "clip_finalize_ms": round(t_fin, 4), "clip_total_ms": round(t_n + t_fin, 4), "fused_sgd_flat_ms": round(t_sgd, 4),
        "grad_sumsq_flat_bytes": b_norm, "grad_sumsq_flat_share_of_3.35TBps": round(b_norm / (t_n * 1e-3) / PEAK_BW, 3),
    }))


if __name__ == "__main__":
    main()
