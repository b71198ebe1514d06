"""Per-op time of ``augment_normalize`` (csrc/augment.cu) against ``normalize_nhwc`` at 256 x 3 x 224 x 224, bf16 channels_last,
with bytes computed from the shapes and the share of 3.35 TB/s (H100 SXM HBM3); for context, torchvision v2 run per sample on
CUDA tensors.  Prints one JSON line per row, each with the card's name, power limit and SM clock.

AutoAugment rows (two launches through a uint8 scratch batch): one per ImageNet sub-policy with both ops forced on, one
per policy for a drawn batch, and the host ``draw()`` time of each policy.  The bytes are the same read-once-write-once
bound; the scratch batch's write and read are not counted.

    python tools/augment_bench.py [--batch 256] [--size 224] [--iters 50] [--tv-samples 64]
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

PEAK = 3.35e12


def _time(fn, iters):
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--size", type=int, default=224)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--tv-samples", type=int, default=64)
    a = ap.parse_args()
    from pytorch_distributed_b200 import _ext
    from pytorch_distributed_b200.ops import augment as A
    C = _ext.lib()
    n, H = a.batch, a.size
    src = torch.randint(0, 256, (n, 3, H, H), dtype=torch.uint8, device="cuda")
    ca = torch.tensor([0.0171, 0.0175, 0.0174], device="cuda")
    cb = torch.tensor([-2.1, -2.0, -1.8], device="cuda")
    moved = n * 3 * H * H * (1 + 2)                   # uint8 read + bf16 write
    ms = _time(lambda: C.normalize_nhwc(src, ca, cb, 1, True), a.iters)
    rows = [{"op": "normalize_nhwc", "ms": ms, "bytes": moved}]
    for op, name in enumerate(A.op_names()):
        prm = torch.zeros(n, A.AUG_PRM)
        for s in range(n):
            code = A.encode(op, s % A.NUM_BINS, bool(s & 1), H, H)
            prm[s, :len(code)] = torch.tensor(code)
        prm[:, 7] = 1.0
        prm[:, 8:12] = torch.tensor([50, 60, 40, 30])   # an erase box in every sample
        prm = prm.cuda()
        # a per-image statistic reads the sample twice (L2 serves the second read at this size, HBM bytes are counted once)
        ms = _time(lambda: C.augment_normalize(src, prm, ca, cb, 1, True), a.iters)
        rows.append({"op": name, "ms": ms, "bytes": moved})
    for r in rows:
        r["GBps"] = r["bytes"] / (r["ms"] * 1e-3) / 1e9
        r["share_of_3.35TBps"] = r["bytes"] / PEAK / (r["ms"] * 1e-3)
        r["bound"] = "memory"
    # torchvision v2 per sample on CUDA tensors (TrivialAugmentWide + Normalize + RandomErasing), scaled to the batch
    from torchvision.transforms import InterpolationMode
    from torchvision.transforms import v2 as T
    tf = T.Compose([T.TrivialAugmentWide(interpolation=InterpolationMode.BILINEAR), T.ToDtype(torch.float32, scale=True),
                    T.Normalize([0.485, 0.456, 0.406], [0.229, 0.224, 0.225]), T.RandomErasing(0.1)])
    k = min(a.tv_samples, n)
    ms = _time(lambda: [tf(src[s]) for s in range(k)], max(3, a.iters // 10)) * n / k
    rows.append({"op": "torchvision_v2_per_sample", "ms": ms, "bytes": moved, "GBps": moved / (ms * 1e-3) / 1e9,
                 "share_of_3.35TBps": moved / PEAK / (ms * 1e-3), "bound": "launch/host"})
    rows += autoaugment_rows(C, A, src, ca, cb, n, H, a.iters, moved)
    card = device_info()
    for r in rows:
        r.update(card, batch=n, size=H)
        if "ms" in r:
            r["us"] = r["ms"] * 1e3
            r["TBps"] = r["bytes"] / (r["ms"] * 1e-3) / 1e12
        print(json.dumps(r))


def device_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader",
                        "-i", str(torch.cuda.current_device())], capture_output=True, text=True)
    name, power, clock = ([v.strip() for v in q.stdout.split(",")] + ["?"] * 3)[:3] if q.returncode == 0 else ["?"] * 3
    return {"device": torch.cuda.get_device_name(), "power_limit": power, "sm_clock": clock, "nvidia_smi_name": name}


def autoaugment_rows(C, A, src, ca, cb, n, H, iters, moved):
    rows = []
    table = torch.from_numpy(A.chain_table("imagenet", H, H))
    for i, sub in enumerate(A.sub_policies("imagenet")):
        idx = torch.tensor([16 * i + 12 + (s & 3) for s in range(n)])    # both entries applied, the four sign patterns
        prm = table[idx].clone()
        prm[:, 7] = 1.0
        prm[:, 8:12] = torch.tensor([50, 60, 40, 30])
        prm = prm.cuda()
        ms = _time(lambda: C.augment_normalize(src, prm, ca, cb, 1, True), iters)
        rows.append({"op": "imagenet[%d] %s+%s" % (i, sub[0][0], sub[1][0]), "ms": ms, "bytes": moved})
    for policy in A.AUTOAUGMENT_POLICIES:
        aug = A.BatchAugment(policy, 0.1, seed=0)
        prm = aug.draw(n, H, H).cuda()
        ms = _time(lambda: C.augment_normalize(src, prm, ca, cb, 1, True), iters)
        rows.append({"op": "drawn batch: %s" % policy, "ms": ms, "bytes": moved})
    for policy in ("ta_wide",) + A.AUTOAUGMENT_POLICIES:
        aug = A.BatchAugment(policy, 0.1, seed=0)
        aug.draw(n, H, H)
        t0 = time.perf_counter()
        for _ in range(20):
            aug.draw(n, H, H)
        rows.append({"op": "host draw(): %s" % policy, "host_ms": (time.perf_counter() - t0) / 20 * 1e3})
    for r in rows:
        if "ms" in r:
            r["GBps"] = r["bytes"] / (r["ms"] * 1e-3) / 1e9
            r["share_of_3.35TBps"] = r["bytes"] / PEAK / (r["ms"] * 1e-3)
            r["bound"] = "memory"
    return rows


if __name__ == "__main__":
    main()
