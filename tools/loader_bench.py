#!/usr/bin/env python
"""Host-side throughput of the native shard loader vs the PIL/torchvision transform chain on the same pixels.

    python tools/loader_bench.py --records 2048 --threads 1,2,4,8
    python tools/loader_bench.py --device-resample --threads 1,2,4

Synthetic records (short side 256, 4:3) so that only the transform cost is measured; JPEG decoding - which the
ImageFolder path pays on every sample and the shard path paid once offline - is reported separately.

``--device-resample`` measures the staging mode instead (the threads copy crop regions and filter taps; the resample
runs on the GPU): host images/s per thread, and on a CUDA machine the ``resample_normalize`` kernel time per batch
(CUDA events over many launches), the bytes it reads and writes, and the bandwidth that implies.
"""
import argparse
import io
import os
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from pytorch_distributed_b200.utils import shards  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=2048)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--size", type=int, default=224)
    ap.add_argument("--threads", default="1,2,4,8")
    ap.add_argument("--epochs", type=int, default=3)
    ap.add_argument("--device-resample", action="store_true", help="measure the staging mode and the GPU resample kernel")
    ap.add_argument("--launches", type=int, default=200, help="kernel launches timed per batch (--device-resample)")
    a = ap.parse_args()
    rng = np.random.default_rng(0)
    tmp = tempfile.mkdtemp(prefix="ptds_bench_")
    base = rng.integers(0, 256, (64, 86, 3), dtype=np.uint8)
    from PIL import Image
    proto = np.asarray(Image.fromarray(base).resize((341, 256), Image.BICUBIC))      # smooth, photo-like spectrum
    path = os.path.join(tmp, "train-00000.ptds")
    with shards.ShardWriter(path, a.records) as w:
        for i in range(a.records):
            w.add(np.roll(proto, i, axis=1), i % 1000)
    if a.device_resample:
        staging(a, path)
        return
    print("| pipeline | threads / procs | images/s | per core |")
    print("|---|---:|---:|---:|")
    for t in [int(x) for x in a.threads.split(",")]:
        for train in (True, False):
            ld = shards.ShardLoader([path], a.batch, a.size, train=train, workers=t, depth=4, pin=False)
            n = 0
            for _ in ld:                      # warm-up epoch (page cache, thread start)
                pass
            t0 = time.perf_counter()
            for e in range(a.epochs):
                ld.sampler.set_epoch(e + 1)
                for x, y in ld:
                    n += x.shape[0]
            dt = time.perf_counter() - t0
            print("| native shards, %s | %d | %.0f | %.0f |" % ("train (RRC + flip)" if train else "val (resize + centre crop)", t, n / dt,
                                                               n / dt / t))
    # the reference's per-sample work on the same pixels, one process: PIL transforms (+ JPEG decode, quality 90)
    import torchvision.transforms as T
    tf = T.Compose([T.RandomResizedCrop(a.size), T.RandomHorizontalFlip(), T.PILToTensor()])
    img = Image.fromarray(proto)
    buf = io.BytesIO()
    img.save(buf, format="JPEG", quality=90)
    jpeg = buf.getvalue()
    torch.set_num_threads(1)
    for name, fn in (("PIL transforms only", lambda: tf(img)),
                     ("PIL JPEG decode + transforms (ImageFolder path)", lambda: tf(Image.open(io.BytesIO(jpeg)).convert("RGB")))):
        for _ in range(20):
            fn()
        t0 = time.perf_counter()
        k = 400
        for _ in range(k):
            fn()
        dt = time.perf_counter() - t0
        print("| %s | 1 | %.0f | %.0f |" % (name, k / dt, k / dt))


def staging(a, path):
    """Host rate of the staging threads, then (with a GPU) the device time of the resample kernel per batch."""
    print("| staging (device resample) | threads | images/s | per thread | MB staged / batch |")
    print("|---|---:|---:|---:|---:|")
    for t in [int(x) for x in a.threads.split(",")]:
        for train in (True, False):
            ld = shards.ShardLoader([path], a.batch, a.size, train=train, workers=t, depth=4, pin=False, device_resample=True)
            for _ in ld:                      # warm-up epoch (page cache, thread start)
                pass
            n, staged, batches = 0, 0, 0
            t0 = time.perf_counter()
            for e in range(a.epochs):
                ld.sampler.set_epoch(e + 1)
                for s, _ in ld:
                    n += s.n
                    staged += s.data.numel()
                    batches += 1
            dt = time.perf_counter() - t0
            print("| %s | %d | %.0f | %.0f | %.1f |" % ("train (RRC + flip)" if train else "val (resize + centre crop)", t, n / dt,
                                                     n / dt / t, staged / batches / 1e6))
    if not torch.cuda.is_available():
        print("no CUDA device: kernel time not measured")
        return
    import subprocess
    from pytorch_distributed_b200 import _ext
    from pytorch_distributed_b200.utils.data import IMAGENET_MEAN, IMAGENET_STD
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print("\ndevice: %s (name, power limit, max SM clock)" % (q.stdout.strip() or torch.cuda.get_device_name(0)))
    C = _ext.lib()
    a_ = torch.tensor([1.0 / (255.0 * s) for s in IMAGENET_STD], device="cuda")
    b_ = torch.tensor([-m / s for m, s in zip(IMAGENET_MEAN, IMAGENET_STD)], device="cuda")
    print("| resample_normalize, bf16 NHWC | batch | us / batch | MB read | MB written | GB/s | of 3.35 TB/s |")
    print("|---|---:|---:|---:|---:|---:|---:|")
    for train in (True, False):
        ld = shards.ShardLoader([path], a.batch, a.size, train=train, workers=4, depth=4, device_resample=True)
        times, read = [], 0
        for s, _ in ld:
            if s.n < a.batch:
                continue
            arena = s.data.cuda()
            for _ in range(10):
                C.resample_normalize(arena, s.n, s.out_h, s.out_w, s.max_rows, a_, b_, 1, True)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.launches):
                C.resample_normalize(arena, s.n, s.out_h, s.out_w, s.max_rows, a_, b_, 1, True)
            e1.record()
            e1.synchronize()
            times.append(e0.elapsed_time(e1) * 1e3 / a.launches)
            read += arena.numel()
            if len(times) == 4:
                break
        us = sum(times) / len(times)
        rd, wr = read / len(times), a.batch * 3 * a.size * a.size * 2
        gbs = (rd + wr) / us / 1e3
        print("| %s | %d | %.1f | %.1f | %.1f | %.0f | %.1f%% |" % ("train" if train else "val", a.batch, us, rd / 1e6, wr / 1e6, gbs,
                                                              100 * gbs / 3350))


if __name__ == "__main__":
    main()
