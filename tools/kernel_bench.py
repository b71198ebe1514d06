"""Isolated timing of the hand-written single-GPU kernels on ResNet-50 shapes (batch 256, bf16, NHWC).

    python tools/kernel_bench.py > kernel_bench_1gpu.md
    python tools/kernel_bench.py --once        # one launch per kernel, e.g. under a profiler

CUDA events on the launching stream, 3 warm-ups, L2 flushed (a 512 MB fill) before every timed launch; achieved
bandwidth = algorithmic bytes / time, fraction against the 3350 GB/s HBM3 bandwidth of the H100 SXM data sheet.
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from pytorch_distributed_b200 import _ext  # noqa: E402
from pytorch_distributed_b200.ops.bn_act import begin_step, bn_act  # noqa: E402
from pytorch_distributed_b200.ops.stem import bn_relu_maxpool  # noqa: E402

ONCE = "--once" in sys.argv
PEAK, SRC = 3350.0, "data-sheet"
dev = torch.device("cuda")
flush_buf = torch.empty(512 << 20, dtype=torch.uint8, device=dev)


def timeit(fn, reps=5):
    if ONCE:
        fn()
        torch.cuda.synchronize()
        return float("nan")
    for _ in range(3):
        fn()
    ts = []
    for _ in range(reps):
        flush_buf.fill_(1)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2]


def row(name, shape, ms, nbytes):
    gbs = nbytes / (ms * 1e-3) / 1e9 if ms == ms else float("nan")
    print("| %s | %s | %.1f | %.2f | %.0f | %.2f |" % (name, shape, ms * 1e3, nbytes / 1e9, gbs, gbs / PEAK), flush=True)


def main():
    C = _ext.lib()
    print("# Hand-written kernels in isolation, 1 x %s (bf16 NHWC, ResNet-50 shapes at batch 256)\n" % torch.cuda.get_device_name())
    print("CUDA events, median of 5, L2 flushed before each timed launch; fraction is of the %s HBM copy bandwidth (%.0f GB/s).\n" % (SRC, PEAK))
    print("| kernel(s) | shape | us | GB (algorithmic) | GB/s | frac of %s peak |" % SRC)
    print("|---|---|---:|---:|---:|---:|")
    B = 256
    shapes = [(64, 56, True, False), (256, 56, True, True), (128, 28, True, False), (512, 28, True, True), (256, 14, True, False),
              (1024, 14, True, True), (512, 7, True, False), (2048, 7, True, True), (256, 56, False, False)]
    for ch, hw, relu, res in shapes:
        x = torch.randn(B, ch, hw, hw, device=dev).bfloat16().contiguous(memory_format=torch.channels_last).requires_grad_(True)
        r = torch.randn(B, ch, hw, hw, device=dev).bfloat16().contiguous(memory_format=torch.channels_last).requires_grad_(True) if res else None
        w = torch.ones(ch, device=dev, dtype=torch.bfloat16, requires_grad=True)
        b = torch.zeros(ch, device=dev, dtype=torch.bfloat16, requires_grad=True)
        rm, rv = torch.zeros(ch, device=dev), torch.ones(ch, device=dev)
        go = torch.randn_like(x)
        n = x.numel()
        state = {}

        def fwd():
            begin_step(dev)
            state["y"] = bn_act(x, w, b, rm, rv, residual=r, relu=relu, training=True, fused=True)

        work = torch.zeros(2 * ch, device=dev)

        def bwd():   # the two backward kernels only (autograd's grad accumulation would add passes of its own)
            fn = state["y"].grad_fn
            xs, mask, ws, saved = fn.saved_tensors
            work.zero_()
            C.bn_act_backward(go, xs, mask, ws, saved, relu, res, work)

        t_f = timeit(fwd)
        fwd()
        t_b = timeit(bwd)
        tag = "C=%d M=%d%s%s" % (ch, B * hw * hw, " relu" if relu else "", " +res" if res else "")
        row("bn_stats + bn_apply", tag, t_f, n * (2 + 2 + 2 + (2 if res else 0) + (0.125 if relu else 0)))
        row("bn_bwd_reduce + bn_bwd_apply", tag, t_b, n * (2 * (4 + (0.125 if relu else 0)) + 2 + (2 if (res and relu) else 0)))
        if res and hasattr(C, "bn_act_backward2"):     # split residual gradients (PTD_SPLIT_RESGRAD): the add moves into the reduce pass
            go2 = torch.randn_like(x)

            def bwd_add():
                xs, mask, ws, saved = state["y"].grad_fn.saved_tensors
                work.zero_()
                C.bn_act_backward(go + go2, xs, mask, ws, saved, relu, res, work)

            def bwd_split():
                xs, mask, ws, saved = state["y"].grad_fn.saved_tensors
                work.zero_()
                C.bn_act_backward2(go, go2, xs, mask, ws, saved, relu, work)

            mk = 0.125 if relu else 0
            row("ATen add + bn_bwd_reduce + bn_bwd_apply", tag, timeit(bwd_add), n * (6 + (4 + mk) + (4 + mk) + 4))
            row("bn_bwd_reduce_sum + bn_bwd_apply (split gradients)", tag, timeit(bwd_split), n * ((6 + mk) + 2 + 4 + 2))
        for p in (x, r, w, b):
            if p is not None:
                p.grad = None
    # stem
    x = torch.randn(B, 64, 112, 112, device=dev).bfloat16().contiguous(memory_format=torch.channels_last).requires_grad_(True)
    w = torch.ones(64, device=dev, dtype=torch.bfloat16, requires_grad=True)
    b = torch.zeros(64, device=dev, dtype=torch.bfloat16, requires_grad=True)
    rm, rv = torch.zeros(64, device=dev), torch.ones(64, device=dev)
    st = {}

    def sf():
        begin_step(dev)
        st["y"] = bn_relu_maxpool(x, w, b, rm, rv, training=True, fused=True)

    t_f = timeit(sf)
    sf()
    go = torch.randn_like(st["y"])
    swork = torch.zeros(128, device=dev)

    def sb():
        xs, code, ws, saved = st["y"].grad_fn.saved_tensors
        swork.zero_()
        C.stem_backward(go, xs, code, ws, saved, swork)

    t_b = timeit(sb)
    n, npool = x.numel(), st["y"].numel()
    row("bn_stats + stem_fwd (BN+ReLU+MaxPool)", "C=64 M=%d -> %d" % (B * 112 * 112, B * 56 * 56), t_f, n * 4 + npool * 2.5)
    row("stem_bwd_reduce + stem_bwd_apply", "same", t_b, n * 2 * 2 + 2 * npool * 2.5 + n * 2)
    # optimizer (ResNet-50 sized)
    nel = 25_600_000
    g = torch.randn(nel, device=dev).bfloat16()
    master, mom, copy = torch.randn(nel, device=dev), torch.zeros(nel, device=dev), torch.empty(nel, device=dev, dtype=torch.bfloat16)
    hyper = torch.tensor([0.1, 0.9, 1e-4, 0, 1, 0, 0, 0], device=dev)
    t = timeit(lambda: C.fused_sgd_flat(g, master, mom, copy, hyper, None, False, False))
    row("fused_sgd_flat (bf16 grad, fp32 master+momentum, bf16 copy)", "25.6 M params", t, nel * 20)
    # input pipeline
    img = torch.randn(B, 3, 224, 224, device=dev)
    a3, b3 = torch.ones(3, device=dev), torch.zeros(3, device=dev)
    t = timeit(lambda: C.normalize_nhwc(img, a3, b3, 1, True))
    row("normalize_nhwc (fp32 NCHW -> bf16 NHWC)", "256x3x224x224", t, img.numel() * 6)


if __name__ == "__main__":
    main()
