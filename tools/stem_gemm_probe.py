"""Stem convolution: cuDNN (fprop / wgrad) vs im2col + wgmma GEMM (+BN statistics) + library wgrad, CUDA-event timings.

    PROBE_DTYPE=bf16|fp16 python tools/stem_gemm_probe.py [batch]   # on an H100; prints one markdown table; cuDNN runs
                                                                    # in the same dtype
"""
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pytorch_distributed_b200 import _ext                                        # noqa: E402
from pytorch_distributed_b200.ops.stem_conv import K_PAD, pack_stem_weight       # noqa: E402


def timed(fn, iters=20, warm=5):
    for _ in range(warm):
        fn()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    for a, b in ev:
        flush.zero_()                       # evict L2 between iterations
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    ts = sorted(a.elapsed_time(b) for a, b in ev)
    return ts[len(ts) // 2] * 1000.0


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 256
    C = _ext.lib()
    torch.backends.cudnn.benchmark = True
    dev = torch.device("cuda", 0)
    dt = {"bf16": torch.bfloat16, "fp16": torch.float16}[os.environ.get("PROBE_DTYPE", "bf16")]
    x = torch.randn(n, 3, 224, 224, device=dev).to(dt).contiguous(memory_format=torch.channels_last)
    w = (torch.randn(64, 3, 7, 7, device=dev) * 0.1).to(dt).contiguous(memory_format=torch.channels_last)
    y_ref = F.conv2d(x, w, stride=2, padding=3)
    dy = torch.randn_like(y_ref)
    stats = torch.zeros(128, device=dev)
    wp = pack_stem_weight(w)
    a = C.stem_im2col(x)
    y = C.conv1x1_bnstats(a, wp.view(64, K_PAD, 1, 1), stats)
    err = (y.float() - y_ref.float()).abs().max().item() / y_ref.float().abs().max().item()
    rows = a.permute(0, 2, 3, 1).reshape(-1, K_PAD)
    dy2 = dy.permute(0, 2, 3, 1).reshape(-1, 64)
    dw_ref = torch.ops.aten.convolution_backward(dy, x, w, None, (2, 2), (3, 3), (1, 1), False, (0, 0), 1, (False, True, False))[1]
    dwp = torch.mm(dy2.t(), rows, out_dtype=torch.float32)
    from pytorch_distributed_b200.ops.stem_conv import unpack_stem_weight
    werr = (unpack_stem_weight(dwp, w).float() - dw_ref.float()).abs().max().item() / dw_ref.float().abs().max().item()
    m = rows.size(0)
    gb_a = m * K_PAD * 2 / 1e9
    gb_y = m * 64 * 2 / 1e9
    print("%s, batch %d, M = %d, rel err y %.2e, dW %.2e" % (str(dt).replace("torch.", ""), n, m, err, werr))
    print("| step | us | GB moved | GB/s |")
    print("|---|---:|---:|---:|")
    t = timed(lambda: F.conv2d(x, w, stride=2, padding=3))
    print("| cuDNN fprop | %.0f | %.2f | %.0f |" % (t, gb_y + x.numel() * 2 / 1e9, (gb_y + x.numel() * 2 / 1e9) / t * 1e6))
    t = timed(lambda: torch.ops.aten.convolution_backward(dy, x, w, None, (2, 2), (3, 3), (1, 1), False, (0, 0), 1, (False, True, False)))
    print("| cuDNN wgrad | %.0f | %.2f | %.0f |" % (t, gb_y + x.numel() * 2 / 1e9, (gb_y + x.numel() * 2 / 1e9) / t * 1e6))
    t = timed(lambda: C.stem_im2col(x))
    print("| im2col kernel | %.0f | %.2f | %.0f |" % (t, gb_a + x.numel() * 2 / 1e9, (gb_a + x.numel() * 2 / 1e9) / t * 1e6))
    t = timed(lambda: C.conv1x1_bnstats(a, wp.view(64, K_PAD, 1, 1), stats))
    print("| wgmma GEMM K=192 N=64 + BN statistics | %.0f | %.2f | %.0f |" % (t, gb_a + gb_y, (gb_a + gb_y) / t * 1e6))
    t = timed(lambda: torch.mm(dy2.t(), rows, out_dtype=torch.float32))
    print("| library wgrad GEMM (dY^T x A), fp32 out | %.0f | %.2f | %.0f |" % (t, gb_a + gb_y, (gb_a + gb_y) / t * 1e6))
    t = timed(lambda: dy2.t() @ rows)
    print("| library wgrad GEMM (dY^T x A), 16-bit out | %.0f | %.2f | %.0f |" % (t, gb_a + gb_y, (gb_a + gb_y) / t * 1e6))
    t = timed(lambda: pack_stem_weight(w))
    print("| weight packing (ATen) | %.0f | | |" % t)


if __name__ == "__main__":
    main()
