"""Times the backward of every ResNet-50 1x1 conv -> BatchNorm pair at batch 256 after the BN reduction pass: the fused
data-gradient GEMM (``gemm_bnbwd_dgrad_kernel``: dx formed in shared memory, dIn = dx W) against ``bn_bwd_apply`` followed
by cuDNN's dgrad.  Reports the bytes each path has to move, GB/s and the share of 3.35 TB/s (H100 SXM HBM3 data sheet).

    python tools/dgrad_probe.py            # bf16;  PROBE_DTYPE=fp16 for fp16
"""
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

# (C_in, C_out, H, ReLU on the BN) of the stride-1 pairs: bn1 of every block, bn3 (split, no mask), layer1's downsample
PAIRS = [(64, 64, 56, True), (256, 64, 56, True), (64, 256, 56, False), (256, 128, 56, True), (512, 128, 28, True),
         (128, 512, 28, False), (512, 256, 28, True), (1024, 256, 14, True), (256, 1024, 14, False), (1024, 512, 14, True),
         (2048, 512, 7, True), (512, 2048, 7, False)]
HBM = 3.35e12


def timed(fn, iters=20):
    for _ in range(3):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters * 1e-3


def main():
    from pytorch_distributed_b200 import _ext
    C = _ext.lib()
    dt = torch.float16 if os.environ.get("PROBE_DTYPE") == "fp16" else torch.bfloat16
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print("card: %s   dtype: %s   batch 256" % (q, dt))
    print("| C_in -> C_out, HxW | relu | fused us | GB/s | of 3.35 TB/s | apply + cuDNN dgrad us | GB/s | of 3.35 TB/s | saved us |")
    print("|---|---|---:|---:|---:|---:|---:|---:|---:|")
    cl = torch.channels_last
    tot_f = tot_u = 0.0
    for cin, cout, h, relu in PAIRS:
        n = 256
        m = n * h * h
        y = torch.randn((n, cout, h, h), device="cuda").to(dt).contiguous(memory_format=cl)
        g = torch.randn_like(y)
        bw, bb = torch.rand(cout, device="cuda") + 0.5, torch.randn(cout, device="cuda")
        rm, rv = torch.zeros(cout, device="cuda"), torch.ones(cout, device="cuda")
        _, saved, mask = C.bn_act_forward(y, None, bw, bb, rm, rv, None, True, 0.1, 1e-5, relu, True, torch.zeros(2 * cout, device="cuda"), False)
        cw = (torch.randn((cout, cin, 1, 1), device="cuda") / cin ** 0.5).to(dt)
        xin = torch.empty((n, cin, h, h), device="cuda", dtype=dt).contiguous(memory_format=cl)
        work = torch.zeros(2 * cout, device="cuda")
        mk = mask if relu else None
        # both paths run the same reduction pass first: time the whole backward and subtract nothing (the reduce is shared)
        fused = timed(lambda: C.conv1x1_bn_backward(g, None, y, mk, bw, saved, cw, relu, work.zero_()))

        def unfused():
            dx = C.bn_act_backward(g, y, mk, bw, saved, relu, False, work.zero_())[0]
            torch.ops.aten.convolution_backward(dx, xin, cw, None, (1, 1), (0, 0), (1, 1), False, (0, 0), 1, (True, False, False))
        unf = timed(unfused)
        e = 2                                        # bytes per element
        mbytes = m * cout // 8 if relu else 0
        red = m * cout * e * 2 + mbytes              # reduction pass: g, y (+ mask)
        b_f = red + m * cout * e * 3 + mbytes + m * cin * e          # + GEMM: read g, y (+ mask), write dx and dIn
        b_u = red + m * cout * e * 3 + mbytes + m * cout * e + m * cin * e   # + apply: g, y -> dx; dgrad: dx -> dIn
        tot_f += fused
        tot_u += unf
        print("| %d -> %d, %dx%d | %s | %.1f | %.0f | %.2f | %.1f | %.0f | %.2f | %.1f |" % (
            cin, cout, h, h, "yes" if relu else "no", fused * 1e6, b_f / fused / 1e9, b_f / fused / HBM, unf * 1e6, b_u / unf / 1e9,
            b_u / unf / HBM, (unf - fused) * 1e6))
    print("sum over the 12 shapes (reduction pass included in both): fused %.1f us, apply + cuDNN dgrad %.1f us" % (tot_f * 1e6, tot_u * 1e6))


if __name__ == "__main__":
    main()
