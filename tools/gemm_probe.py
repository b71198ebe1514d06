"""Correctness + speed of the wgmma 1x1-conv GEMM with fused BN statistics against cuDNN conv + bn_stats.

    PROBE_B=256 PROBE_DTYPE=bf16|fp16 python tools/gemm_probe.py       # on an H100; cuDNN runs in the same dtype
"""
import sys, os
import torch
import torch.nn.functional as F
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pytorch_distributed_b200 import _ext
C = _ext.lib()
torch.backends.cudnn.benchmark = True
B = int(os.environ.get("PROBE_B", "256"))
DT = {"bf16": torch.bfloat16, "fp16": torch.float16}[os.environ.get("PROBE_DTYPE", "bf16")]
shapes = [(64, 64, 56), (64, 256, 56), (256, 64, 56), (256, 128, 56), (128, 512, 28), (512, 128, 28), (512, 256, 28), (256, 1024, 14),
          (1024, 256, 14), (1024, 512, 14), (512, 2048, 7), (2048, 512, 7)]
if len(sys.argv) > 1 and sys.argv[1] == "small":
    shapes, B = [(64, 64, 8), (128, 256, 5), (64, 128, 3)], 4


def t(fn, n=10):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n * 1e3


tot = [0.0, 0.0, 0.0]
for cin, cout, hw in shapes:
    torch.manual_seed(0)
    x = torch.randn(B, cin, hw, hw, device="cuda").to(DT).contiguous(memory_format=torch.channels_last)
    w = (torch.randn(cout, cin, 1, 1, device="cuda") * 0.1).to(DT).contiguous(memory_format=torch.channels_last)
    gs = torch.zeros(2 * cout, device="cuda")
    y = C.conv1x1_bnstats(x, w, gs)
    torch.cuda.synchronize()
    ref = F.conv2d(x.float(), w.float())
    err = (y.float() - ref).abs().max().item() / max(1e-6, ref.abs().max().item())
    s_ref = ref.sum(dim=(0, 2, 3)); q_ref = (ref * ref).sum(dim=(0, 2, 3))
    es = (gs[:cout] - s_ref).abs().max().item() / max(1.0, s_ref.abs().max().item())
    eq = (gs[cout:] - q_ref).abs().max().item() / max(1.0, q_ref.abs().max().item())
    ok = err < 1e-2 and es < 1e-2 and eq < 1e-2
    line = "cin=%4d cout=%4d hw=%2d M=%7d  rel err y %.1e sum %.1e sumsq %.1e %s" % (cin, cout, hw, B * hw * hw, err, es, eq, "OK" if ok else "MISMATCH")
    if len(shapes) > 3:
        t_mine = t(lambda: C.conv1x1_bnstats(x, w, gs))
        t_conv = t(lambda: F.conv2d(x, w))
        work = torch.zeros(2 * cout, device="cuda")
        wt, bt = torch.ones(cout, device="cuda", dtype=DT), torch.zeros(cout, device="cuda", dtype=DT)
        yc = F.conv2d(x, w)
        from pytorch_distributed_b200.ops.bn_act import bn_act, begin_step
        def both():
            yy = F.conv2d(x, w)
            C.bn_act_forward(yy, None, wt, bt, torch.zeros(cout, device="cuda"), torch.ones(cout, device="cuda"), None, True, 0.1, 1e-5, True, False, work, False)
        t_both = t(both)
        tot[0] += t_mine; tot[1] += t_conv; tot[2] += t_both
        line += " | gemm+stats %.1f us, cudnn conv %.1f us, cudnn conv + bn_stats + bn_apply %.1f us" % (t_mine, t_conv, t_both)
    print(line, flush=True)
if len(shapes) > 3:
    print("%s, batch %d" % (str(DT).replace("torch.", ""), B))
    print("sum: gemm+stats %.1f us | cudnn conv %.1f us | conv+stats+apply %.1f us" % tuple(tot))
