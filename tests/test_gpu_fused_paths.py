"""GPU tests of the split-residual-gradient BN backward, the stem im2col + wgmma GEMM path and the static horovod schedule
(all three are the defaults).  Whole-model numerics are judged
against a plain PyTorch fp32 oracle on a shallow bottleneck ResNet (tests/_oracle.py)."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

pytestmark = [pytest.mark.gpu]


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float32, torch.float16])
@pytest.mark.parametrize("relu", [True, False])
@pytest.mark.parametrize("shape", [(8, 64, 56, 56), (4, 256, 14, 14), (3, 2048, 7, 7), (5, 72, 9, 11)])
def test_bn_backward2_matches_emulation(dt, relu, shape):
    from pytorch_distributed_b200 import _ext
    from pytorch_distributed_b200.ops.bn_act import _Emu
    C = _ext.lib()
    torch.manual_seed(0)
    dev = torch.device("cuda", 0)
    n, c, h, w = shape
    cl = torch.channels_last
    x = torch.randn(shape, device=dev).to(dt).contiguous(memory_format=cl)
    res = torch.randn(shape, device=dev).to(dt).contiguous(memory_format=cl)
    wt, bs = torch.rand(c, device=dev) + 0.5, torch.randn(c, device=dev)
    rm, rv = torch.zeros(c, device=dev), torch.ones(c, device=dev)
    work = torch.zeros(4 * c, device=dev)
    y, saved, mask = C.bn_act_forward(x, res, wt, bs, rm, rv, None, True, 0.1, 1e-5, relu, True, work[:2 * c], False)
    dya = torch.randn(shape, device=dev).to(dt).contiguous(memory_format=cl)
    dyb = torch.randn(shape, device=dev).to(dt).contiguous(memory_format=cl)
    dx, g, dw, db = C.bn_act_backward2(dya, dyb, x, mask, wt, saved, relu, work[2 * c:])
    ex, eg, ew, eb = _Emu.bn_act_backward2(dya, dyb, x, mask, wt, saved, relu, None)
    torch.cuda.synchronize()
    assert torch.equal(g, eg)                                      # the rounded, masked sum is bit-exact
    tol = 2e-2 if dt != torch.float32 else 1e-4
    scale = ex.float().abs().max().item()
    assert (dx.float() - ex.float()).abs().max().item() <= tol * scale
    assert torch.allclose(dw, ew, rtol=1e-3, atol=1e-2 * ew.abs().max().item())
    assert torch.allclose(db, eb, rtol=1e-3, atol=1e-2 * eb.abs().max().item())
    # and against the two-step path it replaces: eager add, then the validated single-gradient kernels
    work2 = torch.zeros(2 * c, device=dev)
    dx1, dres1, dw1, db1 = C.bn_act_backward(dya + dyb, x, mask, wt, saved, relu, True, work2)
    assert torch.equal(dres1 if relu else (dya + dyb), g)
    assert (dx.float() - dx1.float()).abs().max().item() <= tol * scale


def _bf16_model_and_batch(n=32, size=96, classes=64):
    from _oracle import small_resnet
    from pytorch_distributed_b200.parallel.amp import cast_model
    dev = torch.device("cuda", 0)
    base = cast_model(small_resnet(classes).to(dev).to(memory_format=torch.channels_last), torch.bfloat16)
    for p in base.parameters():                      # drop the fp32 stash: the oracle must see the bf16-rounded weights
        if hasattr(p, "_ptd_master_init"):
            del p._ptd_master_init
    torch.manual_seed(1)
    x = torch.randn(n, 3, size, size, device=dev).bfloat16().contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, classes, (n,), device=dev)
    return base, x, y


def _variant_vs_oracle(**flags):
    import copy
    from _oracle import compare, fp32_oracle, model_flags, step
    base, x, y = _bf16_model_and_batch()
    oracle = fp32_oracle(base, x, y)
    with model_flags(**{k: False for k in flags}):      # the path the flag replaces (cuDNN stem / autograd add)
        default = step(copy.deepcopy(base).train(), x, y)
    with model_flags(**flags):
        variant = step(copy.deepcopy(base).train(), x, y)
    torch.cuda.synchronize()
    assert all(torch.isfinite(g).all() for g in variant[1].values())
    bad = compare(variant, default, oracle)
    assert not bad, "error vs the fp32 oracle (name, variant, default path): %s" % (bad[:8],)


def test_split_residual_gradients_vs_fp32_oracle():
    """Whole (shallow) bottleneck ResNet step: SPLIT_RESGRAD vs the default path, both judged against plain fp32 PyTorch."""
    _variant_vs_oracle(SPLIT_RESGRAD=True)


def test_resnet50_full_depth_step_is_bitwise_reproducible():
    """Two identical full-depth ResNet-50 train steps through the split-gradient + stem-GEMM paths give the same bits:
    outputs, every gradient and every BN buffer.  The hand-written kernels add their per-CTA partial sums in a fixed
    order, and cuDNN is held to deterministic algorithms.  (Numerics are judged on the shallow model above.)"""
    import copy
    import pytorch_distributed_b200.models.resnet as R
    from pytorch_distributed_b200.models import create_model
    from pytorch_distributed_b200.ops.bn_act import begin_step
    from pytorch_distributed_b200.parallel.amp import cast_model
    torch.manual_seed(0)
    dev = torch.device("cuda", 0)
    m0 = cast_model(create_model("resnet50", num_classes=100).to(dev).to(memory_format=torch.channels_last), torch.bfloat16).train()
    x = torch.randn(16, 3, 96, 96, device=dev).bfloat16().contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 100, (16,), device=dev)
    flags = (torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark)
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    R.SPLIT_RESGRAD, R.STEM_GEMM = True, True
    runs = []
    try:
        for _ in range(2):
            m = copy.deepcopy(m0)
            begin_step(dev)
            out = m(x)
            torch.nn.functional.cross_entropy(out.float(), y).backward()
            runs.append((out.detach(), {n: p.grad for n, p in m.named_parameters()}, dict(m.named_buffers())))
    finally:
        R.SPLIT_RESGRAD, R.STEM_GEMM = False, False
        torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = flags
    torch.cuda.synchronize()
    (o1, g1, b1), (o2, g2, b2) = runs
    assert torch.isfinite(o1).all() and all(g is not None and torch.isfinite(g).all() for g in g1.values())
    assert torch.equal(o1, o2)
    assert [n for n in g1 if not torch.equal(g1[n], g2[n])] == []
    assert [n for n in b1 if not torch.equal(b1[n], b2[n])] == []


@pytest.mark.parametrize("shape", [(4, 3, 64, 64), (2, 3, 75, 91), (16, 3, 224, 224)])
def test_stem_im2col_kernel_matches_definition(shape):
    from pytorch_distributed_b200 import _ext
    from pytorch_distributed_b200.ops.stem_conv import im2col_reference
    torch.manual_seed(0)
    x = torch.randn(shape, device="cuda").bfloat16().contiguous(memory_format=torch.channels_last)
    a = _ext.lib().stem_im2col(x)
    ref = im2col_reference(x)
    assert a.shape == ref.shape and a.is_contiguous(memory_format=torch.channels_last)
    assert torch.equal(a, ref)


def test_stem_gemm_path_matches_cudnn_path():
    """conv7x7 + BN + ReLU + MaxPool: im2col + wgmma GEMM (+ statistics) + stem_forward_pre vs cuDNN conv + fused stem tail."""
    import copy
    import torch.nn as nn
    from pytorch_distributed_b200.models.resnet import BNAct
    from pytorch_distributed_b200.ops.bn_act import begin_step
    from pytorch_distributed_b200.ops.stem import bn_relu_maxpool
    from pytorch_distributed_b200.ops.stem_conv import can_use_stem_gemm, stem_conv_bn_relu_maxpool
    torch.manual_seed(0)
    dev = torch.device("cuda", 0)
    conv = nn.Conv2d(3, 64, 7, stride=2, padding=3, bias=False).to(dev).bfloat16().to(memory_format=torch.channels_last)
    bn = BNAct(64).to(dev).train()
    x = torch.randn(32, 3, 224, 224, device=dev).bfloat16().contiguous(memory_format=torch.channels_last)
    assert can_use_stem_gemm(x, conv)
    res = []
    for mode in ("cudnn", "gemm"):
        c, b = copy.deepcopy(conv), copy.deepcopy(bn)
        begin_step(dev)
        if mode == "gemm":
            y = stem_conv_bn_relu_maxpool(x, c, b)
        else:
            y = bn_relu_maxpool(c(x), b.weight, b.bias, b.running_mean, b.running_var, training=True, momentum=0.1, eps=b.eps,
                                num_batches_tracked=b.num_batches_tracked)
        (y.float() * torch.linspace(-1, 1, y.numel(), device=dev).view_as(y)).sum().backward()
        res.append((y.float(), c.weight.grad.float(), b.weight.grad.float(), b.bias.grad.float(), b.running_mean.clone(), b.running_var.clone()))
    torch.cuda.synchronize()
    names = ("y", "dW", "dgamma", "dbeta", "running_mean", "running_var")
    for n, a, e in zip(names, res[1], res[0]):
        err = (a - e).abs().max().item() / (e.abs().max().item() + 1e-6)
        assert err < 3e-2, (n, err)


def test_stem_gemm_vs_fp32_oracle():
    _variant_vs_oracle(STEM_GEMM=True)


def test_split_and_stem_gemm_vs_fp32_oracle():
    _variant_vs_oracle(STEM_GEMM=True, SPLIT_RESGRAD=True)


@pytest.mark.parametrize("graph", [False, True])
def test_horovod_entrypoint_static_schedule(tmp_path, graph):
    """PTD_HVD_STATIC=1: the fusion groups are frozen after the first step and launched from the hooks (optionally inside a CUDA graph);
    the loss trajectory must match the dynamic (queue + dispatcher thread) run of the same seed."""
    import re
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    n = min(torch.cuda.device_count(), 2)
    base = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(n), "--master-addr", "127.0.0.1"]
    args = ["-a", "resnet18", "-b", str(16 * n), "--synthetic", "--steps-per-epoch", "8", "--val-steps", "1", "--epochs", "1", "--image-size", "64",
            "-p", "1", "--lr", "0.01", "--seed", "3", "--checkpoint-dir", str(tmp_path)]
    losses = {}
    for static, port in (("0", "29851"), ("1", "29852")):
        env = dict(os.environ, PTD_HVD_STATIC=static)
        for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "MASTER_ADDR", "MASTER_PORT"):
            env.pop(k, None)
        cmd = base + ["--master-port", port, os.path.join(root, "horovod_distributed.py")] + args + (["--cuda-graph"] if graph and static == "1" else [])
        p = subprocess.run(cmd, env=env, cwd=root, capture_output=True, text=True, timeout=900)
        assert p.returncode == 0, p.stdout[-3000:] + "\n" + p.stderr[-5000:]
        losses[static] = [float(x) for x in re.findall(r"Loss (\d\.\d+e[+-]\d+)", p.stdout)]
    assert len(losses["1"]) == len(losses["0"]) > 0
    assert all(abs(a - b) <= 0.05 * max(1.0, abs(a)) for a, b in zip(losses["0"], losses["1"])), (losses["0"][:8], losses["1"][:8])
