"""The fused BatchNorm, 1x1-conv and stem autograd ops (``ops/``) and their workspace protocol, on the GPU.

Part a: each op equals the extension entry points it documents, called in order with freshly zeroed work slices, bit
for bit, at ResNet-50 batch-256 shapes, in a bf16-cast, an fp16-cast and bf16 / fp16 autocast (fp32 parameters) setting:
outputs, every input gradient, dgamma / dbeta, the conv weight gradient, the running statistics and
``num_batches_tracked``.  The parts that are not ours (cuDNN's 1x1 dgrad and wgrad, the stem weight-gradient GEMM) are
checked against float64 with the bound K u sum|a||b| plus half an output ulp (tests/_fp64.py); under autocast the fp32
parameter gradient is the 16-bit gradient upcast exactly.

Part b: torch's semantics for what the workspace must survive.  A second backward through a retained graph gives the
bits of the first (``.grad`` after two backwards is exactly twice one); non-reentrant checkpointing gives the same
gradient bits and advances the running statistics twice; a backward whose slices the next step recycled, a workspace
too small for the step and CUDA-graph replays give the bits of a lone eager run; ``momentum`` None / 0 / 1 follows
``nn.BatchNorm2d``; a second-order gradient raises.
"""
import contextlib
import copy
import os
import sys

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _fp64 as R  # noqa: E402

import pytorch_distributed_b200.models.resnet as RN  # noqa: E402
from pytorch_distributed_b200.ops import bn_act as B  # noqa: E402

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
CL = torch.channels_last
EPS, MOM = 1e-5, 0.1
BF16, F16, F32 = torch.bfloat16, torch.float16, torch.float32
# activation dtype, parameter dtype, autocast dtype
MODES = {"bf16": (BF16, BF16, None), "fp16": (F16, F16, None), "bf16-autocast": (BF16, F32, BF16), "fp16-autocast": (F16, F32, F16)}


def lib():
    from pytorch_distributed_b200 import _ext
    return _ext.lib()


@pytest.fixture(autouse=True)
def _deterministic():
    old = torch.backends.cudnn.deterministic
    torch.backends.cudnn.deterministic = True
    try:
        yield
    finally:
        torch.backends.cudnn.deterministic = old


def act(shape, dt, seed, offset=0.5):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(shape, device=DEV, generator=g) * 2 + offset).to(dt).contiguous(memory_format=CL)


def grad_like(t, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randint(-8, 9, t.shape, device=DEV, generator=g) / 8).to(t.dtype).contiguous(memory_format=CL)


def params(c, dt, seed=7):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.rand(c, device=DEV, generator=g) + 0.5).to(dt), (torch.randn(c, device=DEV, generator=g) * 0.2).to(dt)


def stats(c):
    return torch.zeros(c, device=DEV), torch.ones(c, device=DEV), torch.zeros((), dtype=torch.int64, device=DEV)


def autocast(ac):
    return torch.autocast("cuda", dtype=ac) if ac is not None else contextlib.nullcontext()


def cast(module, dt):
    """``module`` on the GPU in ``dt``; BatchNorm running statistics stay fp32, as the kernels require."""
    module = module.to(DEV, dt)
    for m in module.modules():
        if isinstance(m, nn.BatchNorm2d):
            m.running_mean.data, m.running_var.data = m.running_mean.float(), m.running_var.float()
    return module


def same(name, got, want):
    assert got is not None and want is not None, name + ": missing"
    assert got.dtype == want.dtype and got.shape == want.shape, "%s: %s %s vs %s %s" % (name, got.dtype, tuple(got.shape),
                                                                                       want.dtype, tuple(want.shape))
    if not torch.equal(got, want):
        d = (got.double() - want.double()).abs()
        raise AssertionError("%s: %d elements differ, max |diff| %.3g" % (name, int((d != 0).sum()), d.max().item()))


def check_mm(name, got, a, b, out_dt):
    """got ~ a @ b (fp32 accumulation of K products of 16-bit values, exact in fp32), within K u sum|a||b| + half an ulp
    of the stored result."""
    ad, bd = a.double(), b.double()
    ref = ad @ bd
    mag = ad.abs() @ bd.abs()
    del ad, bd
    R.assert_within(name, got, ref, 0.5 * R.ulp(got, out_dt) + a.size(1) * R.U32 * mag)


# ====================================================================================================== a. bitwise
BN_CASES = [(256, 1024, 14, relu, res, split) for relu in (True, False) for res in (True, False) for split in (False, True)] + \
           [(256, 256, 56, True, True, True), (256, 2048, 7, True, True, False)]


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("n,c,hw,relu,res,split", BN_CASES, ids=["%dx%d@%d-relu%d-res%d-split%d" % (n, c, hw, a, b_, s)
                                                                  for n, c, hw, a, b_, s in BN_CASES])
def test_bn_act_equals_entry_points(mode, n, c, hw, relu, res, split):
    adt, pdt, _ = MODES[mode]
    M = lib()
    x = act((n, c, hw, hw), adt, 1)
    r = act((n, c, hw, hw), adt, 2, 0.0) if res else None
    w, b = params(c, pdt)
    dy, dy2 = grad_like(x, 3), grad_like(x, 4)

    B.begin_step(DEV)
    xx = x.clone().requires_grad_(True)
    rr = r.clone().requires_grad_(True) if res else None
    ww, bb = w.clone().requires_grad_(True), b.clone().requires_grad_(True)
    rm, rv, nb = stats(c)
    out = B.bn_act(xx, ww, bb, rm, rv, rr, relu, True, MOM, EPS, num_batches_tracked=nb, split=split)
    if split:
        torch.autograd.backward(list(out), [dy, dy2])
        out = out[0]
    else:
        out.backward(dy)

    rm2, rv2, nb2 = stats(c)
    y, saved, mask = M.bn_act_forward(x, r, w, b, rm2, rv2, nb2, True, MOM, EPS, relu, True, torch.zeros(2 * c, device=DEV), False)
    mask = mask if relu else None
    wb = torch.zeros(2 * c, device=DEV)
    if split:
        dx, dres, dw, db = M.bn_act_backward2(dy, dy2, x, mask, w, saved, relu, wb)
    else:
        dx, dres, dw, db = M.bn_act_backward(dy, x, mask, w, saved, relu, res, wb)
    same("y", out.detach(), y)
    same("dx", xx.grad, dx)
    if res:
        same("d residual", rr.grad, dres)
    same("dgamma", ww.grad, dw)
    same("dbeta", bb.grad, db)
    same("running_mean", rm, rm2)
    same("running_var", rv, rv2)
    assert int(nb) == 1 and int(nb2) == 1


CONV_CASES = [(256, 256, 64, 56, False, False), (256, 1024, 256, 14, False, False), (256, 256, 1024, 14, True, True),
              (256, 512, 2048, 7, True, False)]


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("n,k,co,hw,res,split", CONV_CASES, ids=["%dx%d-%d@%d-res%d-split%d" % s for s in CONV_CASES])
def test_conv1x1_bn_act_equals_entry_points(mode, n, k, co, hw, res, split):
    from pytorch_distributed_b200.ops.conv_bn import conv1x1_bn_act
    adt, pdt, ac = MODES[mode]
    M = lib()
    x = act((n, k, hw, hw), adt, 11, 0.0)
    r = act((n, co, hw, hw), adt, 12, 0.0) if res else None
    conv = nn.Conv2d(k, co, 1, bias=False).to(DEV, pdt).to(memory_format=CL)
    bn = cast(RN.BNAct(co, relu=True), pdt if ac is None else F32)
    with torch.no_grad():
        bn.weight.copy_(params(co, bn.weight.dtype)[0])
        bn.bias.copy_(params(co, bn.weight.dtype)[1])
    dyshape = (n, co, hw, hw)
    dy, dy2 = grad_like(act(dyshape, adt, 0), 13), grad_like(act(dyshape, adt, 0), 14)
    w0, b0 = bn.weight.detach().clone(), bn.bias.detach().clone()
    rm, rv, nb = bn.running_mean.clone(), bn.running_var.clone(), bn.num_batches_tracked.clone()

    B.begin_step(DEV)
    xx = x.clone().requires_grad_(True)
    rr = r.clone().requires_grad_(True) if res else None
    with autocast(ac):
        out = conv1x1_bn_act(xx, conv, bn, rr, split=split)
    if split:
        torch.autograd.backward(list(out), [dy, dy2])
        out = out[0]
    else:
        out.backward(dy)

    wg = conv.weight.detach().to(adt)
    gs = torch.zeros(2 * co, device=DEV)
    z = M.conv1x1_bnstats(x, wg, gs)
    y, saved, mask = M.bn_act_forward(z, r, w0, b0, rm, rv, nb, True, MOM, EPS, True, True, gs, True)
    wb = torch.zeros(2 * co, device=DEV)
    if split:
        dz, dres, dgam, dbet = M.bn_act_backward2(dy, dy2, z, mask, w0, saved, True, wb)
    else:
        dz, dres, dgam, dbet = M.bn_act_backward(dy, z, mask, w0, saved, True, res, wb)
    dx, dwc, _ = torch.ops.aten.convolution_backward(dz, x, wg, None, (1, 1), (0, 0), (1, 1), False, (0, 0), 1, (True, True, False))
    same("y", out.detach(), y)
    same("dx", xx.grad, dx)
    if res:
        same("d residual", rr.grad, dres)
    same("dgamma", bn.weight.grad, dgam)
    same("dbeta", bn.bias.grad, dbet)
    same("conv weight grad", conv.weight.grad, dwc.to(conv.weight.dtype))     # autocast: the bf16 / fp16 gradient upcast exactly
    same("running_mean", bn.running_mean, rm)
    same("running_var", bn.running_var, rv)
    assert int(bn.num_batches_tracked) == 1 and int(nb) == 1
    # cuDNN's dgrad and wgrad against float64 from the same 16-bit operands
    dzr, xr = R.rows(dz), R.rows(x)
    check_mm("dgrad", R.rows(dx), dzr, wg.view(co, k), adt)
    check_mm("wgrad", dwc.view(co, k), dzr.t(), xr, adt)


@pytest.mark.parametrize("mode", list(MODES))
def test_bn_relu_maxpool_equals_entry_points(mode):
    from pytorch_distributed_b200.ops.stem import bn_relu_maxpool
    adt, pdt, _ = MODES[mode]
    M = lib()
    c = 64
    x = act((256, c, 112, 112), adt, 21)
    w, b = params(c, pdt)
    dp = grad_like(torch.empty(256, c, 56, 56, dtype=adt, device=DEV), 22)
    B.begin_step(DEV)
    xx = x.clone().requires_grad_(True)
    ww, bb = w.clone().requires_grad_(True), b.clone().requires_grad_(True)
    rm, rv, nb = stats(c)
    y = bn_relu_maxpool(xx, ww, bb, rm, rv, training=True, momentum=MOM, eps=EPS, num_batches_tracked=nb)
    y.backward(dp)
    rm2, rv2, nb2 = stats(c)
    y2, saved, code = M.stem_forward(x, w, b, rm2, rv2, nb2, True, MOM, EPS, True, torch.zeros(2 * c, device=DEV))
    dx, dw, db = M.stem_backward(dp, x, code, w, saved, torch.zeros(2 * c, device=DEV))
    for name, g_, w_ in (("y", y.detach(), y2), ("dx", xx.grad, dx), ("dgamma", ww.grad, dw), ("dbeta", bb.grad, db),
                         ("running_mean", rm, rm2), ("running_var", rv, rv2)):
        same(name, g_, w_)
    assert int(nb) == 1 and int(nb2) == 1


@pytest.mark.parametrize("mode", list(MODES))
def test_stem_conv_bn_relu_maxpool_equals_entry_points(mode):
    from pytorch_distributed_b200.ops.stem_conv import K_PAD, pack_stem_weight, stem_conv_bn_relu_maxpool, unpack_stem_weight
    adt, pdt, ac = MODES[mode]
    M = lib()
    img = act((256, 3, 224, 224), adt if ac is None else F32, 31, 0.0)
    torch.manual_seed(0)
    conv = nn.Conv2d(3, 64, 7, 2, 3, bias=False).to(DEV, pdt)
    bn = cast(RN.BNAct(64, relu=True), pdt if ac is None else F32)
    with torch.no_grad():
        bn.weight.copy_(params(64, bn.weight.dtype)[0])
        bn.bias.copy_(params(64, bn.weight.dtype)[1])
    w0, b0 = bn.weight.detach().clone(), bn.bias.detach().clone()
    rm, rv, nb = bn.running_mean.clone(), bn.running_var.clone(), bn.num_batches_tracked.clone()
    dp = grad_like(torch.empty(256, 64, 56, 56, dtype=adt, device=DEV), 32)
    B.begin_step(DEV)
    with autocast(ac):
        y = stem_conv_bn_relu_maxpool(img, conv, bn)
    y.backward(dp)

    x16 = img.to(adt)
    wg = conv.weight.detach().to(adt)
    a = M.stem_im2col(x16)
    gs = torch.zeros(128, device=DEV)
    z = M.conv1x1_bnstats(a, pack_stem_weight(wg).view(64, K_PAD, 1, 1), gs)
    y2, saved, code = M.stem_forward_pre(z, w0, b0, rm, rv, nb, True, MOM, EPS, True, gs)
    dz, dgam, dbet = M.stem_backward(dp, z, code, w0, saved, torch.zeros(128, device=DEV))
    dzr, ar = R.rows(dz), a.permute(0, 2, 3, 1).reshape(-1, K_PAD)
    dwp = torch.mm(dzr.t(), ar, out_dtype=torch.float32)
    same("y", y.detach(), y2)
    same("dgamma", bn.weight.grad, dgam)
    same("dbeta", bn.bias.grad, dbet)
    same("conv weight grad", conv.weight.grad, unpack_stem_weight(dwp, wg).to(conv.weight.dtype))
    same("running_mean", bn.running_mean, rm)
    same("running_var", bn.running_var, rv)
    assert int(bn.num_batches_tracked) == 1
    check_mm("stem wgrad", dwp, dzr.t(), ar, F32)
    # the parameter gradient itself (GEMM, unpack, store) against the 7x7 convolution's weight gradient in float64 from the
    # same 16-bit image and BatchNorm input gradient: K = N * OH * OW products per element, then one rounding to 16 bits
    xd, dzd = x16.double(), dz.double()
    ref = torch.nn.grad.conv2d_weight(xd, tuple(conv.weight.shape), dzd, stride=2, padding=3)
    mag = torch.nn.grad.conv2d_weight(xd.abs(), tuple(conv.weight.shape), dzd.abs(), stride=2, padding=3)
    del xd, dzd
    got = conv.weight.grad
    R.assert_within("stem weight grad", got, ref, 0.5 * R.ulp(got, adt) + (dz.numel() // 64) * R.U32 * mag)


# ====================================================================================================== b. workspace protocol
def _op_graph(op, dt=BF16):
    """(loss, leaves) of one training forward of ``op`` at a small shape; the loss weights both aliases of a split."""
    from pytorch_distributed_b200.ops.conv_bn import conv1x1_bn_act
    from pytorch_distributed_b200.ops.stem import bn_relu_maxpool
    from pytorch_distributed_b200.ops.stem_conv import stem_conv_bn_relu_maxpool
    B.begin_step(DEV)
    torch.manual_seed(0)
    if op == "bn_act":
        x = act((8, 256, 14, 14), dt, 41).requires_grad_(True)
        r = act((8, 256, 14, 14), dt, 42, 0.0).requires_grad_(True)
        w, b = (t.requires_grad_(True) for t in params(256, F32))
        rm, rv, nb = stats(256)
        out = B.bn_act(x, w, b, rm, rv, r, True, True, MOM, EPS, num_batches_tracked=nb, split=True)
        leaves = [x, r, w, b]
    elif op == "conv1x1_bn_act":
        x = act((8, 256, 28, 28), dt, 43, 0.0).requires_grad_(True)
        r = act((8, 128, 28, 28), dt, 44, 0.0).requires_grad_(True)
        conv = nn.Conv2d(256, 128, 1, bias=False).to(DEV, dt).to(memory_format=CL)
        bn = RN.BNAct(128).to(DEV)
        out = conv1x1_bn_act(x, conv, bn, r, split=True)
        leaves = [x, r, conv.weight, bn.weight, bn.bias]
    elif op == "bn_relu_maxpool":
        x = act((8, 64, 56, 56), dt, 45).requires_grad_(True)
        w, b = (t.requires_grad_(True) for t in params(64, F32))
        rm, rv, nb = stats(64)
        out = bn_relu_maxpool(x, w, b, rm, rv, training=True, num_batches_tracked=nb)
        leaves = [x, w, b]
    else:
        x = act((8, 3, 64, 64), dt, 46, 0.0)
        conv = nn.Conv2d(3, 64, 7, 2, 3, bias=False).to(DEV, dt)
        bn = RN.BNAct(64).to(DEV)
        out = stem_conv_bn_relu_maxpool(x, conv, bn)
        leaves = [conv.weight, bn.weight, bn.bias]
    outs = out if isinstance(out, tuple) else (out,)
    loss = sum(((o.float() * (0.5 + 0.25 * i)).sin() * torch.linspace(-1, 1, o.numel(), device=DEV).view_as(o)).sum()
               for i, o in enumerate(outs))
    return loss, leaves


OPS = ["bn_act", "conv1x1_bn_act", "bn_relu_maxpool", "stem_conv_bn_relu_maxpool"]


@pytest.mark.parametrize("op", OPS)
def test_retained_graph_op(op):
    loss, leaves = _op_graph(op)
    g1 = torch.autograd.grad(loss, leaves, retain_graph=True)
    g2 = torch.autograd.grad(loss, leaves, retain_graph=True)
    for i, (a, b) in enumerate(zip(g1, g2)):
        same("%s second autograd.grad, leaf %d" % (op, i), b, a)
    loss.backward(retain_graph=True)
    loss.backward()
    for i, (leaf, g) in enumerate(zip(leaves, g1)):
        same("%s .grad after two backwards, leaf %d" % (op, i), leaf.grad, g + g)


@pytest.mark.parametrize("op", OPS)
def test_second_order_gradient_raises(op):
    loss, leaves = _op_graph(op)
    g = torch.autograd.grad(loss, leaves[0], create_graph=True)[0]
    with pytest.raises(RuntimeError, match="differentiate twice"):
        g.float().sum().backward()


def _bottleneck(mode="bf16", seed=0):
    adt, pdt, ac = MODES[mode]
    torch.manual_seed(seed)
    blk = RN.Bottleneck(256, 128, stride=1, downsample=RN._Downsample(256, 512, 1, None))
    return cast(blk, pdt).to(memory_format=CL).train()


def _block_loss(out):
    ya, yb = RN._pair(out)
    return ((ya.float() * torch.linspace(-1, 1, ya.numel(), device=DEV).view_as(ya)).sum()
            + (yb.float() * 0.5).cos().sum())


def _block_step(blk, x, fn=None, twice=False, ac=None):
    B.begin_step(DEV)
    xin = x.clone().requires_grad_(True)
    with autocast(ac):
        out = (fn or blk)(xin)
    loss = _block_loss(out)
    if twice:
        loss.backward(retain_graph=True)
    loss.backward()
    return [xin.grad] + [p.grad for p in blk.parameters()], [b.clone() for b in blk.buffers()]


@pytest.mark.parametrize("mode", ["bf16", "bf16-autocast"])
def test_retained_graph_bottleneck(mode):
    ac = MODES[mode][2]
    x = act((16, 256, 28, 28), MODES[mode][0], 50)
    one, _ = _block_step(_bottleneck(mode), x, ac=ac)
    two, _ = _block_step(_bottleneck(mode), x, twice=True, ac=ac)
    for i, (a, b) in enumerate(zip(two, one)):
        same("gradient %d after two backwards" % i, a, b + b)


@pytest.mark.parametrize("mode", ["bf16", "bf16-autocast"])
def test_checkpoint_bottleneck(mode):
    from torch.utils.checkpoint import checkpoint
    ac = MODES[mode][2]
    x = act((16, 256, 28, 28), MODES[mode][0], 51)
    ref, _ = _block_step(_bottleneck(mode), x, ac=ac)
    ck = _bottleneck(mode)
    got, bufs = _block_step(ck, x, fn=lambda t: checkpoint(ck, t, use_reentrant=False), ac=ac)
    for i, (a, b) in enumerate(zip(got, ref)):
        same("gradient %d under checkpoint" % i, a, b)
    twice = _bottleneck(mode)
    B.begin_step(DEV)
    with autocast(ac):
        twice(x.clone().requires_grad_(True))
        twice(x.clone().requires_grad_(True))
    for (name, b), want in zip(ck.named_buffers(), twice.buffers()):
        same("checkpointed " + name, b, want)
    assert int(ck.bn1.num_batches_tracked) == 2


def _small_resnet(seed):
    torch.manual_seed(seed)
    m = RN.ResNet(RN.Bottleneck, [1, 1, 1, 1], num_classes=10)
    return cast(m, BF16).to(memory_format=CL).train()


def _model_grads(m, out, y):
    F.cross_entropy(out.float(), y).backward()
    return [out.detach()] + [p.grad for p in m.parameters()] + [b.clone() for b in m.buffers()]


def _images():
    return act((8, 3, 64, 64), BF16, 60, 0.0), torch.tensor([1, 4, 2, 7, 0, 9, 3, 3], device=DEV)


def test_recycled_slices_two_models():
    x, y = _images()
    lone = [_model_grads(m, m(x), y) for m in (_small_resnet(0), _small_resnet(1))]
    ma, mb = _small_resnet(0), _small_resnet(1)
    oa = ma(x)
    ob = mb(x)                  # recycles the slices of ma's step
    got = [_model_grads(ma, oa, y), _model_grads(mb, ob, y)]
    for k in range(2):
        for i, (a, b) in enumerate(zip(got[k], lone[k])):
            same("model %d tensor %d" % (k, i), a, b)


def test_workspace_overflow():
    x, y = _images()
    m = _small_resnet(0)
    ref = _model_grads(m, m(x), y)
    old = B._workspaces.get(DEV)
    B._workspaces[DEV] = B._Workspace(DEV, capacity=64)
    try:
        m = _small_resnet(0)
        got = _model_grads(m, m(x), y)
        assert B._workspaces[DEV].used == 0
    finally:
        B._workspaces[DEV] = old
    for i, (a, b) in enumerate(zip(got, ref)):
        same("tensor %d" % i, a, b)


def test_cuda_graph_replay_of_a_block():
    """Capture begin_step, a Bottleneck's forward and its backward; three replays with new inputs equal eager steps."""
    blk = _bottleneck("bf16")
    params_ = list(blk.parameters())
    static_x = act((16, 256, 28, 28), BF16, 70).requires_grad_(True)

    def step():
        B.begin_step(DEV)
        out = blk(static_x)
        return (RN._pair(out)[0],) + torch.autograd.grad(_block_loss(out), [static_x] + params_)

    state0 = copy.deepcopy(blk.state_dict())
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()                                       # warm-up on a side stream, as torch.cuda.graphs requires
    torch.cuda.current_stream().wait_stream(s)
    blk.load_state_dict(state0)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = step()
    blk.load_state_dict(state0)                      # capture ran no kernels: the running statistics are still state0
    for k in range(3):
        x = act((16, 256, 28, 28), BF16, 71 + k)
        before = copy.deepcopy(blk.state_dict())
        with torch.no_grad():
            static_x.copy_(x)
        graph.replay()
        torch.cuda.synchronize()
        got = [t.clone() for t in outs]
        got_state = copy.deepcopy(blk.state_dict())
        eager = _bottleneck("bf16")
        eager.load_state_dict(before)
        B.begin_step(DEV)
        xe = x.clone().requires_grad_(True)
        out = eager(xe)
        want = (RN._pair(out)[0],) + torch.autograd.grad(_block_loss(out), [xe] + list(eager.parameters()))
        for i, (a, b) in enumerate(zip(got, want)):
            same("replay %d tensor %d" % (k, i), a, b.detach())
        for name, t in eager.state_dict().items():
            same("replay %d %s" % (k, name), got_state[name], t)
    del graph


def _momentum_layers(momentum):
    from pytorch_distributed_b200.models.resnet import SyncBNAct, convert_sync_batchnorm
    from pytorch_distributed_b200.models.surgery import fuse_bn_relu
    seq = nn.Sequential(nn.BatchNorm2d(64, momentum=momentum), nn.ReLU())
    assert fuse_bn_relu(seq) == 1
    return [("BNAct", RN.BNAct(64, relu=False, momentum=momentum)), ("SyncBNAct world 1", SyncBNAct(64, momentum=momentum)),
            ("convert_sync_batchnorm", convert_sync_batchnorm(nn.BatchNorm2d(64, momentum=momentum))), ("surgery", seq)]


@pytest.mark.parametrize("momentum", [None, 0.0, 1.0])
def test_momentum_follows_batchnorm2d(momentum):
    for name, layer in _momentum_layers(momentum):
        layer = layer.to(DEV).train()
        bn = layer[0] if isinstance(layer, nn.Sequential) else layer
        ref = nn.BatchNorm2d(64, momentum=momentum).to(DEV, torch.float64)
        for step in range(3):
            x = act((8, 64, 14, 14), BF16, 80 + step, 0.3 * step).requires_grad_(True)
            layer(x)
            ref(x.detach().double())
        assert int(bn.num_batches_tracked) == 3, name
        for attr in ("running_mean", "running_var"):
            got, want = getattr(bn, attr).double(), getattr(ref, attr)
            err = (got - want).abs().max().item()
            assert err <= 1e-4 * max(1.0, want.abs().max().item()), "%s %s (momentum %s): |err| %.3g" % (name, attr, momentum, err)


def test_momentum_none_resnet_stem_and_blocks():
    """A ResNet whose layers have momentum=None (as after copying torchvision modules) trains with the cumulative average
    on every BatchNorm: after two different batches the stem's and a block's running statistics are the mean of the two
    batches' statistics (factors 1, then 1/2), which a constant factor (0.1 or 1) does not give."""
    m = _small_resnet(0)
    for mod in m.modules():
        if isinstance(mod, nn.BatchNorm2d):
            mod.momentum = None
    seen = {"stem": [], "layer2.0.bn2": []}
    h1 = m.conv1.register_forward_hook(lambda mod, a, out: seen["stem"].append(out.detach().double()))
    h2 = m.layer2[0].bn2.register_forward_pre_hook(lambda mod, a: seen["layer2.0.bn2"].append(a[0].detach().double()))
    x, y = _images()
    try:
        for k in range(2):
            F.cross_entropy(m((x * (1 + k) + 0.5 * k).to(x.dtype)).float(), y).backward()
    finally:
        h1.remove()
        h2.remove()
    for name, bn in (("stem", m.bn1), ("layer2.0.bn2", m.layer2[0].bn2)):
        assert len(seen[name]) == 2 and int(bn.num_batches_tracked) == 2, name
        ref = nn.BatchNorm2d(bn.num_features, momentum=None).to(DEV, torch.float64)
        with torch.no_grad():
            for z in seen[name]:
                ref(z)
        for attr in ("running_mean", "running_var"):
            got, want = getattr(bn, attr).double(), getattr(ref, attr)
            err = (got - want).abs().max().item()
            assert err <= 1e-4 * max(1.0, want.abs().max().item()), "%s %s: |err| %.3g" % (name, attr, err)


# ====================================================================================================== c. full-depth ResNet-50
# One training step of ResNet-50 (batch 64 at 224, FUSED_CONV1X1, STEM_GEMM and SPLIT_RESGRAD on) is recorded block by
# block: each block's input(s) (the two aliases a split producer hands out), running statistics before the step, output
# and the gradient(s) that arrived at its output aliases, and after backward its parameter gradients and statistics.
# Each block is then re-run from those recordings in float64 (reference) and through the unfused path in the step's
# precision (baseline: cuDNN + F.batch_norm, autograd adds), so depth cannot amplify anything and a wiring error (wrong
# alias, residual, slice or ReLU flag) is an O(1) error in one named block.  Criterion: relative Frobenius error against
# float64 <= max(2 x the baseline's, 4u), per tensor, and per channel for BatchNorm and conv weight gradients.
C_MODES = {"bf16": (BF16, BF16, None), "fp16": (F16, F16, None), "bf16-autocast": (BF16, F32, BF16)}
UNIT = {BF16: 2.0 ** -8, F16: 2.0 ** -11}
BLOCKS = ["stem"] + ["layer%d.%d" % (i + 1, j) for i, n in enumerate((3, 4, 6, 3)) for j in range(n)]
LOSS_SCALE = 1024.0             # static loss scale, as amp uses for fp16: keeps the deep gradients out of fp16's subnormals
_STEPS = {}


def _snap(mod, prefix=""):
    return {prefix + k: v.detach().clone() for k, v in mod.named_buffers()}


def _resnet50_step(mode):
    """(model, {block name: record}) of one fused training step; cached per mode."""
    if mode in _STEPS:
        return _STEPS[mode]
    from pytorch_distributed_b200.models import create_model
    from pytorch_distributed_b200.parallel.amp import cast_model
    adt, _, ac = C_MODES[mode]
    assert RN.FUSED_CONV1X1 and RN.STEM_GEMM and RN.SPLIT_RESGRAD
    torch.manual_seed(0)
    m = create_model("resnet50", num_classes=1000).to(DEV).to(memory_format=CL)
    if ac is None:
        cast_model(m, adt, keep_batchnorm_fp32=True)
    m.train()
    g = torch.Generator(device=DEV).manual_seed(1)
    img = torch.randn(64, 3, 224, 224, device=DEV, generator=g).to(adt if ac is None else F32).contiguous(memory_format=CL)
    target = torch.randint(0, 1000, (64,), device=DEV, generator=g)
    mods = dict(m.named_modules())
    recs = {name: {} for name in BLOCKS}
    recs["stem"].update(before=_snap(m.bn1, "bn1."), image=img)

    def grab(store, i):
        def h(grad):                 # None: no gradient reached this alias
            store[i] = None if grad is None else grad.detach().clone()
        return h

    def pre(mod, args, rec):
        xs = args[0] if isinstance(args[0], tuple) else (args[0],)
        rec.update(before=_snap(mod), inputs=[t.detach().clone() for t in xs], gin=[None] * len(xs))
        for i, t in enumerate(xs):
            t.register_hook(grab(rec["gin"], i))

    def post(mod, args, out, rec):
        outs = out if isinstance(out, tuple) else (out,)
        rec.update(out=outs[0].detach().clone(), gout=[None] * len(outs))
        for i, t in enumerate(outs):
            t.register_hook(grab(rec["gout"], i))

    hooks = []
    for name in BLOCKS[1:]:
        hooks.append(mods[name].register_forward_pre_hook(lambda mod, a, rec=recs[name]: pre(mod, a, rec)))
        hooks.append(mods[name].register_forward_hook(lambda mod, a, o, rec=recs[name]: post(mod, a, o, rec)))
    try:
        B.begin_step(DEV)
        with autocast(ac):
            out = m(img)
        (F.cross_entropy(out.float(), target) * LOSS_SCALE).backward()
    finally:
        for h in hooks:
            h.remove()
    for name in BLOCKS[1:]:
        recs[name].update(pgrads={k: p.grad.detach().clone() for k, p in mods[name].named_parameters()}, after=_snap(mods[name]))
    first = recs["layer1.0"]
    recs["stem"].update(out=first["inputs"][0], gout=[first["gin"][0]], gin=[],
                        pgrads={"conv1.weight": m.conv1.weight.grad.clone(), "bn1.weight": m.bn1.weight.grad.clone(),
                                "bn1.bias": m.bn1.bias.grad.clone()}, after=_snap(m.bn1, "bn1."))
    _STEPS[mode] = (m, recs)
    return _STEPS[mode]


def _unfused(mod, before, strip=""):
    c = copy.deepcopy(mod)
    for x in c.modules():
        if isinstance(x, RN.BNAct):
            x.fused = False
    with torch.no_grad():
        for k, v in c.named_buffers():
            v.copy_(before[strip + k])
    return c


def _eval_block(name, mode, ref):
    """The block re-run from its recordings: float64 (``ref``) or the unfused path in the step's precision."""
    from _oracle import model_flags
    m, recs = _resnet50_step(mode)
    rec = recs[name]
    adt, _, ac = C_MODES[mode]
    gs = [t for t in rec["gout"] if t is not None]
    up = sum(t.double() for t in gs) if ref else (gs[0] if len(gs) == 1 else gs[0] + gs[1])
    ctx = contextlib.nullcontext() if ref else autocast(ac)
    with model_flags(FUSED_CONV1X1=False, SPLIT_RESGRAD=False, STEM_GEMM=False):
        if name == "stem":
            conv, bn = copy.deepcopy(m.conv1), _unfused(m.bn1, rec["before"], "bn1.")
            img = rec["image"]
            if ref:                                    # the 16-bit values the step multiplied (autocast casts them too)
                conv.weight.data = conv.weight.data.to(adt).double()
                bn, img = bn.double(), img.to(adt).double()
            with ctx:
                y = F.max_pool2d(bn(conv(img)), 3, 2, 1)
            names = ["conv1.weight", "bn1.weight", "bn1.bias"]
            grads = torch.autograd.grad(y, [conv.weight, bn.weight, bn.bias], up.to(y.dtype))
            return dict(out=y.detach(), gin=[], pgrads=dict(zip(names, grads)), after=_snap(bn, "bn1."))
        blk = _unfused(dict(m.named_modules())[name], rec["before"])
        xs = [t.double() if ref else t for t in rec["inputs"]]
        if ref:
            for mod in blk.modules():
                if isinstance(mod, nn.Conv2d):
                    mod.weight.data = mod.weight.data.to(adt)
            blk = blk.double()
        leaves = [xs[0].clone().requires_grad_(True), xs[-1].clone().requires_grad_(True)]    # main, skip
        with ctx:
            y = blk((leaves[0], leaves[1]))
        names = [k for k, _ in blk.named_parameters()]
        grads = torch.autograd.grad(y, leaves + [p for _, p in blk.named_parameters()], up.to(y.dtype))
        gin = list(grads[:2]) if len(xs) == 2 else [grads[0].double() + grads[1].double()]
        return dict(out=y.detach(), gin=gin, pgrads=dict(zip(names, grads[2:])), after=_snap(blk))


def channel_bound(base, ref, u):
    """Per-channel (first dimension) error bound, in units of the channel's scale s = max(|ref channel|, |ref| / sqrt(C)):
    max(2 x the baseline's largest scaled channel error, 4u) x s, and at least twice the baseline's own error in that
    channel.  Channel errors are heavy-tailed (a channel whose sums cancel has a large error on every path), so one
    path's channel is held to the other path's worst channel, not to the same channel's error, which is often small by
    chance; a wrong channel (an O(1) error) stands far above either."""
    r = ref.double().reshape(ref.size(0), -1)
    b = base.double().reshape(ref.size(0), -1)
    s = torch.clamp_min(r.norm(dim=1), (r.norm() / r.size(0) ** 0.5).item()).clamp_min(1e-300)
    eb = (b - r).norm(dim=1)
    worst = (eb / s).max().item()
    return torch.maximum(2 * eb, max(2 * worst, 4 * u) * s)


def check_tensor(label, got, base, ref, u, per_channel=False):
    """Relative Frobenius error of ``got`` against float64 <= max(2 x the baseline's, 4u); returns got's / baseline's."""
    ref = ref.double()
    rn = ref.norm().clamp_min(1e-300)
    ef = ((got.double() - ref).norm() / rn).item()
    eb = ((base.double() - ref).norm() / rn).item()
    if ef > max(2 * eb, 4 * u):
        raise AssertionError("%s: relative error %.3g > max(2 x baseline %.3g, 4u = %.3g)" % (label, ef, eb, 4 * u))
    if per_channel:
        bound = channel_bound(base, ref, u)
        err = (got.double() - ref).reshape(ref.size(0), -1).norm(dim=1)
        bad = err > bound
        if bad.any():
            c = int((err / bound).argmax())
            raise AssertionError("%s: %d channels outside their bound; channel %d: error %.3g > %.3g"
                                 % (label, int(bad.sum()), c, err[c].item(), bound[c].item()))
    return ef / max(eb, 1e-30)


def check_block(name, rec, base, ref, u):
    """All of one block's checks; returns the largest fused / baseline error ratio."""
    ratios = [check_tensor(name + " output", rec["out"], base["out"], ref["out"], u)]
    labels = ["main input", "skip input"] if len(rec["gin"]) == 2 else ["input (main + skip)"] * len(rec["gin"])
    for i, lab in enumerate(labels):
        ratios.append(check_tensor("%s gradient into the %s" % (name, lab), rec["gin"][i], base["gin"][i], ref["gin"][i], u))
    for k in ref["pgrads"]:
        ratios.append(check_tensor("%s %s gradient" % (name, k), rec["pgrads"][k], base["pgrads"][k], ref["pgrads"][k], u, True))
    for k in ref["after"]:
        if k.endswith("num_batches_tracked"):
            assert int(rec["after"][k]) == int(rec["before"][k]) + 1, "%s %s: %d -> %d" % (name, k, int(rec["before"][k]),
                                                                                          int(rec["after"][k]))
        else:
            ratios.append(check_tensor("%s %s" % (name, k), rec["after"][k], base["after"][k], ref["after"][k], u))
    return max(ratios)


@pytest.mark.parametrize("block", BLOCKS)
@pytest.mark.parametrize("mode", list(C_MODES))
def test_resnet50_block_against_fp64(mode, block):
    _, recs = _resnet50_step(mode)
    rec = recs[block]
    assert rec["gout"][0] is not None, "no gradient reached the block's output"
    if block == "layer4.2":
        assert rec["gout"][1] is None          # the last block's second alias has no consumer
    elif block not in ("stem",):
        assert len(rec["gout"]) == 2 and rec["gout"][1] is not None, "split output expected"
    ratio = check_block(block, rec, _eval_block(block, mode, False), _eval_block(block, mode, True), UNIT[C_MODES[mode][0]])
    print("resnet50 %s %s: largest fused/baseline error ratio %.3f" % (mode, block, ratio))


def _mutated(rec):
    out = dict(rec)
    for k in ("gin", "pgrads", "after"):
        out[k] = copy.copy(rec[k])
    return out


def test_resnet50_block_checker_rejects_wiring_errors():
    mode, name = "bf16", "layer2.1"
    _, recs = _resnet50_step(mode)
    rec, u = recs[name], UNIT[BF16]
    base, ref = _eval_block(name, mode, False), _eval_block(name, mode, True)
    check_block(name, rec, base, ref, u)
    bad = _mutated(rec)                                        # the two alias gradients swapped
    bad["gin"] = [rec["gin"][1], rec["gin"][0]]
    with pytest.raises(AssertionError, match="gradient into the"):
        check_block(name, bad, base, ref, u)
    bad = _mutated(rec)                                        # one dgamma channel off by 4x its bound
    k = "bn2.weight"
    bound = channel_bound(base["pgrads"][k], ref["pgrads"][k], u)
    g = rec["pgrads"][k].clone()
    g[5] += (4 * bound[5]).to(g.dtype)
    bad["pgrads"][k] = g
    with pytest.raises(AssertionError, match="bn2.weight"):
        check_block(name, bad, base, ref, u)
    bad = _mutated(rec)                                        # one dbeta doubled
    bad["pgrads"]["bn1.bias"] = rec["pgrads"]["bn1.bias"] * 2
    with pytest.raises(AssertionError, match="bn1.bias"):
        check_block(name, bad, base, ref, u)
    bad = _mutated(rec)                                        # num_batches_tracked bumped twice
    bad["after"]["bn3.num_batches_tracked"] = rec["after"]["bn3.num_batches_tracked"] + 1
    with pytest.raises(AssertionError, match="num_batches_tracked"):
        check_block(name, bad, base, ref, u)


def test_stem_conv_momentum_none_takes_the_unfused_batchnorm():
    from pytorch_distributed_b200.ops.stem_conv import stem_conv_bn_relu_maxpool
    torch.manual_seed(0)
    conv = nn.Conv2d(3, 64, 7, 2, 3, bias=False).to(DEV, BF16)
    bn = RN.BNAct(64, momentum=None).to(DEV).train()
    ref = nn.BatchNorm2d(64, momentum=None).to(DEV, torch.float64)
    for k in range(2):
        x = act((4, 3, 64, 64), BF16, 90 + k, 0.3 * k)
        stem_conv_bn_relu_maxpool(x, conv, bn)
        with torch.no_grad():
            ref(F.conv2d(x, conv.weight, stride=2, padding=3).double())
    assert int(bn.num_batches_tracked) == 2
    for attr in ("running_mean", "running_var"):
        got, want = getattr(bn, attr).double(), getattr(ref, attr)
        assert (got - want).abs().max().item() <= 1e-4 * max(1.0, want.abs().max().item()), attr
