"""The workspace protocol of the fused BatchNorm autograd op and torch's BatchNorm semantics, on CPU through the PyTorch
emulation of the kernels (``fused="emulate"``), which adds its sums into the work slice it is given and computes from
what the slice then holds, as the kernels do.

- A second backward through a retained graph gets fresh zeros: the same bits as the first, not the sum of both.
- Non-reentrant checkpointing recomputes the forward: same gradient bits, running statistics advanced twice.
- A backward whose slice the next step recycled (``begin_step``), and a workspace too small for the step, give the bits
  of a lone run.
- ``momentum`` None (cumulative average), 0 and 1 follow ``torch.nn.BatchNorm2d`` over three steps.
- A second-order gradient through the op raises.
"""
import contextlib
import copy

import pytest
import torch
import torch.nn as nn
from torch.utils.checkpoint import checkpoint

import pytorch_distributed_b200.models.resnet as RN
from pytorch_distributed_b200.ops import bn_act as B

CPU = torch.device("cpu")


def _act(shape, dt, seed, offset=0.5):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * 2 + offset).to(dt).contiguous(memory_format=torch.channels_last)


def _leaves(c, seed=3):
    g = torch.Generator().manual_seed(seed)
    w = (torch.rand(c, generator=g) + 0.5).requires_grad_(True)
    b = (torch.randn(c, generator=g) * 0.2).requires_grad_(True)
    return w, b


def _bn_graph(relu, res, split, dt=torch.float32):
    """One emulated bn_act training forward; returns (scalar loss, leaves, running statistics)."""
    B.begin_step(CPU)
    c = 16
    x = _act((4, c, 5, 6), dt, 1).requires_grad_(True)
    r = _act((4, c, 5, 6), dt, 2, 0.0).requires_grad_(True) if res else None
    w, b = _leaves(c)
    rm, rv, nbt = torch.zeros(c), torch.ones(c), torch.zeros((), dtype=torch.long)
    y = B.bn_act(x, w, b, rm, rv, r, relu, True, 0.1, 1e-5, fused="emulate", num_batches_tracked=nbt, split=split)
    wts = torch.linspace(-1, 1, 4 * c * 30).view(4, 6, 5, c).permute(0, 3, 2, 1)
    if split:
        loss = (y[0].float() * wts).sin().sum() + (y[1].float() * 0.7).cos().sum()
    else:
        loss = (y.float() * wts).sin().sum()
    leaves = [x, w, b] + ([r] if res else [])
    return loss, leaves, (rm, rv, nbt)


@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("relu,res", [(True, True), (True, False), (False, True)])
@pytest.mark.parametrize("dt", [torch.float32, torch.bfloat16])
def test_retained_graph_bn_act(relu, res, split, dt):
    loss, leaves, _ = _bn_graph(relu, res, split, dt)
    g1 = torch.autograd.grad(loss, leaves, retain_graph=True)
    g2 = torch.autograd.grad(loss, leaves, retain_graph=True)
    for i, (a, b) in enumerate(zip(g1, g2)):
        assert torch.equal(a, b), "second autograd.grad differs from the first (leaf %d)" % i
    loss.backward(retain_graph=True)
    loss.backward()
    for i, (leaf, g) in enumerate(zip(leaves, g1)):
        assert torch.equal(leaf.grad, g + g), ".grad after two backwards is not twice one backward (leaf %d)" % i


def test_backward_slice_is_handed_out_once():
    ws = B._Workspace(CPU, capacity=4096)
    lw = ws.layer(64, None)
    first = lw.bwd()
    assert first.data_ptr() == ws.buf[128:].data_ptr()
    first.fill_(1.0)
    again = lw.bwd()
    assert again.numel() == 128 and not again.any() and again.data_ptr() != first.data_ptr()


def _bottleneck(seed=0):
    torch.manual_seed(seed)
    blk = RN.Bottleneck(32, 16, stride=2, downsample=RN._Downsample(32, 64, 2, "emulate"), fused="emulate")
    return blk.to(memory_format=torch.channels_last).train()


def _block_step(blk, x, fn=None, backward_twice=False):
    B.begin_step(CPU)
    xin = x.clone().requires_grad_(True)
    out = (fn or blk)(xin)
    ya, yb = RN._pair(out)
    loss = (ya * torch.linspace(-1, 1, ya.numel()).view_as(ya)).sum() + (yb * 0.5).cos().sum()
    if backward_twice:
        loss.backward(retain_graph=True)
    loss.backward()
    return [xin.grad] + [p.grad for p in blk.parameters()] + [b.clone() for b in blk.buffers()]


@contextlib.contextmanager
def _split(on):
    old = RN.SPLIT_RESGRAD
    RN.SPLIT_RESGRAD = on
    try:
        yield
    finally:
        RN.SPLIT_RESGRAD = old


@pytest.mark.parametrize("split", [False, True])
def test_retained_graph_bottleneck(split):
    x = _act((2, 32, 8, 8), torch.float32, 5)
    with _split(split):
        one = _block_step(_bottleneck(), x)
        two = _block_step(_bottleneck(), x, backward_twice=True)
    blk = _bottleneck()
    nparam = len(list(blk.parameters()))
    for i in range(1 + nparam):
        assert torch.equal(two[i], one[i] + one[i]), "gradient %d after two backwards" % i


@pytest.mark.parametrize("split", [False, True])
def test_checkpoint_bottleneck(split):
    """Non-reentrant checkpointing: the same gradient bits; the running statistics advance twice (the forward runs twice,
    as for nn.BatchNorm2d), to the bits of two plain forwards over the same batch."""
    x = _act((2, 32, 8, 8), torch.float32, 6)
    with _split(split):
        plain = _bottleneck()
        ref = _block_step(plain, x)
        ck = _bottleneck()
        got = _block_step(ck, x, fn=lambda t: checkpoint(ck, t, use_reentrant=False))
        twice = _bottleneck()
        with torch.no_grad():
            B.begin_step(CPU)
            twice(x)
            twice(x)
    nparam = len(list(plain.parameters()))
    for i in range(1 + nparam):
        assert torch.equal(got[i], ref[i]), "gradient %d under checkpoint" % i
    for (name, b), want in zip(ck.named_buffers(), twice.buffers()):
        assert torch.equal(b, want), name
        if name.endswith("num_batches_tracked"):
            assert int(b) == 2


def _small_resnet(seed=0):
    torch.manual_seed(seed)
    m = RN.ResNet(RN.Bottleneck, [1, 1, 1, 1], num_classes=10, fused_bn="emulate")
    return m.to(memory_format=torch.channels_last).train()


def _model_grads(m, out, y):
    nn.functional.cross_entropy(out, y).backward()
    return [p.grad.clone() for p in m.parameters()] + [b.clone() for b in m.buffers()]


def test_recycled_slices_two_models():
    """Two training forwards (the second recycles the first one's slices), then both backwards: each equals a lone run."""
    x = _act((2, 3, 32, 32), torch.float32, 7, 0.0)
    y = torch.tensor([1, 4])
    lone = [_model_grads(m, m(x), y) for m in (_small_resnet(0), _small_resnet(1))]
    ma, mb = _small_resnet(0), _small_resnet(1)
    oa = ma(x)
    ob = mb(x)
    got = [_model_grads(ma, oa, y), _model_grads(mb, ob, y)]
    for k in range(2):
        for i, (a, b) in enumerate(zip(got[k], lone[k])):
            assert torch.equal(a, b), "model %d tensor %d" % (k, i)


def test_workspace_overflow():
    """A workspace of 64 floats: every layer's ``take`` falls back to fresh zeros, with the bits of the normal run."""
    x = _act((2, 3, 32, 32), torch.float32, 8, 0.0)
    y = torch.tensor([3, 2])
    m = _small_resnet()
    ref = _model_grads(m, m(x), y)
    old = B._workspaces.get(CPU)
    B._workspaces[CPU] = B._Workspace(CPU, capacity=64)
    try:
        m = _small_resnet()
        got = _model_grads(m, m(x), y)
        assert B._workspaces[CPU].used == 0
    finally:
        if old is None:
            B._workspaces.pop(CPU, None)
        else:
            B._workspaces[CPU] = old
    for i, (a, b) in enumerate(zip(got, ref)):
        assert torch.equal(a, b), i


def _momentum_layers(momentum):
    """(name, layer under test, nn.BatchNorm2d in float64 with the same settings)."""
    from pytorch_distributed_b200.models.resnet import SyncBNAct, convert_sync_batchnorm
    from pytorch_distributed_b200.models.surgery import fuse_bn_relu
    out = [("BNAct", RN.BNAct(16, relu=False, momentum=momentum, fused="emulate")),
           ("SyncBNAct world 1", SyncBNAct(16, momentum=momentum, fused="emulate"))]
    out.append(("convert_sync_batchnorm", convert_sync_batchnorm(nn.BatchNorm2d(16, momentum=momentum))))
    seq = nn.Sequential(nn.BatchNorm2d(16, momentum=momentum), nn.ReLU())
    assert fuse_bn_relu(seq) == 1
    out.append(("surgery", seq))
    return out


@pytest.mark.parametrize("momentum", [None, 0.0, 1.0, 0.1])
def test_momentum_follows_batchnorm2d(momentum):
    for name, layer in _momentum_layers(momentum):
        ref = nn.BatchNorm2d(16, momentum=momentum).double()
        layer.train()
        for step in range(3):
            x = _act((3, 16, 5, 4), torch.float32, 20 + step, 0.3 * step)
            layer(x)
            ref(x.double())
        bn = layer[0] if isinstance(layer, nn.Sequential) else layer
        assert int(bn.num_batches_tracked) == 3, name
        for attr in ("running_mean", "running_var"):
            got, want = getattr(bn, attr), getattr(ref, attr)
            err = (got.double() - want).abs().max().item()
            assert err <= 1e-5 * max(1.0, want.abs().max().item()), "%s %s (momentum %s): |err| %.3g" % (name, attr, momentum, err)


def test_momentum_none_differs_from_default():
    """Negative control: momentum 0.1 does not pass for a cumulative-average reference."""
    layer = RN.BNAct(16, relu=False, momentum=0.1, fused="emulate").train()
    ref = nn.BatchNorm2d(16, momentum=None).double()
    for step in range(3):
        x = _act((3, 16, 5, 4), torch.float32, 20 + step, 0.3 * step)
        layer(x)
        ref(x.double())
    assert (layer.running_mean.double() - ref.running_mean).abs().max().item() > 1e-3


def test_second_order_gradient_raises():
    loss, leaves, _ = _bn_graph(True, True, False)
    gx = torch.autograd.grad(loss, leaves[0], create_graph=True)[0]
    with pytest.raises(RuntimeError, match="differentiate twice"):
        gx.sum().backward()
