"""The backward of a 1x1 conv -> BatchNorm pair through ``conv1x1_bn_backward``: the BN reduction pass, then the wgmma
data-gradient GEMM that applies the BN backward to its A operand (``csrc/gemm_bnstats.cu``).  Its dx must be the bits
of ``bn_bwd_apply``, its data gradient is judged against float64, and the autograd op against the two-op backward."""
import pytest
import torch

pytestmark = [pytest.mark.gpu]

CL = torch.channels_last
# (C_in, C_out, H) of every ResNet-50 1x1 conv -> BN pair at stride 1, and (64, 128, 9 x 11) for an M tail (5 * 99 rows)
PAIRS = [(64, 64, 56), (256, 64, 56), (64, 256, 56), (256, 128, 56), (512, 128, 28), (128, 512, 28), (512, 256, 28),
         (1024, 256, 14), (256, 1024, 14), (1024, 512, 14), (2048, 512, 7), (512, 2048, 7)]


def _lib():
    from pytorch_distributed_b200 import _ext
    return _ext.lib()


def _pair_inputs(cin, cout, h, w, n, dt, relu, seed=0):
    """A BN forward over a random conv output y: (y, mask, bn weight, saved, conv weight, incoming gradients)."""
    C = _lib()
    g = torch.Generator(device="cuda").manual_seed(seed)
    dev = torch.device("cuda", 0)
    y = torch.randn((n, cout, h, w), device=dev, generator=g).mul_(2).add_(0.5).to(dt).contiguous(memory_format=CL)
    bw = torch.rand(cout, device=dev, generator=g) + 0.5
    bb = torch.randn(cout, device=dev, generator=g)
    rm, rv = torch.zeros(cout, device=dev), torch.ones(cout, device=dev)
    _, saved, mask = C.bn_act_forward(y, None, bw, bb, rm, rv, None, True, 0.1, 1e-5, relu, True, torch.zeros(2 * cout, device=dev), False)
    cw = (torch.randn((cout, cin, 1, 1), device=dev, generator=g) / cin ** 0.5).to(dt)
    dya = torch.randn(y.shape, device=dev, generator=g).to(dt).contiguous(memory_format=CL)
    dyb = torch.randn(y.shape, device=dev, generator=g).to(dt).contiguous(memory_format=CL)
    return y, mask, bw, saved, cw, dya, dyb


def _dgrad_bound(dx, cw, dt):
    """|dIn - dx @ W| bound: rounding the result to dt, plus fp32 accumulation of K exact products."""
    k = cw.size(0)
    dxd = dx.permute(0, 2, 3, 1).reshape(-1, k).double()
    wd = cw.reshape(k, -1).double()
    ref = dxd @ wd
    mag = dxd.abs() @ wd.abs()
    u = 2.0 ** -8 if dt == torch.bfloat16 else 2.0 ** -11
    return ref, u * ref.abs() + 2 * k * 2.0 ** -24 * mag + 1e-30


def _rows(t):
    return t.permute(0, 2, 3, 1).reshape(-1, t.size(1)).double()


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("relu", [True, False])
@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("pair", PAIRS + [(64, 128, (9, 11))])
def test_fused_dx_is_bn_bwd_apply_bits_and_dgrad_within_fp64_bound(pair, split, relu, dt):
    C = _lib()
    cin, cout, hw = pair
    h, w = hw if isinstance(hw, tuple) else (hw, hw)
    n = 5 if isinstance(hw, tuple) else max(2, 12544 * 2 // (h * w))
    y, mask, bw, saved, cw, dya, dyb = _pair_inputs(cin, cout, h, w, n, dt, relu)
    work = torch.zeros(2 * cout, device="cuda")
    din, dx, g, dgamma, dbeta = C.conv1x1_bn_backward(dya, dyb if split else None, y, mask if relu else None, bw, saved, cw, relu, work)
    work_ref = torch.zeros(2 * cout, device="cuda")
    if split:
        rdx, rg, rdw, rdb = C.bn_act_backward2(dya, dyb, y, mask, bw, saved, relu, work_ref)
        assert torch.equal(g, rg)
    else:
        rdx, _, rdw, rdb = C.bn_act_backward(dya, y, mask, bw, saved, relu, False, work_ref)
        assert g is None
    torch.cuda.synchronize()
    assert torch.equal(dx, rdx)
    assert torch.equal(dgamma, rdw) and torch.equal(dbeta, rdb)
    assert din.is_contiguous(memory_format=CL) and din.shape == (n, cin, h, w)
    ref, bound = _dgrad_bound(dx, cw, dt)
    assert bool(((_rows(din) - ref).abs() <= bound).all())
    # the same bound holds for cuDNN's data gradient of the same dx
    cud = torch.ops.aten.convolution_backward(dx, torch.empty((n, cin, h, w), device="cuda", dtype=dt).contiguous(memory_format=CL), cw,
                                              None, (1, 1), (0, 0), (1, 1), False, (0, 0), 1, (True, False, False))[0]
    assert bool(((_rows(cud) - ref).abs() <= bound).all())


def test_fused_backward_is_reproducible_and_graph_replay_matches_eager():
    C = _lib()
    y, mask, bw, saved, cw, dya, dyb = _pair_inputs(1024, 512, 14, 14, 32, torch.bfloat16, True, seed=3)

    def run():
        return C.conv1x1_bn_backward(dya, dyb, y, mask, bw, saved, cw, True, torch.zeros(1024, device="cuda"))

    a, b = run(), run()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        run()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        c = run()
    graph.replay()
    torch.cuda.synchronize()
    for x, y_, z in zip(a, b, c):
        if x is not None:
            assert torch.equal(x, y_) and torch.equal(x, z)


def _block(cin, cout, relu, dt, seed):
    from pytorch_distributed_b200.models.resnet import BNAct
    torch.manual_seed(seed)
    conv = torch.nn.Conv2d(cin, cout, 1, bias=False).cuda().to(dt).to(memory_format=CL)
    bn = BNAct(cout, relu=relu).cuda().train()
    with torch.no_grad():
        bn.weight.uniform_(0.5, 1.5)
        bn.bias.normal_()
    return conv, bn


def _step(monkeypatch, fused, cin, cout, n, hw, dt, relu, residual, split, seed=0):
    """One forward + backward of conv1x1_bn_act; returns the gradients and how often the fused op was applied."""
    from pytorch_distributed_b200.ops import conv_bn
    monkeypatch.setattr(conv_bn, "FUSED_DGRAD", fused)
    calls = []
    orig = conv_bn._Conv1x1BnFn.apply
    monkeypatch.setattr(conv_bn._Conv1x1BnFn, "apply", lambda *a: calls.append(1) or orig(*a))
    conv, bn = _block(cin, cout, relu, dt, seed)
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    x = torch.randn((n, cin, hw, hw), device="cuda", generator=g).to(dt).contiguous(memory_format=CL).requires_grad_()
    res = None
    if residual:
        res = torch.randn((n, cout, hw, hw), device="cuda", generator=g).to(dt).contiguous(memory_format=CL).requires_grad_()
    out = conv_bn.conv1x1_bn_act(x, conv, bn, res, split=split)
    seeds = [torch.randn(o.shape, device="cuda", generator=g).to(dt) for o in (out if isinstance(out, tuple) else (out,))]
    torch.autograd.backward(list(out) if isinstance(out, tuple) else [out], seeds)
    torch.cuda.synchronize()
    grads = dict(x=x.grad, w=conv.weight.grad, gamma=bn.weight.grad, beta=bn.bias.grad, res=None if res is None else res.grad)
    return grads, len(calls), (x, conv.weight)


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("case", ["bn1", "bn3_split", "downsample"])
def test_autograd_matches_two_op_backward(monkeypatch, case, dt):
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    monkeypatch.setattr(torch.backends.cudnn, "benchmark", False)
    relu = case != "downsample"
    residual = split = case == "bn3_split"
    cin, cout = (256, 64) if case == "bn1" else (64, 256)
    new, n_new, (x, w) = _step(monkeypatch, True, cin, cout, 8, 28, dt, relu, residual, split)
    old, n_old, _ = _step(monkeypatch, False, cin, cout, 8, 28, dt, relu, residual, split)
    assert n_new == 1 and n_old == 0
    for k in ("w", "gamma", "beta", "res"):
        assert (new[k] is None and old[k] is None) or torch.equal(new[k], old[k]), k
    # the conv input's gradient comes from a different GEMM (judged against float64 in the kernel test above): here the two
    # paths agree within two output roundings
    assert new["x"].shape == old["x"].shape
    diff = (new["x"].double() - old["x"].double()).abs()
    u = 2.0 ** -8 if dt == torch.bfloat16 else 2.0 ** -11
    assert bool((diff <= 2 * u * old["x"].double().abs() + 1e-3 * old["x"].double().abs().max()).all())


@pytest.mark.parametrize("case", ["disabled", "residual_without_split", "fp32", "odd_channels", "wide_input"])
def test_fallbacks_keep_the_two_op_backward(monkeypatch, case):
    fused, dt, cin, cout, residual, split = True, torch.bfloat16, 64, 256, False, False
    if case == "disabled":
        fused = False
    elif case == "residual_without_split":
        residual = True
    elif case == "fp32":
        dt = torch.float32
    elif case == "odd_channels":
        cin = 72
    else:
        cin = 512
    _, n, _ = _step(monkeypatch, fused, cin, cout, 4, 14, dt, True, residual, split)
    assert n == 0


def test_synchronised_bn_keeps_the_two_op_backward(monkeypatch):
    from pytorch_distributed_b200.ops import conv_bn

    class _Sync:                      # a world > 1 context: the pair must not take the one-rank fused backward
        native = object()
    conv, bn = _block(64, 256, True, torch.bfloat16, 0)
    monkeypatch.setattr(bn, "sync_context", lambda: _Sync())
    calls = []
    monkeypatch.setattr(conv_bn._Conv1x1BnFn, "apply", lambda *a: calls.append(1))
    monkeypatch.setattr(conv_bn._Conv1x1Stats, "apply", lambda *a: (_ for _ in ()).throw(RuntimeError("two-op path")))
    x = torch.randn((4, 64, 14, 14), device="cuda").to(torch.bfloat16).contiguous(memory_format=CL).requires_grad_()
    with pytest.raises(RuntimeError, match="two-op path"):
        conv_bn.conv1x1_bn_act(x, conv, bn)
    assert not calls
