"""FusedSGD resume on the GPU keeps the fp32 momentum (and masters) exactly, whichever way the optimizer meets its engine:
bound to a flat arena before the state is loaded (DDP order), bound after it (apex order: amp.initialize, then apex DDP,
then the first step binds), or never bound (multi-tensor mode)."""
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda"
CL = torch.channels_last


def _build(entry, argv):
    from pytorch_distributed_b200 import cli, driver
    from pytorch_distributed_b200.models import create_model
    torch.cuda.set_device(0)
    args = cli.parse_args(entry, ["-a", "resnet50", "-b", "8", "--synthetic", "--image-size", "64", "--quiet"] + argv)
    st = driver.STRATEGIES[entry]()
    torch.manual_seed(0)
    model = create_model(args.arch, num_classes=args.num_classes, fused_bn=args.fused_bn)
    model, opt = st.build(model, args, torch.device(DEV, 0), 0)
    model.train()
    return st, model, opt


def _step(st, model, opt, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(8, 3, 64, 64, device=DEV, generator=g).to(st.input_dtype).contiguous(memory_format=CL)
    y = torch.randint(0, 1000, (8,), device=DEV, generator=g)
    opt.zero_grad()
    loss = torch.nn.functional.cross_entropy(st.forward(model, x).float(), y)
    st.backward(loss, opt)
    opt.step()
    torch.cuda.synchronize()


@pytest.mark.parametrize("entry,argv", [("distributed", ["--no-overlap-optimizer"]), ("apex_distributed", ["--opt-level", "O2", "--precision", "bf16"])],
                         ids=["bound_before_load", "bound_after_load"])
def test_flat_resume_keeps_fp32_momentum(entry, argv):
    st, model, opt = _build(entry, argv)
    for i in range(2):
        _step(st, model, opt, i)
    assert opt.is_flat and opt._flat.model_copy is not None          # low-precision model, fp32 momentum
    sd = copy.deepcopy(opt.state_dict())
    want = opt._flat.momentum.clone()
    st2, model2, opt2 = _build(entry, argv)
    opt2.load_state_dict(sd)
    if not opt2.is_flat:
        opt2._try_bind()                                               # what its first step does
    assert opt2.is_flat
    got = opt2._flat.momentum
    own = torch.zeros_like(want, dtype=torch.bool)
    for i, p in enumerate(opt2._flat.engine.params):
        o = opt2._flat.engine.param_elem_off[i]
        own[o:o + p.numel()] = True
    assert torch.equal(got[own], want[own])
    assert not torch.equal(want[own], want[own].bfloat16().float())   # bf16 rounding would have been visible


def test_multi_tensor_resume_keeps_fp32_state():
    from pytorch_distributed_b200.ops.fused_sgd import FusedSGD
    torch.manual_seed(0)
    ps = [torch.nn.Parameter(torch.randn(256, 128, device=DEV).bfloat16()) for _ in range(3)]
    opt = FusedSGD(ps, lr=0.1, momentum=0.9, weight_decay=1e-4)
    assert not opt.is_flat
    for _ in range(2):
        for p in ps:
            p.grad = torch.randn_like(p) * 1e-3
        opt.step()
    sd = copy.deepcopy(opt.state_dict())
    twin = [torch.nn.Parameter(p.detach().clone()) for p in ps]
    opt2 = FusedSGD(twin, lr=0.1, momentum=0.9, weight_decay=1e-4)
    opt2.load_state_dict(sd)
    for p, q in zip(ps, twin):
        for k in ("momentum_buffer", "master"):
            assert opt2.state[q][k].dtype == torch.float32 and torch.equal(opt2.state[q][k], opt.state[p][k])
    for p, q in zip(ps, twin):
        p.grad = torch.randn_like(p) * 1e-3
        q.grad = p.grad.clone()
    opt.step()
    opt2.step()
    torch.cuda.synchronize()
    for p, q in zip(ps, twin):
        assert torch.equal(p, q) and torch.equal(opt.state[p]["momentum_buffer"], opt2.state[q]["momentum_buffer"])
