"""FusedSGD.load_state_dict keeps momentum and masters in fp32: torch's Optimizer.load_state_dict casts loaded state to
each parameter's dtype, which would round a bf16 model's fp32 momentum to bf16 on resume."""
import copy

import torch

from pytorch_distributed_b200.ops.fused_sgd import FusedSGD


def _trained(dtype):
    torch.manual_seed(0)
    ps = [torch.nn.Parameter(torch.randn(64, 32).to(dtype)), torch.nn.Parameter(torch.randn(32).to(dtype))]
    opt = FusedSGD(ps, lr=0.1, momentum=0.9, weight_decay=1e-4)
    for _ in range(2):
        for p in ps:
            p.grad = (torch.randn(p.shape) * 1e-3).to(dtype)
        opt.step()
    return ps, opt


def test_resume_keeps_fp32_momentum_and_masters_of_a_bf16_model():
    ps, opt = _trained(torch.bfloat16)
    sd = copy.deepcopy(opt.state_dict())
    for p in ps:
        assert opt.state[p]["momentum_buffer"].dtype == torch.float32 and opt.state[p]["master"].dtype == torch.float32
    twin = [torch.nn.Parameter(p.detach().clone()) for p in ps]
    opt2 = FusedSGD(twin, lr=0.1, momentum=0.9, weight_decay=1e-4)
    opt2.load_state_dict(sd)
    for p, q in zip(ps, twin):
        for k in ("momentum_buffer", "master"):
            assert opt2.state[q][k].dtype == torch.float32 and torch.equal(opt2.state[q][k], opt.state[p][k])
    # and the next step continues exactly as the uninterrupted optimizer does
    for p, q in zip(ps, twin):
        p.grad = (torch.randn(p.shape) * 1e-3).to(p.dtype)
        q.grad = p.grad.clone()
    opt.step()
    opt2.step()
    for p, q in zip(ps, twin):
        assert torch.equal(p, q) and torch.equal(opt.state[p]["momentum_buffer"], opt2.state[q]["momentum_buffer"])


def test_resume_of_an_fp32_model_is_unchanged():
    ps, opt = _trained(torch.float32)
    sd = copy.deepcopy(opt.state_dict())
    twin = [torch.nn.Parameter(p.detach().clone()) for p in ps]
    opt2 = FusedSGD(twin, lr=0.1, momentum=0.9, weight_decay=1e-4)
    opt2.load_state_dict(sd)
    for p, q in zip(ps, twin):
        assert "master" not in opt2.state[q] and torch.equal(opt2.state[q]["momentum_buffer"], opt.state[p]["momentum_buffer"])
