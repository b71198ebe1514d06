"""wgmma / TMA GEMM (1x1 convolution with BatchNorm statistics in the epilogue) against PyTorch fp32."""
import copy

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def C():
    from pytorch_distributed_b200 import _ext
    return _ext.lib()


@pytest.mark.parametrize("shape", [(4, 64, 64, 8), (2, 128, 256, 5), (3, 64, 128, 3), (2, 256, 64, 16), (1, 512, 2048, 7),
                                   (2, 2048, 512, 7), (8, 64, 256, 28), (1, 192, 320, 11)])
def test_conv1x1_bnstats_matches_fp32_reference(shape):
    B, cin, cout, hw = shape
    torch.manual_seed(0)
    x = torch.randn(B, cin, hw, hw, device="cuda").bfloat16().contiguous(memory_format=torch.channels_last)
    w = (torch.randn(cout, cin, 1, 1, device="cuda") * 0.1).bfloat16()
    gs = torch.zeros(2 * cout, device="cuda")
    y = C().conv1x1_bnstats(x, w, gs)
    ref = F.conv2d(x.float(), w.float())
    assert y.shape == ref.shape and y.is_contiguous(memory_format=torch.channels_last)
    torch.testing.assert_close(y.float(), ref, rtol=1e-2, atol=1e-2 * float(ref.abs().max()))
    # the statistics are those of the STORED (bf16-rounded) tensor - what a separate BatchNorm pass would reduce
    yf = y.float()
    s_own, q_own = yf.sum(dim=(0, 2, 3)), (yf * yf).sum(dim=(0, 2, 3))
    torch.testing.assert_close(gs[:cout], s_own, rtol=1e-4, atol=1e-4 * float(s_own.abs().max() + 1))
    torch.testing.assert_close(gs[cout:], q_own, rtol=1e-4, atol=1e-4 * float(q_own.abs().max() + 1))
    s_ref, q_ref = ref.sum(dim=(0, 2, 3)), (ref * ref).sum(dim=(0, 2, 3))
    torch.testing.assert_close(gs[:cout], s_ref, rtol=1e-2, atol=1e-2 * float(s_ref.abs().max() + 1))
    torch.testing.assert_close(gs[cout:], q_ref, rtol=1e-2, atol=1e-2 * float(q_ref.abs().max() + 1))
    # accumulates (BN workspace semantics): a second call doubles the sums
    C().conv1x1_bnstats(x, w, gs)
    torch.testing.assert_close(gs[:cout], 2 * s_own, rtol=1e-4, atol=2e-4 * float(s_own.abs().max() + 1))


def test_bottleneck_with_fused_conv1x1_matches_unfused():
    from pytorch_distributed_b200.models import resnet
    from pytorch_distributed_b200.ops.bn_act import begin_step
    from pytorch_distributed_b200.parallel.amp import cast_model
    torch.manual_seed(0)
    blk = resnet.Bottleneck(256, 64).cuda().to(memory_format=torch.channels_last)
    cast_model(blk, torch.bfloat16)
    ref = copy.deepcopy(blk)
    x = torch.randn(8, 256, 14, 14, device="cuda").bfloat16().contiguous(memory_format=torch.channels_last)
    outs = []
    for m, fused in ((blk, True), (ref, False)):
        resnet.FUSED_CONV1X1 = fused
        xx = x.clone().requires_grad_(True)
        begin_step(x.device)
        y = resnet._pair(m(xx))[0]     # a training block hands out two aliases of its output (SPLIT_RESGRAD)
        y.float().square().mean().backward()
        outs.append((y.detach().float(), xx.grad.float(), [p.grad.float() for p in m.parameters()], [b.float() for b in m.buffers()]))
    resnet.FUSED_CONV1X1 = False
    (ya, dxa, ga, ba), (yb, dxb, gb, bb) = outs
    torch.testing.assert_close(ya, yb, rtol=3e-2, atol=3e-2)
    torch.testing.assert_close(dxa, dxb, rtol=5e-2, atol=5e-2 * float(dxb.abs().max()))
    for a, b in zip(ga, gb):
        cos = torch.nn.functional.cosine_similarity(a.flatten(), b.flatten(), dim=0).item()
        assert cos > 0.99, cos
    for a, b in zip(ba, bb):
        torch.testing.assert_close(a, b, rtol=1e-2, atol=1e-2)
