"""The float64 references of tests/_fp64.py against fp64 autograd of the plain PyTorch composition, on small CPU tensors."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _fp64 as R  # noqa: E402

EPS = 1e-5


def _bn_case(shape, res, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(shape, generator=g, dtype=torch.float64) * 3 + 1
    w = torch.rand(shape[1], generator=g, dtype=torch.float64) + 0.5
    b = torch.randn(shape[1], generator=g, dtype=torch.float64)
    r = torch.randn(shape, generator=g, dtype=torch.float64) if res else None
    dy = torch.randn(shape, generator=g, dtype=torch.float64)
    return x, w, b, r, dy


@pytest.mark.parametrize("res", [False, True])
@pytest.mark.parametrize("relu", [False, True])
def test_bn_references_match_autograd(res, relu):
    x, w, b, r, dy = _bn_case((3, 16, 5, 7), res)
    xx, ww, bb = (t.clone().requires_grad_(True) for t in (x, w, b))
    rm, rv = torch.zeros(16, dtype=torch.float64), torch.ones(16, dtype=torch.float64)
    out = F.batch_norm(xx, rm, rv, ww, bb, training=True, momentum=0.1, eps=EPS)
    if res:
        out = out + r
    if relu:
        out = F.relu(out)
    out.backward(dy)

    st = R.batch_stats(R.rows(x), EPS)
    pre, _ = R.bn_apply_ref(R.rows(x), st["mean"], st["invstd"], w, b, R.rows(r) if res else None, relu)
    ref = pre.clamp_min(0) if relu else pre
    torch.testing.assert_close(ref, R.rows(out.detach()), rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(rm, st["mean"] * 0.1, rtol=1e-12, atol=1e-12)
    M = x.numel() // 16
    torch.testing.assert_close(rv, 0.9 + 0.1 * st["var"] * M / (M - 1), rtol=1e-12, atol=1e-12)

    dz = R.rows(dy) * (pre > 0) if relu else R.rows(dy)
    bw = R.bn_backward_ref(dz, R.rows(x), st["mean"], st["invstd"], w, depth=1)
    torch.testing.assert_close(bw["dx"], R.rows(xx.grad), rtol=1e-10, atol=1e-12)
    torch.testing.assert_close(bw["dgamma"], ww.grad, rtol=1e-10, atol=1e-12)
    torch.testing.assert_close(bw["dbeta"], bb.grad, rtol=1e-10, atol=1e-12)


@pytest.mark.parametrize("shape", [(2, 16, 9, 9), (3, 8, 8, 10), (2, 24, 13, 6)])
def test_stem_references_match_autograd(shape):
    N, C, H, W = shape
    x, s = R.tie_free_stem_input(N, C, H, W, seed=1)
    w = torch.rand(C, dtype=torch.float64) + 0.5
    b = R.stem_bias_between_levels(x, s, w, EPS)
    xx, ww, bb = (t.clone().requires_grad_(True) for t in (x, w, b))
    pre = F.batch_norm(xx, None, None, ww, bb, training=True, eps=EPS)
    out = F.max_pool2d(F.relu(pre), 3, 2, 1)
    dp = torch.randint(-8, 9, out.shape, generator=torch.Generator().manual_seed(2)).double() / 8
    out.backward(dp)

    st = R.batch_stats(R.rows(x), EPS)
    y, code, _, margin = R.stem_forward_ref(x, st["mean"], st["invstd"], w, b)
    assert margin > 1e3                     # the bias keeps every pre-activation far from 0
    torch.testing.assert_close(y, out.detach(), rtol=1e-12, atol=1e-12)
    # the code reproduces the pooled value: 15 <=> y == 0, otherwise y is the pre-activation at (2oh-1+kh, 2ow-1+kw)
    OH, OW = y.shape[2:]
    prep = F.pad(pre.detach(), (1, 1, 1, 1))
    assert (y[code == 15] == 0).all()
    for k in range(9):
        v = prep[:, :, k // 3:k // 3 + 2 * OH:2, k % 3:k % 3 + 2 * OW:2]
        sel = code == k
        assert (v[sel] > 0).all()
        torch.testing.assert_close(y[sel], v[sel], rtol=1e-12, atol=1e-12)
    assert int((code < 9).sum()) + int((code == 15).sum()) == code.numel()

    dz = R.stem_dz_ref(dp, code, H, W)
    bw = R.bn_backward_ref(R.rows(dz), R.rows(x), st["mean"], st["invstd"], w, depth=1)
    torch.testing.assert_close(bw["dx"], R.rows(xx.grad), rtol=1e-10, atol=1e-12)
    torch.testing.assert_close(bw["dgamma"], ww.grad, rtol=1e-10, atol=1e-12)
    torch.testing.assert_close(bw["dbeta"], bb.grad, rtol=1e-10, atol=1e-12)


@pytest.mark.parametrize("shape", [(2, 8, 9, 9), (1, 16, 12, 15), (3, 4, 7, 8)])
def test_tie_free_stem_input_has_no_tie_in_any_window(shape):
    N, C, H, W = shape
    x, s = R.tie_free_stem_input(N, C, H, W, seed=3)
    assert torch.equal(x.to(torch.bfloat16).double(), x) and torch.equal(x.half().double(), x)
    cols = F.unfold(x, 3, padding=1, stride=2).view(N, C, 9, -1)
    valid = F.unfold(torch.ones(1, 1, H, W, dtype=torch.float64), 3, padding=1, stride=2).view(1, 1, 9, -1).bool()
    same = cols[:, :, :, None, :] == cols[:, :, None, :, :]
    both = valid[:, :, :, None, :] & valid[:, :, None, :, :]
    off_diag = ~torch.eye(9, dtype=torch.bool)[None, None, :, :, None]
    assert not (same & both & off_diag).any()


def test_conv1x1_reference_and_its_checker():
    g = torch.Generator().manual_seed(4)
    x = torch.randn(2, 64, 5, 3, generator=g).bfloat16()
    w = torch.randn(128, 64, 1, 1, generator=g).bfloat16()
    ref = F.conv2d(x.double(), w.double())
    y = ref.bfloat16()
    R.check_conv1x1(y, x, w, max_changed=0.0)
    bad = y.clone()
    bad[1, 7, 2, 1] = (bad[1, 7, 2, 1].double() + 2 * R.ulp(bad[1, 7, 2, 1], torch.bfloat16)).bfloat16()
    with pytest.raises(AssertionError):
        R.check_conv1x1(bad, x, w)


def test_ulp_and_geometry_mirrors():
    v = torch.tensor([1.0, 1.5, 2.0, 0.75, 0.0, -3.0], dtype=torch.float64)
    assert R.ulp(v, torch.bfloat16).tolist()[:4] == [2.0 ** -7, 2.0 ** -7, 2.0 ** -6, 2.0 ** -8]
    assert R.ulp(v, torch.float16)[5].item() == 2.0 ** -9 and R.ulp(v, torch.float32)[0].item() == 2.0 ** -23
    g = R.gemm_geometry(M=128 * 132 + 1, N=256, K=64, sms=132)
    assert g["block_n"] == 256 and g["m_tiles"] == 133 and g["ctas_per_n"] == 132
    assert g["max_tiles_per_cta"] == 2 and g["ctas_with_max_tiles"] == 1
    b = R.bn_reduce_geometry(M=2, C=2056, sms=132, resident=4)
    assert b["tpr"] == 256 and b["chunks"] == 2 and b["ragged"] and b["grid"] == 1
    s = R.stem_bwd_geometry(256, 64, 112, 112, sms=132)
    assert s["rows_per_block"] == 4 and not s["crosses_images"]
