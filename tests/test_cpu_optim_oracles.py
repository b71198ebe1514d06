"""The optimizer / gradient-wire references of tests/_fp64.py against plain PyTorch on CPU: sgd_step_fp64 against float64
torch.optim.SGD, the launch-geometry mirrors on hand-built tensor lists, and the wire-rounding and top-k references."""
import itertools
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _fp64 as R  # noqa: E402

CHUNK = R.MTA_CHUNK


@pytest.mark.parametrize("momentum,dampening,nesterov,wd,first",
                         [c for c in itertools.product([0.0, 0.9], [0.0, 0.1], [False, True], [0.0, 1e-4], [True, False])
                          if not (c[2] and (c[0] == 0.0 or c[1] != 0.0))])
def test_sgd_step_fp64_matches_torch_sgd(momentum, dampening, nesterov, wd, first):
    """torch.optim.SGD in float64: `first` is its first step (momentum buffer = gradient); otherwise one warm-up step
    builds the buffer, and the step under test starts from the state it left."""
    g = torch.Generator().manual_seed(0)
    p0 = torch.randn(257, generator=g, dtype=torch.float64)
    grads = [torch.randn(257, generator=g, dtype=torch.float64) for _ in range(2)]
    lr = 0.05
    p = torch.nn.Parameter(p0.clone())
    opt = torch.optim.SGD([p], lr=lr, momentum=momentum, dampening=dampening, nesterov=nesterov, weight_decay=wd)
    m = torch.zeros_like(p0)
    if not first:
        p.grad = grads[0].clone()
        opt.step()
        if momentum:
            m = opt.state[p]["momentum_buffer"].clone()
    before = p.detach().clone()
    p.grad = grads[1].clone()
    opt.step()
    ref = R.sgd_step_fp64(before, m, grads[1], (lr, momentum, wd, dampening, 1.0), nesterov, first)
    torch.testing.assert_close(ref["p"], p.detach(), rtol=1e-14, atol=1e-15)
    if momentum:
        torch.testing.assert_close(ref["m"], opt.state[p]["momentum_buffer"], rtol=1e-14, atol=1e-15)
    assert (ref["p_bound"] > 0).all() and (ref["m_bound"] > 0).all()


def test_sgd_step_fp64_gmul_unscales():
    p, m, gr = torch.ones(4, dtype=torch.float64), torch.zeros(4, dtype=torch.float64), torch.full((4,), 65536.0, dtype=torch.float64)
    ref = R.sgd_step_fp64(p, m, gr, (0.5, 0.0, 0.0, 0.0, 2.0 ** -16), False, True)
    assert torch.equal(ref["p"], torch.full((4,), 0.5, dtype=torch.float64))


def test_sgd_bound_rejects_a_two_ulp_error():
    """An fp32 step computed in fp32 passes check_sgd; the same master moved by 2 ulp does not."""
    g = torch.Generator().manual_seed(1)
    p, gr = torch.randn(1000, generator=g), torch.randn(1000, generator=g)
    m = torch.randn(1000, generator=g)
    hyper = (0.1, 0.9, 1e-4, 0.0, 1.0)
    a = gr + 1e-4 * p
    m1 = 0.9 * m + 1.0 * a
    p1 = p - 0.1 * m1
    ref = R.sgd_step_fp64(p, m, gr, hyper, False, False)
    R.check_sgd("fp32", p1, m1, ref)
    bad = p1.clone()
    bad[17] = bad[17] + 2 * R.ulp(bad[17:18], torch.float32)[0].float()
    with pytest.raises(AssertionError, match="master"):
        R.check_sgd("edited", bad, m1, ref)


def _flat_ranges(launches):
    out = {}
    for L in launches:
        for t, (c0, c1) in L["ranges"].items():
            out.setdefault(t, []).append((c0, c1))
    return out


@pytest.mark.parametrize("numels", [
    [0, 5, 0, 0, 7],
    [CHUNK, CHUNK - 1, CHUNK + 1, 3 * CHUNK, 3 * CHUNK - 1, 3 * CHUNK + 1],
    [1] * 95,
    [CHUNK * 700 + 3],
    [5, CHUNK * 319, CHUNK + 1, 0, 9] + [1] * 40,
])
def test_mta_geometry_covers_every_chunk_once(numels):
    launches = R.mta_geometry(numels)
    for L in launches:
        assert 0 < L["blocks"] <= R.MTA_BLOCKS and len(L["tensors"]) <= R.MTA_TENSORS
        assert L["blocks"] == sum(c1 - c0 for c0, c1 in L["ranges"].values())
        assert len(set(L["tensors"])) == len(L["tensors"])
    assert [L["reason"] for L in launches[:-1]] == [L["reason"] for L in launches[:-1] if L["reason"] in ("tensors", "blocks")]
    assert launches[-1]["reason"] == "end"
    ranges = _flat_ranges(launches)
    for i, n in enumerate(numels):
        if n == 0:
            assert i not in ranges
            continue
        rs = ranges[i]
        assert rs[0][0] == 0 and rs[-1][1] == R.cdiv(n, CHUNK)
        assert all(a[1] == b[0] for a, b in zip(rs, rs[1:]))      # contiguous, no chunk twice


def test_mta_geometry_hand_built_cases():
    # 30-tensor limit: the 31st tensor starts a new launch
    L = R.mta_geometry([1] * 31)
    assert [x["reason"] for x in L] == ["tensors", "end"] and L[1]["tensors"] == [30]
    # exactly 320 chunks fill one launch; the next tensor starts another, flushed for blocks
    L = R.mta_geometry([CHUNK * 320, 1])
    assert [x["reason"] for x in L] == ["blocks", "end"] and L[0]["ranges"] == {0: (0, 320)}
    # 320 * CHUNK + 1 elements: one chunk spills into a second launch
    L = R.mta_geometry([CHUNK * 320 + 1])
    assert [x["ranges"] for x in L] == [{0: (0, 320)}, {0: (320, 321)}]
    # a tensor of more than 320 chunks spans three launches, re-registered in each
    L = R.mta_geometry([3, CHUNK * 700 + 5])
    assert [x["ranges"] for x in L] == [{0: (0, 1), 1: (0, 319)}, {1: (319, 639)}, {1: (639, 701)}]
    assert [x["reason"] for x in L] == ["blocks", "blocks", "end"]
    # zero-size tensors are skipped: no launch at all for an all-empty list
    assert R.mta_geometry([0, 0]) == []
    # numel = 8192 k +- 1
    assert R.mta_geometry([CHUNK * 2 - 1])[0]["ranges"] == {0: (0, 2)}
    assert R.mta_geometry([CHUNK * 2 + 1])[0]["ranges"] == {0: (0, 3)}


def test_sgd_flat_geometry():
    n = 25_557_032 + 8 * 1000
    g = R.sgd_flat_geometry(n, 132)
    assert g["grid"] == 132 * 8 and g["iters"] == R.cdiv(n // 8, 132 * 8 * 256) and g["iters"] > 1
    g = R.sgd_flat_geometry(8 * 256 * 3, 132)
    assert g["grid"] == 3 and g["iters"] == 1


def test_wire_round_is_round_to_nearest_even():
    f16 = torch.float16
    x = torch.tensor([65504.0, 65519.99, 65520.0, -70000.0, 2.0 ** -25, 3 * 2.0 ** -26, 2.0 ** -24 * 1.5, 1 + 2.0 ** -11])
    y = R.wire_round(x, 1.0, f16)
    assert y[0] == 65504 and y[1] == 65504 and torch.isinf(y[2]) and y[3] == float("-inf")
    assert y[4] == 0 and y[5] == 2.0 ** -24 and y[6] == 2.0 ** -23 and y[7] == 1.0     # ties to even, subnormals
    b = R.wire_round(torch.tensor([1 + 2.0 ** -8, 1 + 3 * 2.0 ** -8]), 1.0, torch.bfloat16)
    assert b.tolist() == [1.0, 1 + 2.0 ** -6]


def test_assert_bits_equal_catches_one_rounding():
    x = torch.randn(1000).to(torch.bfloat16)
    R.assert_bits_equal("same", x, x.clone())
    y = x.clone()
    y.view(torch.int16)[3] += 1
    with pytest.raises(AssertionError, match="bitwise"):
        R.assert_bits_equal("edited", y, x)


def test_topk_reference_matches_accuracy_and_rejects_bad_targets():
    from pytorch_distributed_b200.utils.meters import accuracy
    g = torch.Generator().manual_seed(0)
    logits = torch.randn(64, 37, generator=g).to(torch.bfloat16).float()
    logits[:, 5] = logits[:, 3]                       # ties at the target value count as correct
    target = torch.randint(0, 37, (64,), generator=g)
    target[:8] = 5
    a1, a5 = accuracy(logits, target, (1, 5))
    c1, c5 = R.topk_correct_ref(logits, target)
    assert c1 == round(a1.item() * 64 / 100) and c5 == round(a5.item() * 64 / 100)
    bad = target.clone()
    bad[0], bad[1] = -1, 37
    r1, r5 = R.topk_correct_ref(logits, bad)
    ok = R.topk_correct_ref(logits[2:], target[2:])
    assert (r1, r5) == tuple(ok)
