"""The collective references of tests/_fp64.py on CPU: the rank-order all-reduce against a float64 sum, proof that the
bitwise checks can tell a staggered summation order from rank order, and the slice-ownership and loop-geometry mirrors
against parallel/plan.build_layout."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _fp64 as R  # noqa: E402

from pytorch_distributed_b200.parallel import plan as P  # noqa: E402

F32, BF16, F16 = torch.float32, torch.bfloat16, torch.float16


def _ranks(W, n, dtype, seed=0):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(n, generator=g) * torch.exp2(torch.randint(-6, 7, (n,), generator=g).float())).to(dtype)
            for _ in range(W)]


@pytest.mark.parametrize("W", [2, 3, 7, 16])
@pytest.mark.parametrize("dtype", [F32, BF16, F16], ids=lambda d: str(d).replace("torch.", ""))
def test_allreduce_ref_within_fp32_bound_of_fp64(W, dtype):
    """W - 1 fp32 additions (the first add into +0.0 is exact), then one rounding to the wire dtype."""
    xs = _ranks(W, 20000, dtype, seed=W)
    got = R.allreduce_ref(xs)
    assert got.dtype == dtype
    exact = torch.stack([x.double() for x in xs]).sum(0)
    mag = torch.stack([x.double().abs() for x in xs]).sum(0)
    R.assert_within("allreduce_ref", got, exact, 1.01 * (W - 1) * R.U32 * mag + 0.5 * R.ulp(got, dtype))
    scaled = R.allreduce_ref(xs, dtype, 0.37, prepacked=True)
    acc = torch.zeros(20000)
    for x in xs:
        acc += x.float()
    R.assert_bits_equal("prepacked", scaled, (acc * np.float32(0.37)).to(dtype))


def test_allreduce_ref_adds_in_rank_order_from_plus_zero():
    neg0 = torch.tensor([-0.0])
    assert torch.signbit(R.allreduce_ref([neg0, neg0])).item() is False      # +0 + -0 + -0 = +0
    big = [torch.tensor([3e38]), torch.tensor([3e38]), torch.tensor([-3e38])]
    assert torch.isinf(R.allreduce_ref(big)).all()                           # (3e38 + 3e38) overflows first


def test_staggered_order_differs_on_the_overflow_case():
    """fp32 wire values 3e38, 3e38, -3e38 on ranks 0, 1, 2: rank order gives inf on every rank, a sum that starts at the
    caller's rank gives inf on rank 0 and 3e38 on ranks 1 and 2, so the non-finite decision would differ by rank."""
    xs = [torch.tensor([3e38]), torch.tensor([3e38]), torch.tensor([-3e38])]
    ref = R.allreduce_ref(xs)
    st = [R.staggered_ref(xs, r) for r in range(3)]
    assert torch.isinf(ref).all() and torch.isinf(st[0]).all()
    assert torch.isfinite(st[1]).all() and torch.isfinite(st[2]).all()
    R.assert_bits_equal("rank 0 starts at rank 0", st[0], ref)
    for r in (1, 2):
        with pytest.raises(AssertionError, match="bitwise"):
            R.assert_bits_equal("staggered rank %d" % r, st[r], ref)


def test_staggered_order_differs_on_random_world3_data():
    """On an fp32 wire the last bit of a three-term sum depends on the order for a real fraction of random values.  (On
    16-bit wires the final rounding to 8 or 11 bits hides almost every such difference.)"""
    xs = _ranks(3, 100000, F32, seed=5)
    ref = R.allreduce_ref(xs)
    for r in (1, 2):
        st = R.staggered_ref(xs, r)
        frac = (st.view(torch.int32) != ref.view(torch.int32)).double().mean().item()
        assert frac > 1e-2, "rank %d: only %.3g of the elements differ" % (r, frac)
        with pytest.raises(AssertionError, match="bitwise"):
            R.assert_bits_equal("staggered rank %d" % r, st, ref)


RAGGED = [[1000], [5, 64, 3, 1, 129, 4096, 7], [64 * 3 * 7 * 7, 64, 64, 4097, 33 * 17, 1, 2048], [8193, 1000, 2048 * 1000 // 64]]


@pytest.mark.parametrize("W", list(range(2, 17)))
def test_slice_owner_agrees_with_build_layout(W):
    for numels in RAGGED:
        offs, total = P.tensor_layout(numels)
        for grid in (1, 3, 7):
            lay = P.build_layout(numels, W, grid, offs, total)
            assert lay.block_elems % (W * 8) == 0
            slice_elems = lay.block_elems // W
            seen = 0
            for b in range(grid):
                for s in lay.segs[lay.seg_begin[b]:lay.seg_begin[b + 1]]:
                    pos = torch.arange(int(s["arena_off"]), int(s["arena_off"]) + int(s["len"]))
                    t = int(s["tensor"])
                    assert offs[t] + int(s["src_off"]) == pos[0].item()
                    assert (pos // lay.block_elems == b).all(), "segment outside CTA %d" % b
                    own = R.slice_owner(lay, pos)
                    assert torch.equal(own, (pos - b * lay.block_elems) // slice_elems)
                    assert int(own.min()) >= 0 and int(own.max()) < W
                    seen += int(s["len"])
            assert seen == sum(numels)
            # every rank owns exactly one slice of each CTA range
            allpos = torch.arange(lay.region_elems)
            counts = torch.bincount(R.slice_owner(lay, allpos), minlength=W)
            assert (counts == grid * slice_elems).all()


def test_loop_units_split():
    T = R.COLL_THREADS
    assert R.loop_units(100, 8) == dict(units=100, main_units=0, tail_units=100)          # 16 KiB ranges never unroll
    assert R.loop_units(8 * T, 8) == dict(units=8 * T, main_units=8 * T, tail_units=0)
    g = R.loop_units(8 * T + 5, 8)
    assert g["main_units"] == 8 * T and g["tail_units"] == 5
    g = R.loop_units(2 * 8 * T - 1, 8)                                                     # second round short by one
    assert g["main_units"] == 8 * T + 8 * (T - 1) and g["tail_units"] == 7
    assert R.loop_units(4 * T + 3, 4)["tail_units"] == 3
