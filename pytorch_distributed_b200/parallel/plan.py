"""Static launch plans for the fused multi-tensor collectives (pure numpy - testable without a GPU).

A *plan* fixes, once, how a list of tensors maps onto a contiguous range of the symmetric arena and how that
range is cut into per-CTA sub-ranges (``csrc/collectives.cu``: CTA ``b`` owns ``[b*block_elems, (b+1)*block_elems)``
on every rank).  This is the H100-native counterpart of torch's bucket assignment
(``dist._compute_bucket_assignment_by_size``; reference call site /root/reference/distributed.py:147).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Sequence

import numpy as np

ALIGN_ELEMS = 64          # every tensor starts on a 64-element boundary inside the arena
SEG_DTYPE = np.dtype([("tensor", "<i4"), ("len", "<i4"), ("src_off", "<i8"), ("arena_off", "<i8")])
assert SEG_DTYPE.itemsize == 24

WIRE_CODES = {"fp32": 0, "bf16": 1, "fp16": 2}
WIRE_BYTES = {"fp32": 4, "bf16": 2, "fp16": 2}


def round_up(x: int, m: int) -> int:
    return (x + m - 1) // m * m


def tensor_layout(numels: Sequence[int], align: int = ALIGN_ELEMS):
    """Offsets (in elements) of each tensor inside the plan's range, and the padded total."""
    offs, cur = [], 0
    for n in numels:
        offs.append(cur)
        cur += round_up(int(n), align)
    return offs, cur


def choose_grid(total_elems: int, elem_bytes: int, max_ctas: int, bytes_per_cta: int = 256 << 10) -> int:
    nbytes = total_elems * elem_bytes
    return int(max(1, min(max_ctas, (nbytes + bytes_per_cta - 1) // bytes_per_cta)))


@dataclass
class PlanLayout:
    numels: List[int]
    offsets: List[int]
    total: int            # padded elements actually covered by tensors
    grid: int
    world: int
    block_elems: int
    seg_begin: np.ndarray = field(repr=False, default=None)
    segs: np.ndarray = field(repr=False, default=None)

    @property
    def region_elems(self) -> int:
        return self.grid * self.block_elems


def build_layout(numels: Sequence[int], world: int, grid: int, offsets: Sequence[int] | None = None,
                 total: int | None = None) -> PlanLayout:
    """Cut ``[0, total)`` into ``grid`` equal CTA ranges (each a multiple of world*8 elements so that every rank's
    slice of every CTA range is 16-byte aligned for any wire dtype) and emit the per-CTA segment table."""
    numels = [int(n) for n in numels]
    if offsets is None:
        offsets, total = tensor_layout(numels)
    offsets = [int(o) for o in offsets]
    total = int(total)
    quantum = world * 8
    block_elems = max(round_up((total + grid - 1) // grid, quantum), quantum)
    seg_begin = np.zeros(grid + 1, dtype=np.int32)
    segs = []
    order = np.argsort(np.asarray(offsets, dtype=np.int64), kind="stable") if offsets else []
    ti = 0
    for b in range(grid):
        lo, hi = b * block_elems, (b + 1) * block_elems
        # advance to the first tensor that may overlap this range
        while ti < len(order) and offsets[order[ti]] + numels[order[ti]] <= lo:
            ti += 1
        k = ti
        while k < len(order) and offsets[order[k]] < hi:
            t = int(order[k])
            s, e = max(lo, offsets[t]), min(hi, offsets[t] + numels[t])
            if e > s:
                segs.append((t, e - s, s - offsets[t], s))
            k += 1
        seg_begin[b + 1] = len(segs)
    seg_arr = np.array(segs, dtype=SEG_DTYPE) if segs else np.zeros(0, dtype=SEG_DTYPE)
    return PlanLayout(numels, offsets, total, grid, world, block_elems, seg_begin, seg_arr)


def compute_buckets(numels: Sequence[int], elem_bytes: int, cap_bytes: int, first_cap_bytes: int | None = None,
                    max_tensors: int = 256, tail_cap_bytes: int | None = None) -> List[List[int]]:
    """Greedy size-capped bucket assignment over tensors in the given (gradient-ready) order.

    Mirrors torch's reducer defaults (first bucket 1 MiB so communication starts early, then ``cap_bytes``); a bucket
    is also closed when it holds ``max_tensors`` tensors (pointer pack limit of one kernel launch).
    ``tail_cap_bytes``: the LAST bucket is the only one whose all-reduce cannot hide behind backward compute - it is on
    the critical path between the last gradient and the optimizer - so the final tensors (as many as fit in
    ``tail_cap_bytes``) are split off into their own small bucket.
    """
    if tail_cap_bytes is not None and len(numels) > 1:
        k, acc = len(numels), 0
        while k > 1 and acc + int(numels[k - 1]) * elem_bytes <= tail_cap_bytes and len(numels) - k < max_tensors:
            k -= 1
            acc += int(numels[k]) * elem_bytes
        if 0 < k < len(numels):
            head = compute_buckets(numels[:k], elem_bytes, cap_bytes, first_cap_bytes, max_tensors)
            return head + [list(range(k, len(numels)))]
    buckets, cur, cur_bytes = [], [], 0
    cap = first_cap_bytes if first_cap_bytes is not None else cap_bytes
    for i, n in enumerate(numels):
        nb = int(n) * elem_bytes
        if cur and (cur_bytes + nb > cap or len(cur) >= max_tensors):
            buckets.append(cur)
            cur, cur_bytes = [], 0
            cap = cap_bytes
        cur.append(i)
        cur_bytes += nb
    if cur:
        buckets.append(cur)
    return buckets
