"""The multi-rank fused collectives of ``csrc/collectives.cu`` at world sizes 2 to 16, emulated on one GPU, checked
bitwise against a rank-order reference (tests/_fp64.py).

Emulation.  One zeroed CUDA buffer of W x R bytes holds W arenas (rank r's at ``buf + r * R``, its signal pad first);
``SymmArena.from_pointers`` builds W genuine contexts over it (world = W, each with its own sequence counters).  The
kernels reach peers only through plain or ``.sys`` loads and stores of ``c.base[p]``, so they run unchanged when every
peer lives on the same device.  Ranks run one after another, never concurrently.

Safety rule: no launch depends on another launch running at the same time, and no kernel ever waits.
* Before each round (one call of one flag kernel on every rank) the harness writes ``flags[channel][b][p]`` in every
  rank's pad, for every CTA b of the plan, to 2^30 past the last sequence number the round can reach
  (``arm_barriers``).  The kernels' own barrier stores overwrite these with real sequence numbers, which are still at
  least what the later ranks of the round wait for.
* Before each LL call (metrics, LL all-reduce) it writes every inbox word ``{value, seq}`` a rank reads before the
  rank that owns it has run (``arm_inbox``).
* Both read the words back on the host and assert them before anything is launched; a flag kernel launched outside an
  armed round is refused by ``launch``.

Schedules that stay faithful to each kernel: two-shot prepacked (rank r writes slice r everywhere; afterwards every
arena holds the whole result), two-shot with pack and write-back (rank r re-packs its own arena, so only its slice is
checked, right after its launch), one-shot (every rank packed into the staging half of the call's parity first),
broadcast (root first), the host-synchronised kinds 3-6 (no flags), the barrier and the LL kernels.
"""
import functools
import math
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _fp64 as R  # noqa: E402

from pytorch_distributed_b200.parallel import plan as P  # noqa: E402

pytestmark = pytest.mark.gpu

DEV = "cuda"
F32, BF16, F16 = torch.float32, torch.bfloat16, torch.float16
WIRE_DT = {"fp32": F32, "bf16": BF16, "fp16": F16}
SRC_DTS = [F32, BF16, F16]
WORLDS = [2, 3, 4, 7, 8, 16]
WIRES = ["fp32", "bf16", "fp16"]
PRESET_LEAD = 1 << 30
CH = 0                           # the signal channel every emulated launch uses
KIND_TWO_SHOT, KIND_ONE_SHOT, KIND_BCAST, KIND_PACK, KIND_REDUCE, KIND_PUSH, KIND_UNPACK = range(7)
FLAG_PREPACKED = 1


def C():
    from pytorch_distributed_b200 import _ext
    return _ext.lib()


@functools.lru_cache(maxsize=1)
def r50_shapes():
    from pytorch_distributed_b200.models import create_model
    shapes = [tuple(p.shape) for p in create_model("resnet50").parameters()]
    assert len(shapes) == 161 and sum(math.prod(s) for s in shapes) == 25_557_032
    return shapes


class _Words:
    """Device int32 words exposed to torch.as_tensor (the arenas' local sequence counters)."""

    def __init__(self, ptr: int, n: int):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<i4", "data": (ptr, False), "strides": None, "version": 2}


class _PlanHost:
    """What parallel.comm.Plan asks of a communicator; every offset comes from the emulated arena instead."""
    max_blocks = 64

    def __init__(self, world: int):
        self.world = world

    def device_of(self, rank_slot: int = 0) -> torch.device:
        return torch.device(DEV, 0)

    def alloc(self, nbytes: int) -> int:
        raise AssertionError("emulated plans take their arena offsets from EmulatedWorld.alloc")


class EmulatedWorld:
    def __init__(self, W: int, data_bytes: int):
        self.C = C()
        self.W = W
        self.header = P.round_up(self.C.SIGNAL_PAD_BYTES, 128 << 10)
        self.R = P.round_up(self.header + data_bytes, 1 << 16)
        self.buf = torch.zeros(W * self.R, dtype=torch.uint8, device=DEV)
        base = self.buf.data_ptr()
        self.ptrs = [base + r * self.R for r in range(W)]
        self.arenas = [self.C.SymmArena.from_pointers(r, W, self.ptrs, 0, self.R, 0) for r in range(W)]
        nseq = self.C.MAX_CHANNELS * self.C.MAX_BLOCKS
        self.seq = [torch.as_tensor(_Words(a.ll_seq_ptr() - 4 * nseq, nseq + 1), device=DEV) for a in self.arenas]
        self.found_inf_off = P.round_up(self.C.SIGNAL_PAD_BYTES, 64)
        self.bump = self.header
        self.expect_seq = torch.zeros(self.C.MAX_BLOCKS, dtype=torch.int32)   # barrier sequence of (CH, b) on every rank
        self.expect_ll = 0
        self.armed = None
        torch.cuda.synchronize()

    # ------------------------------------------------------------------ memory
    def alloc(self, nbytes: int) -> int:
        off = P.round_up(self.bump, 4096)
        assert off + nbytes <= self.R, "emulated arena too small"
        self.bump = off + nbytes
        return off

    def view(self, r: int, off_bytes: int, n: int, dtype) -> torch.Tensor:
        esz = torch.tensor([], dtype=dtype).element_size()
        lo = r * self.R + off_bytes
        return self.buf[lo:lo + n * esz].view(dtype)

    def flags(self, r: int) -> torch.Tensor:
        M = self.C
        return self.view(r, 0, M.MAX_CHANNELS * M.MAX_BLOCKS * M.MAX_WORLD, torch.int32).view(M.MAX_CHANNELS, M.MAX_BLOCKS, M.MAX_WORLD)

    def inbox(self, r: int) -> torch.Tensor:
        M = self.C
        off = M.MAX_CHANNELS * M.MAX_BLOCKS * M.MAX_WORLD * 4
        return self.view(r, off, 2 * M.MAX_WORLD * 8 * 2, torch.int32).view(2, M.MAX_WORLD, 8, 2)

    def found_inf(self, r: int) -> torch.Tensor:
        return self.view(r, self.found_inf_off, 1, torch.int32)

    def found_inf_all(self) -> list:
        torch.cuda.synchronize()
        return [int(self.found_inf(r).item()) for r in range(self.W)]

    def clear_found_inf(self) -> None:
        for r in range(self.W):
            self.found_inf(r).zero_()

    def plans(self, numels, wire: str, regions: int, max_ctas: int = 32, bytes_per_cta: int = 256 << 10) -> list:
        """One plan per emulated rank (same layout, own device call counters) over ``regions`` consecutive plan regions."""
        from pytorch_distributed_b200.parallel.comm import Plan
        host = _PlanHost(self.W)
        pls = [Plan(host, numels, wire, max_ctas, False, data_off_bytes=-1, bytes_per_cta=bytes_per_cta) for _ in range(self.W)]
        off = self.alloc(pls[0].region_bytes * regions)
        for pl in pls:
            pl.data_off_bytes = off
        return pls

    # ------------------------------------------------------------------ safety rule
    def _block_seqs(self, grid: int) -> torch.Tensor:
        M = self.C
        return torch.stack([s[CH * M.MAX_BLOCKS:CH * M.MAX_BLOCKS + grid] for s in self.seq]).cpu()

    def arm_barriers(self, grid: int, barriers: int) -> None:
        """Preset every flag a round of `barriers` barriers per launch over `grid` CTAs waits on, then verify on the host."""
        assert self.armed is None
        torch.cuda.synchronize()
        want = self.expect_seq[:grid]
        seqs = self._block_seqs(grid)
        assert (seqs == want).all(), "sequence counters %s, expected %s" % (seqs.tolist(), want.tolist())
        preset = (want + barriers + PRESET_LEAD)[:, None].expand(grid, self.W).to(DEV)
        for r in range(self.W):
            self.flags(r)[CH, :grid, :self.W] = preset
        torch.cuda.synchronize()
        back = torch.stack([self.flags(r)[CH, :grid, :self.W] for r in range(self.W)]).cpu()
        assert (back - (want + barriers)[None, :, None] >= PRESET_LEAD).all(), "flag presets not in place"
        self.armed = grid

    def finish_round(self, grid: int, barriers: int) -> None:
        """After a round every pad holds every source rank's final sequence number, and every counter advanced."""
        assert self.armed == grid
        self.armed = None
        self.expect_seq[:grid] += barriers
        want = self.expect_seq[:grid]
        torch.cuda.synchronize()
        flags = torch.stack([self.flags(r)[CH, :grid, :self.W] for r in range(self.W)]).cpu()
        assert (flags == want[None, :, None]).all(), "barrier flags %s after the round, expected %s" % (flags.unique().tolist(), want.tolist())
        assert (self._block_seqs(grid) == want).all()
        assert all(a.status() == 0 for a in self.arenas)

    def arm_inbox(self, n: int, values: torch.Tensor) -> int:
        """LL call: preset inbox(dst)[parity][src] = {values[src], seq} for src >= dst (what dst reads before src has run);
        the words src < dst must still be stale, so that the kernel's own stores are what the test sees there."""
        assert self.armed is None
        torch.cuda.synchronize()
        M = self.C
        lls = torch.stack([s[M.MAX_CHANNELS * M.MAX_BLOCKS] for s in self.seq]).cpu()
        assert (lls == self.expect_ll).all()
        seq = self.expect_ll + 1
        par = seq & 1
        bits = values.to(DEV, torch.float32).contiguous().view(torch.int32)
        for dst in range(self.W):
            ib = self.inbox(dst)
            ib[par, dst:self.W, :n, 0] = bits[dst:, :n]
            ib[par, dst:self.W, :n, 1] = seq
        torch.cuda.synchronize()
        for dst in range(self.W):
            ib = self.inbox(dst)[par].cpu()
            assert torch.equal(ib[dst:self.W, :n, 0], bits[dst:, :n].cpu()) and (ib[dst:self.W, :n, 1] == seq).all()
            assert (ib[:dst, :n, 1] != seq).all(), "inbox words of ranks that have not run already carry the sequence"
        self.armed = "ll"
        return seq

    def finish_ll(self) -> None:
        assert self.armed == "ll"
        self.armed = None
        self.expect_ll += 1
        torch.cuda.synchronize()
        M = self.C
        assert all(int(s[M.MAX_CHANNELS * M.MAX_BLOCKS].item()) == self.expect_ll for s in self.seq)
        assert all(a.status() == 0 for a in self.arenas)

    # ------------------------------------------------------------------ launches
    def launch(self, r: int, pl, kind: int, tensors, scale: float = 1.0, writeback: bool = False, root: int = 0,
               check_inf: bool = False, prepacked: bool = False, result_off: int = -1, data_off=None) -> None:
        if kind <= KIND_BCAST:
            assert self.armed == pl.grid, "flag kernel launched outside an armed round"
        self.arenas[r].launch_plan(CH, 0, kind, P.WIRE_CODES[pl.wire], False, pl.grid, list(tensors), pl.seg_begin.data_ptr(),
                                   pl.segs.data_ptr(), pl.data_off_bytes if data_off is None else data_off, pl.block_elems,
                                   pl.calls.data_ptr(), self.ptrs[r] + self.found_inf_off if check_inf else 0, float(scale),
                                   bool(writeback), int(root), FLAG_PREPACKED if prepacked else 0, int(result_off))


# ================================================================================================ data and checkers
def _rand(n: int, dtype, gen: torch.Generator) -> torch.Tensor:
    """Normal values over 19 binades (2^-12 .. 2^6): wide enough that fp32 sums of 16-bit values are order-sensitive, with
    no nonzero |value| below 2^-100, so the extension's flush-to-zero cannot matter."""
    x = torch.randn(n, device=DEV, generator=gen) * torch.exp2(torch.randint(-12, 7, (n,), device=DEV, generator=gen).float())
    return x.to(dtype)


def rank_tensors(shapes, rank: int, seed: int = 0) -> list:
    """Rank `rank`'s gradient list: the given shapes in fp32 / bf16 / fp16 by turns, plus one dense view at an odd element
    offset (not 16-byte aligned)."""
    g = torch.Generator(device=DEV).manual_seed(1000 * seed + rank)
    ts = [_rand(math.prod(s), SRC_DTS[i % 3], g).view(s) for i, s in enumerate(shapes)]
    base = _rand(8195, SRC_DTS[len(shapes) % 3], g)
    ts.append(base[1:8194])
    assert ts[-1].data_ptr() % 16 != 0
    return ts


def numels_of(ts) -> list:
    return [t.numel() for t in ts]


class Layout:
    """Per source dtype: the flat concatenation order of a tensor list and the arena positions of its elements."""

    def __init__(self, ts, offsets):
        self.idx, self.pos = {}, {}
        for dt in SRC_DTS:
            ii = [i for i, t in enumerate(ts) if t.dtype == dt]
            self.idx[dt] = ii
            self.pos[dt] = torch.cat([torch.arange(offsets[i], offsets[i] + ts[i].numel(), device=DEV) for i in ii])

    def flat(self, ts, dt) -> torch.Tensor:
        return torch.cat([ts[i].reshape(-1) for i in self.idx[dt]])


def check_tensors(name, ts, lay: Layout, wire_vals: torch.Tensor, mask_fn=None) -> None:
    """Each tensor holds wire_vals at its arena positions, cast to its own dtype (optionally only where mask_fn(pos))."""
    for dt in SRC_DTS:
        got, pos = lay.flat(ts, dt), lay.pos[dt]
        exp = wire_vals[pos].to(dt)
        if mask_fn is not None:
            m = mask_fn(pos)
            got, exp = got[m], exp[m]
        R.assert_bits_equal("%s %s tensors" % (name, str(dt).replace("torch.", "")), got, exp)


def check_packed(name, arena_region: torch.Tensor, ts, lay: Layout, scale: float) -> None:
    """Kind 3 (and every pack phase): each element is fp32(src) * fp32(scale) rounded once to the wire dtype."""
    for dt in SRC_DTS:
        R.assert_bits_equal("%s %s" % (name, str(dt).replace("torch.", "")), arena_region[lay.pos[dt]],
                            R.wire_round(lay.flat(ts, dt), scale, arena_region.dtype))


def check_owned_slice(name, arena_region: torch.Tensor, ref: torch.Tensor, layout, rank: int) -> None:
    """The two-shot checker for one rank right after its launch: its slice of every CTA range equals the reference."""
    m = R.slice_owner(layout, torch.arange(layout.region_elems, device=DEV)) == rank
    R.assert_bits_equal(name, arena_region[m], ref[m])


def assert_plan_reaches(pl, ts, *, min_grid=2, straddle_cta=True, straddle_slice=True):
    lay = pl.layout
    assert pl.grid >= min_grid, "plan has %d CTAs" % pl.grid
    slice_elems = lay.block_elems // lay.world
    spans_cta = spans_slice = False
    for off, n in zip(lay.offsets, numels_of(ts)):
        spans_cta |= off // lay.block_elems != (off + n - 1) // lay.block_elems
        spans_slice |= off // slice_elems != (off + n - 1) // slice_elems
    assert spans_cta or not straddle_cta, "no tensor crosses a CTA range boundary"
    assert spans_slice or not straddle_slice, "no tensor crosses a slice boundary"


# ================================================================================================ K1 two-shot
@pytest.mark.parametrize("wire", WIRES)
@pytest.mark.parametrize("W", WORLDS)
def test_twoshot_prepacked_every_arena_bitwise(W, wire):
    """FLAG_PREPACKED (bucket views): rank r reduces and stores slice r into every arena; after the round every arena
    holds the rank-order sum, times the scale with one rounding.  Scale 1 and 0.37, with the non-finite check on."""
    wdt = WIRE_DT[wire]
    esz = P.WIRE_BYTES[wire]
    shapes = r50_shapes()
    numels = [math.prod(s) for s in shapes] + [8193]
    world = EmulatedWorld(W, P.tensor_layout(numels)[1] * esz * 2 + (8 << 20))
    pls = world.plans(numels, wire, 1)
    pl = pls[0]
    assert_plan_reaches(pl, [torch.empty(n, device="meta") for n in numels])
    assert R.twoshot_units(pl.layout, esz)["iters"] >= 2
    n = pl.layout.region_elems
    for call, scale in enumerate((1.0, 0.37)):
        data = []
        for r in range(W):
            g = torch.Generator(device=DEV).manual_seed(100 * call + r)
            v = world.view(r, pl.data_off_bytes, n, wdt)
            v.copy_(_rand(n, wdt, g))
            data.append(v.clone())
        views = [world.view(r, pl.data_off_bytes, 8, wdt) for r in range(W)]
        ref = R.allreduce_ref(data, wdt, scale, prepacked=True)
        world.clear_found_inf()
        world.arm_barriers(pl.grid, 2)
        for r in range(W):
            world.launch(r, pls[r], KIND_TWO_SHOT, [views[r]], scale=scale, check_inf=True, prepacked=True)
        world.finish_round(pl.grid, 2)
        assert world.found_inf_all() == [0] * W
        for r in range(W):
            R.assert_bits_equal("W=%d %s x%g arena of rank %d" % (W, wire, scale, r), world.view(r, pl.data_off_bytes, n, wdt), ref)


@pytest.mark.parametrize("wire", WIRES)
@pytest.mark.parametrize("W", WORLDS)
def test_twoshot_pack_writeback_owned_slices(W, wire):
    """Pack x 1/W (kind 3 on every rank first), then the two-shot kernel rank by rank with write-back: right after rank
    r's launch its slice of every CTA range, in its arena and in its tensors, is the rank-order sum."""
    wdt = WIRE_DT[wire]
    esz = P.WIRE_BYTES[wire]
    ts = [rank_tensors(r50_shapes(), r) for r in range(W)]
    numels = numels_of(ts[0])
    world = EmulatedWorld(W, P.tensor_layout(numels)[1] * esz + (8 << 20))
    pls = world.plans(numels, wire, 1)
    pl = pls[0]
    assert_plan_reaches(pl, ts[0])
    lay = Layout(ts[0], pl.layout.offsets)
    n = pl.layout.region_elems
    scale = 1.0 / W
    for r in range(W):
        world.launch(r, pls[r], KIND_PACK, ts[r], scale=scale)
    torch.cuda.synchronize()
    packed = [world.view(r, pl.data_off_bytes, n, wdt).clone() for r in range(W)]
    for r in range(W):
        check_packed("W=%d %s pack of rank %d" % (W, wire, r), packed[r], ts[r], lay, scale)
    ref = R.allreduce_ref(packed, wdt)
    world.clear_found_inf()
    world.arm_barriers(pl.grid, 2)
    for r in range(W):
        world.launch(r, pls[r], KIND_TWO_SHOT, ts[r], scale=scale, writeback=True, check_inf=True)
        torch.cuda.synchronize()
        check_owned_slice("W=%d %s slice of rank %d" % (W, wire, r), world.view(r, pl.data_off_bytes, n, wdt), ref, pl.layout, r)
        check_tensors("W=%d %s write-back of rank %d" % (W, wire, r), ts[r], lay, ref,
                      lambda pos, r=r: R.slice_owner(pl.layout, pos) == r)
    world.finish_round(pl.grid, 2)
    assert world.found_inf_all() == [0] * W


# ================================================================================================ K1b one-shot
def _oneshot_setup(W, wire, form):
    """"ddp": the engine's small-bucket form - fc.bias and every other 1-D ResNet-50 parameter plus the unaligned view,
    16 KiB CTA ranges, result in a separate gradient-arena slot.  "large": the whole ResNet-50 list over 256 KiB CTA
    ranges (the unrolled main loop), result in the plan's third region."""
    shapes = r50_shapes()
    if form == "ddp":
        shapes = [s for s in reversed(shapes) if len(s) == 1]
        bpc = 16 << 10
    else:
        bpc = 256 << 10
    ts0 = rank_tensors(shapes, 0)
    numels = numels_of(ts0)
    esz = P.WIRE_BYTES[wire]
    total = P.tensor_layout(numels)[1]
    world = EmulatedWorld(W, total * esz * 5 + (8 << 20))
    pls = world.plans(numels, wire, 3, bytes_per_cta=bpc)
    result_off = world.alloc(pls[0].region_bytes) if form == "ddp" else -1
    return world, pls, shapes, result_off


@pytest.mark.parametrize("form", ["ddp", "large"])
@pytest.mark.parametrize("wire", WIRES)
@pytest.mark.parametrize("W", WORLDS)
def test_oneshot_every_rank_bitwise_and_identical(W, wire, form):
    """Three consecutive calls (both staging halves) with new data each: every rank's result range and write-back equal
    the rank-order sum, so the ranks are bitwise equal to each other."""
    wdt = WIRE_DT[wire]
    esz = P.WIRE_BYTES[wire]
    world, pls, shapes, result_off = _oneshot_setup(W, wire, form)
    pl = pls[0]
    n = pl.layout.region_elems
    geo = R.oneshot_units(pl.layout, esz)
    assert pl.grid >= 2 and geo["tail_units"] > 0
    assert (geo["main_units"] > 0) == (form == "large"), geo
    res_off = result_off if result_off >= 0 else pl.data_off_bytes + 2 * pl.region_bytes
    scale = 1.0 / W
    for call in range(3):
        ts = [rank_tensors(shapes, r, seed=call + 1) for r in range(W)]
        if call == 0:
            assert_plan_reaches(pl, ts[0], straddle_slice=False)
            lay = Layout(ts[0], pl.layout.offsets)
        stage = pl.data_off_bytes + (call & 1) * pl.region_bytes
        for r in range(W):
            world.launch(r, pls[r], KIND_PACK, ts[r], scale=scale, data_off=stage)
        torch.cuda.synchronize()
        staged = [world.view(r, stage, n, wdt).clone() for r in range(W)]
        for r in range(W):
            check_packed("W=%d %s %s call %d staging of rank %d" % (W, wire, form, call, r), staged[r], ts[r], lay, scale)
        ref = R.allreduce_ref(staged, wdt)
        world.clear_found_inf()
        world.arm_barriers(pl.grid, 1)
        for r in range(W):
            world.launch(r, pls[r], KIND_ONE_SHOT, ts[r], scale=scale, writeback=True, check_inf=True, result_off=result_off)
        world.finish_round(pl.grid, 1)
        assert world.found_inf_all() == [0] * W
        for r in range(W):
            assert (pls[r].calls.cpu() == call + 1).all()
        results = [world.view(r, res_off, n, wdt) for r in range(W)]
        for r in range(W):
            R.assert_bits_equal("W=%d %s %s call %d result of rank %d" % (W, wire, form, call, r), results[r], ref)
            check_tensors("W=%d %s %s call %d write-back of rank %d" % (W, wire, form, call, r), ts[r], lay, ref)
        for r in range(1, W):
            R.assert_bits_equal("W=%d %s %s call %d rank %d vs rank 0" % (W, wire, form, call, r), results[r], results[0])


# ================================================================================================ found_inf
def _small_list():
    """A few ragged tensors over several CTAs (16 KiB ranges), fp32 sources."""
    return [torch.zeros(n, device=DEV) for n in (5000, 64, 3, 12289, 4096, 7, 20000)]


def _run_reduce(world, pls, kind, ts, wire, scale=1.0):
    """Pack (kind 3; for one-shot into the staging half of the call's parity) and one round of `kind` with the non-finite
    check."""
    pl = pls[0]
    stage = pl.data_off_bytes
    if kind == KIND_ONE_SHOT:
        stage += (int(pl.calls[0].item()) & 1) * pl.region_bytes
    for r in range(world.W):
        world.launch(r, pls[r], KIND_PACK, ts[r], scale=scale, data_off=stage)
    world.clear_found_inf()
    world.arm_barriers(pls[0].grid, 2 if kind == KIND_TWO_SHOT else 1)
    for r in range(world.W):
        world.launch(r, pls[r], kind, ts[r], scale=scale, check_inf=True)
    world.finish_round(pls[0].grid, 2 if kind == KIND_TWO_SHOT else 1)
    return world.found_inf_all()


@pytest.mark.parametrize("kind", [KIND_TWO_SHOT, KIND_ONE_SHOT], ids=["twoshot", "oneshot"])
@pytest.mark.parametrize("W", WORLDS)
def test_found_inf_reaches_every_rank(W, kind):
    """An inf or NaN in rank q's data inside a slice another rank owns sets found_inf on every rank; fp16 wire values
    40000 + 40000 overflow in the sum and set it; clean data leaves it 0."""
    base = _small_list()
    numels = numels_of(base)
    world = EmulatedWorld(W, 8 << 20)
    plans = {w: world.plans(numels, w, 3, bytes_per_cta=16 << 10) for w in ("fp32", "fp16")}
    pl = plans["fp32"][0]
    assert pl.grid >= 2
    g = torch.Generator(device=DEV).manual_seed(W)

    def clean():
        return [[(torch.randn(n, device=DEV, generator=g) * 0.1) for n in numels] for _ in range(W)]

    assert _run_reduce(world, plans["fp32"], kind, clean(), "fp32") == [0] * W
    for q, owner, val in ((W - 1, 0, math.inf), (0, W - 1, math.nan), (W // 2, (W // 2 + 1) % W, -math.inf)):
        ts = clean()
        # the first element of tensor 3 (12289 elements, crosses slices) that `owner` reduces
        t, lo = 3, pl.layout.offsets[3]
        own = R.slice_owner(pl.layout, torch.arange(lo, lo + numels[t], device=DEV))
        i = int(torch.nonzero(own == owner)[0])
        ts[q][t][i] = val
        got = _run_reduce(world, plans["fp32"], kind, ts, "fp32")
        assert got == [1] * W, "%r on rank %d in rank %d's slice: found_inf %s" % (val, q, owner, got)
    ts = clean()
    for r in range(W):
        ts[r][0][7] = 40000.0 if r in (0, W - 1) else 0.0
    got = _run_reduce(world, plans["fp16"], kind, ts, "fp16")
    assert got == [1] * W, "fp16 wire 40000 + 40000: found_inf %s" % got
    assert _run_reduce(world, plans["fp16"], kind, clean(), "fp16") == [0] * W


@pytest.mark.parametrize("W", [w for w in WORLDS if w >= 3])
def test_oneshot_overflow_decision_is_the_same_on_every_rank(W):
    """fp32 wire values 3e38, 3e38, -3e38 on ranks 0, 1, 2 (0 elsewhere): the rank-order sum overflows, so every rank
    must hold inf and skip the step.  A sum that starts at the caller's rank gives 3e38 on ranks 1 and 2."""
    numels = [3, 4096, 5000]
    world = EmulatedWorld(W, 4 << 20)
    pls = world.plans(numels, "fp32", 3, bytes_per_cta=16 << 10)
    assert pls[0].grid >= 2
    ts = [[torch.zeros(n, device=DEV) for n in numels] for _ in range(W)]
    for r, v in ((0, 3e38), (1, 3e38), (2, -3e38)):
        ts[r][2][4321] = v
    got = _run_reduce(world, pls, KIND_ONE_SHOT, ts, "fp32")
    assert got == [1] * W, "found_inf differs across ranks: %s" % got
    pos = pls[0].layout.offsets[2] + 4321
    n = pls[0].layout.region_elems
    vals = [world.view(r, pls[0].data_off_bytes + 2 * pls[0].region_bytes, n, F32)[pos].item() for r in range(W)]
    assert all(v == math.inf for v in vals), vals


# ================================================================================================ K2 broadcast
@pytest.mark.parametrize("wire", WIRES)
@pytest.mark.parametrize("W", WORLDS)
def test_broadcast_roots_and_parities(W, wire):
    """Root first, then the others, three calls per root (both halves): every non-root tensor is the root's wire value in
    its own dtype, every arena half holds the root's packed range, the root's tensors are unchanged."""
    wdt = WIRE_DT[wire]
    esz = P.WIRE_BYTES[wire]
    shapes = r50_shapes()
    ts0 = rank_tensors(shapes, 0)
    numels = numels_of(ts0)
    world = EmulatedWorld(W, P.tensor_layout(numels)[1] * esz * 2 + (8 << 20))
    pls = world.plans(numels, wire, 2)
    pl = pls[0]
    assert_plan_reaches(pl, ts0, straddle_slice=False)
    geo = R.push_units(pl.layout, esz)
    assert geo["main_units"] > 0 and geo["tail_units"] > 0, geo
    lay = Layout(ts0, pl.layout.offsets)
    n = pl.layout.region_elems
    call = 0
    for root in sorted({0, W - 1, W // 2}):
        for _ in range(3):
            ts = [rank_tensors(shapes, r, seed=10 + call) for r in range(W)]
            before = [t.clone() for t in ts[root]]
            half = pl.data_off_bytes + (call & 1) * pl.region_bytes
            world.arm_barriers(pl.grid, 1)
            for r in [root] + [q for q in range(W) if q != root]:
                world.launch(r, pls[r], KIND_BCAST, ts[r], root=root)
            world.finish_round(pl.grid, 1)
            call += 1
            assert all((p.calls.cpu() == call).all() for p in pls)
            rootv = world.view(root, half, n, wdt)
            check_packed("W=%d %s root %d packed" % (W, wire, root), rootv, before, lay, 1.0)
            for r in range(W):
                if r == root:
                    for i, (t, b) in enumerate(zip(ts[r], before)):
                        R.assert_bits_equal("root %d tensor %d unchanged" % (root, i), t, b)
                else:
                    R.assert_bits_equal("W=%d %s root %d arena of rank %d" % (W, wire, root, r), world.view(r, half, n, wdt), rootv)
                    check_tensors("W=%d %s root %d call %d rank %d" % (W, wire, root, call, r), ts[r], lay, rootv)


# ================================================================================================ kinds 3-6
@pytest.mark.parametrize("wire", WIRES)
@pytest.mark.parametrize("W", WORLDS)
def test_host_synchronised_kinds(W, wire):
    """DataParallel's flag-free kernels: pack on every rank, reduce-to-caller with write-back on rank 0 and on a middle
    rank (the same rank-order bits whoever calls); push from the last rank, unpack on the others."""
    wdt = WIRE_DT[wire]
    esz = P.WIRE_BYTES[wire]
    shapes = r50_shapes()
    numels = numels_of(rank_tensors(shapes, 0, seed=20))
    world = EmulatedWorld(W, P.tensor_layout(numels)[1] * esz + (8 << 20))
    pls = world.plans(numels, wire, 1)
    pl = pls[0]
    geo = R.loop_units(pl.layout.block_elems * esz // 16, R.REDUCE_U)
    assert pl.grid >= 2 and geo["main_units"] > 0 and geo["tail_units"] > 0, geo
    n = pl.layout.region_elems
    scale = 1.0 / W
    for k, caller in enumerate(sorted({0, W // 2})):
        ts = [rank_tensors(shapes, r, seed=20 + k) for r in range(W)]
        lay = Layout(ts[0], pl.layout.offsets)
        for r in range(W):
            world.launch(r, pls[r], KIND_PACK, ts[r], scale=scale)
        torch.cuda.synchronize()
        packed = [world.view(r, pl.data_off_bytes, n, wdt).clone() for r in range(W)]
        for r in range(W):
            check_packed("W=%d %s pack of rank %d" % (W, wire, r), packed[r], ts[r], lay, scale)
        ref = R.allreduce_ref(packed, wdt)
        world.launch(caller, pls[caller], KIND_REDUCE, ts[caller], writeback=True)
        torch.cuda.synchronize()
        R.assert_bits_equal("W=%d %s reduce to caller %d" % (W, wire, caller), world.view(caller, pl.data_off_bytes, n, wdt), ref)
        check_tensors("W=%d %s reduce write-back of caller %d" % (W, wire, caller), ts[caller], lay, ref)
        for r in range(W):
            if r != caller:
                R.assert_bits_equal("W=%d %s rank %d untouched" % (W, wire, r), world.view(r, pl.data_off_bytes, n, wdt), packed[r])
    root = W - 1
    src = rank_tensors(shapes, root, seed=21)
    world.launch(root, pls[root], KIND_PUSH, src)
    torch.cuda.synchronize()
    rootv = world.view(root, pl.data_off_bytes, n, wdt)
    check_packed("W=%d %s push" % (W, wire), rootv, src, lay, 1.0)
    for r in range(W - 1):
        world.launch(r, pls[r], KIND_UNPACK, ts[r])
    torch.cuda.synchronize()
    for r in range(W - 1):
        R.assert_bits_equal("W=%d %s pushed arena of rank %d" % (W, wire, r), world.view(r, pl.data_off_bytes, n, wdt), rootv)
        check_tensors("W=%d %s unpack of rank %d" % (W, wire, r), ts[r], lay, rootv)


# ================================================================================================ negative controls
def test_checkers_reject_wrong_results():
    """At W = 3, fp32 wire, from a real two-shot round: a correct arena with one element moved by 1 ulp, an arena whose
    slice of one rank was left unreduced, and the host-computed staggered-order result are each rejected."""
    W, wire, wdt = 3, "fp32", F32
    numels = [math.prod(s) for s in r50_shapes()[:40]]
    world = EmulatedWorld(W, 64 << 20)
    pls = world.plans(numels, wire, 1)
    pl = pls[0]
    n = pl.layout.region_elems
    data = []
    for r in range(W):
        v = world.view(r, pl.data_off_bytes, n, wdt)
        v.copy_(_rand(n, wdt, torch.Generator(device=DEV).manual_seed(r)))
        data.append(v.clone())
    ref = R.allreduce_ref(data, wdt)
    views = [world.view(r, pl.data_off_bytes, 8, wdt) for r in range(W)]
    world.arm_barriers(pl.grid, 2)
    for r in range(W):
        world.launch(r, pls[r], KIND_TWO_SHOT, [views[r]], prepacked=True)
    world.finish_round(pl.grid, 2)
    got = world.view(1, pl.data_off_bytes, n, wdt).clone()
    R.assert_bits_equal("correct", got, ref)
    bad = got.clone()
    bad[12345] = torch.nextafter(bad[12345], torch.tensor(math.inf, device=DEV))
    with pytest.raises(AssertionError, match="1 of"):
        R.assert_bits_equal("1 ulp", bad, ref)
    bad = got.clone()
    m = R.slice_owner(pl.layout, torch.arange(n, device=DEV)) == 2
    bad[m] = data[1][m]
    with pytest.raises(AssertionError, match="bitwise"):
        R.assert_bits_equal("slice of rank 2 unreduced", bad, ref)
    with pytest.raises(AssertionError, match="bitwise"):
        check_owned_slice("slice of rank 2 unreduced", bad, ref, pl.layout, 2)
    check_owned_slice("other slices", bad, ref, pl.layout, 0)
    for r in (1, 2):
        with pytest.raises(AssertionError, match="bitwise"):
            R.assert_bits_equal("staggered from rank %d" % r, R.staggered_ref(data, r), ref)


# ================================================================================================ K3 barrier
@pytest.mark.parametrize("W", WORLDS)
def test_barrier_flags_carry_every_rank_sequence(W):
    world = EmulatedWorld(W, 1 << 20)
    for _ in range(3):
        world.arm_barriers(1, 1)
        for r in range(W):
            world.arenas[r].launch_barrier(CH)
        world.finish_round(1, 1)
    assert (world.expect_seq[:1] == 3).all()


# ================================================================================================ LL kernels
@pytest.mark.parametrize("W", WORLDS)
def test_ll_allreduce_rank_order_bitwise(W):
    """Three calls (parities 1, 0, 1) with 3, 8 and 5 floats: after each rank runs, the words it wrote into every
    peer's inbox are {its value, seq}; its output is the rank-order fp32 sum times the scale, the same bits on every rank."""
    world = EmulatedWorld(W, 1 << 20)
    g = torch.Generator(device=DEV).manual_seed(W)
    for call, (nv, scale) in enumerate(((3, 1.0 / W), (8, 1.0), (5, 0.37))):
        ins = [_rand(nv, F32, g) for _ in range(W)]
        outs = [torch.full((nv,), math.nan, device=DEV) for _ in range(W)]
        seq = world.arm_inbox(nv, torch.stack(ins))
        par = seq & 1
        ref = R.ll_allreduce_ref(ins, scale)
        for r in range(W):
            world.arenas[r].launch_ll_allreduce(CH, ins[r], outs[r], scale)
            torch.cuda.synchronize()
            for dst in range(W):
                w = world.inbox(dst)[par, r, :nv]
                assert torch.equal(w[:, 0], ins[r].view(torch.int32)) and (w[:, 1] == seq).all(), "rank %d -> %d" % (r, dst)
            R.assert_bits_equal("W=%d call %d rank %d" % (W, call, r), outs[r], ref)
        world.finish_ll()


@pytest.mark.parametrize("W", WORLDS)
def test_metrics_cross_rank_mean(W):
    """metrics_kernel at world W: each rank's {loss, acc1, acc5} words in every inbox, out[3] = seq over three calls, and
    out[0:3] = the fp64 mean within the depth bound (batch 64: 100 k / 64 is exact in fp32)."""
    world = EmulatedWorld(W, 1 << 20)
    B, K = 64, 1000
    g = torch.Generator(device=DEV).manual_seed(W)
    for call in range(3):
        logits, targets, losses, vals = [], [], [], []
        for r in range(W):
            x = torch.randn(B, K, device=DEV, generator=g).to(BF16)
            t = torch.randint(0, K, (B,), device=DEV, generator=g)
            k = (5 * r + 3 * call) % B
            x[torch.arange(k, device=DEV), t[:k]] = 30.0
            loss = (torch.rand(1, device=DEV, generator=g) * 7).reshape(())
            top1, top5 = R.topk_correct_ref(x, t)
            logits.append(x)
            targets.append(t)
            losses.append(loss)
            vals.append([loss.item(), 100.0 * top1 / B, 100.0 * top5 / B])
        vals = torch.tensor(vals, dtype=torch.float32)
        seq = world.arm_inbox(3, vals)
        par = seq & 1
        for r in range(W):
            out = torch.full((4,), math.nan, device=DEV)
            world.arenas[r].launch_metrics(CH, logits[r], targets[r], losses[r], out)
            torch.cuda.synchronize()
            for dst in range(W):
                w = world.inbox(dst)[par, r, :3].cpu()
                assert torch.equal(w[:, 0], vals[r].view(torch.int32)) and (w[:, 1] == seq).all(), "rank %d -> %d" % (r, dst)
            assert out[3].item() == seq
            o = out[:3].cpu()
            ref, bound = R.metrics_mean_bound(vals, W, o)
            R.assert_within("W=%d call %d metrics of rank %d" % (W, call, r), o, ref, bound)
        world.finish_ll()
