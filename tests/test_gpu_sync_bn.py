"""Synchronised BatchNorm (``csrc/sync_bn.cu`` and the synchronised apply kernels) at world sizes 1 to 16, emulated on one
GPU, on every BatchNorm training path ResNet-50 takes.

Emulation (as in test_gpu_collectives_world.py).  One zeroed CUDA buffer holds W arenas; ``SymmArena.from_pointers``
builds W genuine contexts over it and each rank gets its own synchronised BatchNorm handle (exchange area at the same
offset, own call counters).  Ranks run one after another, never concurrently.

Safety rule: no kernel ever waits.  Before each exchange the harness computes every rank's local sums with the
unsynchronised op (the words each rank will publish), writes the LL words {value, seq} that a rank reads before their
owner has run (source >= destination) into every exchange area, and reads them back on the host before any launch; the
words of sources that run earlier must still be stale, so what the test sees there was stored by the kernel.

Checks per exchange: the published words equal the unsynchronised op's local sums and row count bit for bit; every rank
holds the rank-order fp32 sum of them and the integer global count; saved statistics, running statistics and
num_batches_tracked are the same bits on every rank; forward and backward outputs are within the tests/_fp64.py bounds
of BatchNorm over the concatenated global batch, dgamma / dbeta within the bounds of the rank-local sums (and the bits of
the unsynchronised op's).  At W = 1 the exchange reproduces the unsynchronised statistics and forward outputs bit for
bit; through the public op a one-rank world takes the unsynchronised kernels.  Negative controls: a staggered-order
sum and statistics normalised by the local count are rejected by the same checkers.
"""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _fp64 as R  # noqa: E402

from pytorch_distributed_b200.parallel import plan as P  # noqa: E402

pytestmark = pytest.mark.gpu

DEV = "cuda"
EPS, MOM = 1e-5, 0.1
WORLDS = [1, 2, 3, 4, 7, 8, 16]
BF16, F16, F32 = torch.bfloat16, torch.float16, torch.float32


def C():
    from pytorch_distributed_b200 import _ext
    return _ext.lib()


def sms() -> int:
    return torch.cuda.get_device_properties(0).multi_processor_count


class World:
    def __init__(self, W: int):
        M = C()
        self.W = W
        self.header = P.round_up(M.SIGNAL_PAD_BYTES, 128 << 10)
        self.R = P.round_up(self.header + M.SYNC_BN_AREA_BYTES, 1 << 16)
        self.buf = torch.zeros(W * self.R, dtype=torch.uint8, device=DEV)
        ptrs = [self.buf.data_ptr() + r * self.R for r in range(W)]
        self.arenas = [M.SymmArena.from_pointers(r, W, ptrs, 0, self.R, 0) for r in range(W)]
        self.calls = [torch.zeros(M.MAX_BLOCKS, dtype=torch.int32, device=DEV) for _ in range(W)]
        self.handles = [self.arenas[r].sync_bn(0, self.header, self.calls[r].data_ptr()) for r in range(W)]
        self.slot = 2 * M.SYNC_BN_MAX_C + 2
        self.seq = 0
        torch.cuda.synchronize()

    def words(self, r: int) -> torch.Tensor:
        lo = r * self.R + self.header
        return self.buf[lo:lo + C().SYNC_BN_AREA_BYTES].view(torch.int32).view(2, C().MAX_WORLD, self.slot, 2)

    @staticmethod
    def payload(local: torch.Tensor, count: int) -> torch.Tensor:
        return torch.cat([local.float().view(torch.int32), torch.tensor([count & 0xFFFFFFFF, count >> 32], dtype=torch.int64,
                                                                         device=DEV).to(torch.int32)])

    def exchange(self, local_fn, sync_fn):
        """local_fn(r) -> (local [2C] sums of the unsynchronised op, rows); sync_fn(r) -> (outputs, work slice)."""
        locals_ = [local_fn(r) for r in range(self.W)]
        torch.cuda.synchronize()
        seq, par = self.seq + 1, (self.seq + 1) & 1
        pays = [self.payload(l, m) for l, m in locals_]
        nw = pays[0].numel()
        for dst in range(self.W):
            w = self.words(dst)[par]
            for src in range(dst, self.W):
                w[src, :nw, 0] = pays[src]
                w[src, :nw, 1] = seq
        torch.cuda.synchronize()
        for dst in range(self.W):
            w = self.words(dst)[par].cpu()
            assert all(torch.equal(w[s, :nw, 0], pays[s].cpu()) and (w[s, :nw, 1] == seq).all() for s in range(dst, self.W))
            assert (w[:dst, :nw, 1] != seq).all(), "words of ranks that have not run already carry the sequence"
            assert (self.calls[dst] == self.seq).all()
        outs = [sync_fn(r) for r in range(self.W)]
        torch.cuda.synchronize()
        self.seq = seq
        for dst in range(self.W):
            w = self.words(dst)[par]
            for src in range(self.W):
                assert torch.equal(w[src, :nw, 0], pays[src]) and (w[src, :nw, 1] == seq).all(), "published words"
            assert (self.calls[dst] == seq).all(), "call counters"
            assert self.arenas[dst].status() == 0
        c2 = locals_[0][0].numel()
        ref = rank_order_sum([l for l, _ in locals_])
        total = sum(m for _, m in locals_)
        for r, (_, work) in enumerate(outs):
            assert torch.equal(work[:c2], locals_[r][0]), "local sums differ from the unsynchronised op"
            assert torch.equal(work[c2:2 * c2], ref), "global sums are not the rank-order fp32 sum"
            assert int(work[2 * c2:2 * c2 + 2].view(torch.int64).item()) == total, "global count"
        return [o for o, _ in outs], ref, total


def rank_order_sum(vals):
    g = torch.zeros_like(vals[0])
    for v in vals:
        g = g + v
    return g


def staggered_sum(vals, start=1):
    g = torch.zeros_like(vals[0])
    for k in range(len(vals)):
        g = g + vals[(start + k) % len(vals)]
    return g


def sync_work(c: int) -> torch.Tensor:
    return torch.zeros(4 * c + 4, dtype=F32, device=DEV)


def rank_rows(W: int, base: int):
    """per-rank batch sizes that differ between ranks"""
    return [base + (r % 3) for r in range(W)]


def act(n, c, hw, dt, seed, offset=0.5):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(n, c, hw, hw, device=DEV, generator=g) * 2 + offset
    return x.to(dt).contiguous(memory_format=torch.channels_last)


def params(c, wdt, seed=7):
    g = torch.Generator(device=DEV).manual_seed(seed)
    w = (torch.rand(c, device=DEV, generator=g) + 0.5).to(wdt)
    b = (torch.randn(c, device=DEV, generator=g) * 0.2).to(wdt)
    return w, b


def assert_same_bits(name, ts):
    assert all(torch.equal(t, ts[0]) for t in ts), name + " differs across ranks"


def depth(rows_per_rank, c, W):
    return max(R.bn_depth(m, c, sms()) for m in rows_per_rank) + W


# ================================================================================================ bn_act forward / backward
def _bn_forward_world(world, xs, w, b, relu, res):
    M = C()
    c = xs[0].size(1)
    st0 = [(torch.zeros(c, device=DEV), torch.ones(c, device=DEV), torch.zeros((), dtype=torch.int64, device=DEV)) for _ in xs]

    def local(r):
        work = torch.zeros(2 * c, device=DEV)
        rm, rv, nb = (t.clone() for t in st0[r])
        M.bn_act_forward(xs[r], res[r] if res else None, w, b, rm, rv, nb, True, MOM, EPS, relu, True, work, False)
        return work, xs[r].numel() // c

    def sync(r):
        work = sync_work(c)
        rm, rv, nb = st0[r]
        y, saved, mask = M.bn_act_forward(xs[r], res[r] if res else None, w, b, rm, rv, nb, True, MOM, EPS, relu, True, work, False,
                                          world.handles[r])
        return (y, saved, mask, rm, rv, nb), work

    return world.exchange(local, sync)


@pytest.mark.parametrize("W", WORLDS)
@pytest.mark.parametrize("dt,c,hw,relu,res", [(BF16, 256, 56, True, True), (F16, 64, 56, True, False), (F32, 512, 28, False, True),
                                              (BF16, 2048, 7, True, True)])
def test_bn_act_forward_backward(W, dt, c, hw, relu, res):
    M = C()
    world = World(W)
    rows = rank_rows(W, 2 if hw >= 56 else 4)
    xs = [act(n, c, hw, dt, 100 + r) for r, n in enumerate(rows)]
    rs = [act(n, c, hw, dt, 200 + r, 0.0) for r, n in enumerate(rows)] if res else None
    w, b = params(c, F32 if dt == F32 else dt)
    outs, gsum, total = _bn_forward_world(world, xs, w, b, relu, rs)
    ys, saved, masks, rms, rvs, nbs = zip(*outs)
    for name, ts in (("saved", saved), ("running_mean", rms), ("running_var", rvs), ("num_batches_tracked", nbs)):
        assert_same_bits(name, ts)
    assert int(nbs[0]) == 1
    xg = torch.cat([R.rows(x) for x in xs])
    d = depth([x.numel() // c for x in xs], c, W)
    st = R.check_stats("sync fwd", saved[0], xg, d, EPS)
    R.check_running("sync fwd", rms[0], rvs[0], torch.zeros(c, device=DEV), torch.ones(c, device=DEV), st, MOM)
    for r in range(W):
        R.check_bn_forward("sync fwd rank %d" % r, ys[r], masks[r], R.rows(xs[r]), saved[r][:c], saved[r][c:], w, b,
                           R.rows(rs[r]) if res else None, relu, max_band=1e-2)
    if W == 1:                       # the synchronised path of a single rank is the unsynchronised op, bit for bit
        rm, rv, nb = torch.zeros(c, device=DEV), torch.ones(c, device=DEV), torch.zeros((), dtype=torch.int64, device=DEV)
        y1, s1, m1 = M.bn_act_forward(xs[0], rs[0] if res else None, w, b, rm, rv, nb, True, MOM, EPS, relu, True,
                                      torch.zeros(2 * c, device=DEV), False)
        assert torch.equal(y1, ys[0]) and torch.equal(s1, saved[0]) and torch.equal(rm, rms[0]) and torch.equal(rv, rvs[0])
        assert (m1 is None and masks[0] is None) or torch.equal(m1, masks[0])
    else:                            # negative control: statistics normalised by the local count are rejected
        n0 = xs[0].numel() // c
        mean = gsum[:c] / n0
        fake = torch.cat([mean, torch.rsqrt((gsum[c:] / n0 - mean * mean).clamp_min(0) + EPS)])
        with pytest.raises(AssertionError):
            R.check_stats("local count", fake, xg, d, EPS)

    # ---- backward (plain and split residual gradient), from the forward's global statistics
    dys = [act(n, c, hw, dt, 300 + r, 0.0) for r, n in enumerate(rows)]
    dy2 = [act(n, c, hw, dt, 400 + r, 0.0) for r, n in enumerate(rows)]
    for split in (False, True):
        def local(r):
            work = torch.zeros(2 * c, device=DEV)
            if split:
                M.bn_act_backward2(dys[r], dy2[r], xs[r], masks[r], w, saved[r], relu, work)
            else:
                M.bn_act_backward(dys[r], xs[r], masks[r], w, saved[r], relu, bool(res), work)
            return work, xs[r].numel() // c

        def sync(r):
            work = sync_work(c)
            if split:
                out = M.bn_act_backward2(dys[r], dy2[r], xs[r], masks[r], w, saved[r], relu, work, world.handles[r])
            else:
                out = M.bn_act_backward(dys[r], xs[r], masks[r], w, saved[r], relu, bool(res), work, world.handles[r])
            return out, work

        outs, gsum_b, _ = world.exchange(local, sync)
        name = "sync bwd%s" % ("2" if split else "")
        dzs = []
        for r in range(W):
            dz = R.rows(dys[r]).double()
            if split:
                dz = R.rows((dys[r].float() + dy2[r].float()).to(dt)).double()
            if relu:
                dz = dz * R.unpack_mask(masks[r], dz.size(0), c)
            dzs.append(dz)
        ref = R.bn_backward_ref(torch.cat(dzs), xg, saved[0][:c], saved[0][c:], w, d)
        lo = 0
        for r in range(W):
            dx, dw, db = outs[r][0], outs[r][-2], outs[r][-1]
            m = dzs[r].size(0)
            R.assert_within(name + " dx rank %d" % r, R.rows(dx), ref["dx"][lo:lo + m],
                            0.5 * R.ulp(R.rows(dx), dt) + ref["dx_bound"][lo:lo + m])
            loc = R.bn_backward_ref(dzs[r], R.rows(xs[r]), saved[0][:c], saved[0][c:], w, d)
            R.assert_within(name + " dgamma (rank-local) %d" % r, dw, loc["dgamma"], 0.5 * R.ulp(dw, dw.dtype) + loc["dgamma_bound"])
            R.assert_within(name + " dbeta (rank-local) %d" % r, db, loc["dbeta"], 0.5 * R.ulp(db, db.dtype) + loc["dbeta_bound"])
            lo += m
        if W == 1:
            work = torch.zeros(2 * c, device=DEV)
            if split:
                o1 = M.bn_act_backward2(dys[0], dy2[0], xs[0], masks[0], w, saved[0], relu, work)
            else:
                o1 = M.bn_act_backward(dys[0], xs[0], masks[0], w, saved[0], relu, bool(res), work)
            # dgamma / dbeta are stored from the same local sums; dx goes through the synchronised apply kernel, whose
            # multiply-adds the compiler may contract differently: it is held to the fp64 bounds above
            assert torch.equal(o1[-2], outs[0][-2]) and torch.equal(o1[-1], outs[0][-1])


# ================================================================================================ GEMM statistics paths
@pytest.mark.parametrize("W", WORLDS)
@pytest.mark.parametrize("dt,k,n,hw", [(BF16, 256, 64, 56), (F16, 512, 128, 28), (BF16, 1024, 2048, 7)])
def test_conv1x1_bnstats_then_apply(W, dt, k, n, hw):
    M = C()
    world = World(W)
    rows = rank_rows(W, 2 if hw >= 56 else 4)
    xs = [act(b, k, hw, dt, 500 + r, 0.0) for r, b in enumerate(rows)]
    g = torch.Generator(device=DEV).manual_seed(9)
    wt = (torch.randn(n, k, 1, 1, device=DEV, generator=g) / k ** 0.5).to(dt)
    w, b = params(n, dt)
    ys = {}

    def local(r):
        gs = torch.zeros(2 * n, device=DEV)
        ys[r] = M.conv1x1_bnstats(xs[r], wt, gs)
        return gs, ys[r].numel() // n

    def sync(r):
        work = sync_work(n)
        y = M.conv1x1_bnstats(xs[r], wt, work, world.handles[r])
        assert torch.equal(y, ys[r]), "the synchronised GEMM must store the same output"
        return (y, work), work

    outs, gsum, total = world.exchange(local, sync)
    rm = [torch.zeros(n, device=DEV) for _ in range(W)]
    rv = [torch.ones(n, device=DEV) for _ in range(W)]
    nb = [torch.zeros((), dtype=torch.int64, device=DEV) for _ in range(W)]
    saved, yapp = [], []
    for r, (y, work) in enumerate(outs):   # the apply pass reads the exchanged slice (stats_ready): no second exchange
        ya, sv, _ = M.bn_act_forward(y, None, w, b, rm[r], rv[r], nb[r], True, MOM, EPS, True, False, work, True, world.handles[r])
        saved.append(sv)
        yapp.append(ya)
    assert all((cl == world.seq).all() for cl in world.calls)
    if W == 1:
        r0m, r0v = torch.zeros(n, device=DEV), torch.ones(n, device=DEV)
        gs = torch.zeros(2 * n, device=DEV)
        y1 = M.conv1x1_bnstats(xs[0], wt, gs)
        _, s1, _ = M.bn_act_forward(y1, None, w, b, r0m, r0v, None, True, MOM, EPS, True, False, gs, True)
        assert torch.equal(s1, saved[0]) and torch.equal(r0v, rv[0])
    assert_same_bits("saved", saved)
    assert_same_bits("running_var", rv)
    yg = torch.cat([R.rows(y) for y, _ in outs])
    geo = R.gemm_geometry(max(rows) * hw * hw, n, k, sms())
    R.check_stats("gemm sync", saved[0], yg, geo["depth"] + W, EPS)
    for r, (y, _) in enumerate(outs):       # the apply output, normalised with the global statistics
        R.check_bn_forward("gemm sync rank %d" % r, yapp[r], None, R.rows(y), saved[r][:n], saved[r][n:], w, b, None, True)


# ================================================================================================ stem
@pytest.mark.parametrize("W", WORLDS)
@pytest.mark.parametrize("dt", [BF16, F16, F32])
def test_stem_forward_backward(W, dt):
    from test_gpu_fp64 import check_stem_forward
    M = C()
    world = World(W)
    c, hw = 64, 112
    rows = rank_rows(W, 1)
    x64, scale = R.tie_free_stem_input(sum(rows), c, hw, hw, device=DEV, seed=W)   # no ties in any pooling window
    w, _ = params(c, F32 if dt == F32 else dt)
    b = R.stem_bias_between_levels(x64, scale, w, EPS).to(w.dtype)      # from the GLOBAL batch's statistics
    xs = list(x64.to(dt).contiguous(memory_format=torch.channels_last).split(rows))
    xs = [x.contiguous(memory_format=torch.channels_last) for x in xs]
    del x64
    st0 = [(torch.zeros(c, device=DEV), torch.ones(c, device=DEV), torch.zeros((), dtype=torch.int64, device=DEV)) for _ in xs]

    def local(r):
        work = torch.zeros(2 * c, device=DEV)
        rm, rv, nb = (t.clone() for t in st0[r])
        M.stem_forward(xs[r], w, b, rm, rv, nb, True, MOM, EPS, True, work)
        return work, xs[r].numel() // c

    def sync(r):
        work = sync_work(c)
        rm, rv, nb = st0[r]
        y, saved, code = M.stem_forward(xs[r], w, b, rm, rv, nb, True, MOM, EPS, True, work, world.handles[r])
        return (y, saved, code, rm, rv, nb), work

    outs, gsum, total = world.exchange(local, sync)
    ys, saved, codes, rms, rvs, nbs = zip(*outs)
    for name, ts in (("saved", saved), ("running_mean", rms), ("running_var", rvs), ("num_batches_tracked", nbs)):
        assert_same_bits(name, ts)
    xg = torch.cat([R.rows(x) for x in xs])
    d = depth([x.numel() // c for x in xs], c, W)
    st = R.check_stats("stem sync", saved[0], xg, d, EPS)
    R.check_running("stem sync", rms[0], rvs[0], torch.zeros(c, device=DEV), torch.ones(c, device=DEV), st, MOM)
    crefs = [check_stem_forward("stem sync rank %d" % r, xs[r], w, b, ys[r], saved[r], codes[r]) for r in range(W)]
    if W == 1:
        rm, rv, nb = torch.zeros(c, device=DEV), torch.ones(c, device=DEV), torch.zeros((), dtype=torch.int64, device=DEV)
        o1 = M.stem_forward(xs[0], w, b, rm, rv, nb, True, MOM, EPS, True, torch.zeros(2 * c, device=DEV))
        assert all(torch.equal(a, b_) for a, b_ in zip(o1, outs[0][:3]))
    g = torch.Generator(device=DEV).manual_seed(11)
    dps = [(torch.randint(-8, 9, y.shape, device=DEV, generator=g) / 8).to(dt).contiguous(memory_format=torch.channels_last) for y in ys]

    def local_b(r):
        work = torch.zeros(2 * c, device=DEV)
        M.stem_backward(dps[r], xs[r], codes[r], w, saved[r], work)
        return work, xs[r].numel() // c

    def sync_b(r):
        work = sync_work(c)
        return M.stem_backward(dps[r], xs[r], codes[r], w, saved[r], work, world.handles[r]), work

    outs_b, gsum_b, _ = world.exchange(local_b, sync_b)
    dzs = [R.rows(R.stem_dz_ref(dps[r], crefs[r], hw, hw)) for r in range(W)]
    bd = max(R.stem_bwd_geometry(n, c, hw, hw, sms())["depth"] for n in rows) + W
    ref = R.bn_backward_ref(torch.cat(dzs), xg, saved[0][:c], saved[0][c:], w, bd)      # dx from the GLOBAL sums and count
    lo = 0
    for r in range(W):
        dx, dw, db = outs_b[r]
        m = dzs[r].size(0)
        R.assert_within("stem sync dx rank %d" % r, R.rows(dx), ref["dx"][lo:lo + m], 0.5 * R.ulp(R.rows(dx), dt) + ref["dx_bound"][lo:lo + m])
        loc = R.bn_backward_ref(dzs[r], R.rows(xs[r]), saved[0][:c], saved[0][c:], w, bd)
        R.assert_within("stem sync dgamma (rank-local) %d" % r, dw, loc["dgamma"], 0.5 * R.ulp(dw, dw.dtype) + loc["dgamma_bound"])
        R.assert_within("stem sync dbeta (rank-local) %d" % r, db, loc["dbeta"], 0.5 * R.ulp(db, db.dtype) + loc["dbeta_bound"])
        single = M.stem_backward(dps[r], xs[r], codes[r], w, saved[r], torch.zeros(2 * c, device=DEV))
        assert torch.equal(single[1], dw) and torch.equal(single[2], db), "dgamma / dbeta must be the rank-local sums"
        lo += m


@pytest.mark.parametrize("W", WORLDS)
@pytest.mark.parametrize("dt", [BF16, F16])
def test_stem_gemm_then_stem_forward_pre(W, dt):
    from pytorch_distributed_b200.ops.stem_conv import K_PAD, pack_stem_weight
    M = C()
    world = World(W)
    rows = rank_rows(W, 1)
    imgs = [act(n, 3, 224, dt, 800 + r, 0.0) for r, n in enumerate(rows)]
    g = torch.Generator(device=DEV).manual_seed(3)
    wc = (torch.randn(64, 3, 7, 7, device=DEV, generator=g) * 0.1).to(dt)
    packed = pack_stem_weight(wc).view(64, K_PAD, 1, 1)
    a = [M.stem_im2col(x) for x in imgs]
    ys = {}

    def local(r):
        gs = torch.zeros(128, device=DEV)
        ys[r] = M.conv1x1_bnstats(a[r], packed, gs)
        return gs, ys[r].numel() // 64

    def sync(r):
        work = sync_work(64)
        y = M.conv1x1_bnstats(a[r], packed, work, world.handles[r])
        return (y, work), work

    outs, gsum, total = world.exchange(local, sync)
    w, b = params(64, dt)
    saved, rvs, pooled = [], [], []
    for r, (y, work) in enumerate(outs):
        assert torch.equal(y, ys[r])
        rm, rv, nb = torch.zeros(64, device=DEV), torch.ones(64, device=DEV), torch.zeros((), dtype=torch.int64, device=DEV)
        yp, s, _ = M.stem_forward_pre(y, w, b, rm, rv, nb, True, MOM, EPS, True, work, world.handles[r])
        saved.append(s)
        rvs.append(rv)
        pooled.append(yp)
    assert_same_bits("saved", saved)
    assert_same_bits("running_var", rvs)
    yg = torch.cat([R.rows(ys[r]) for r in range(W)])
    geo = R.gemm_geometry(max(rows) * 112 * 112, 64, K_PAD, sms())
    R.check_stats("stem gemm sync", saved[0], yg, geo["depth"] + W, EPS)
    for r in range(W):                       # pooled output with the global statistics (1 ulp + the apply bound)
        yref, _, e_sel, _ = R.stem_forward_ref(ys[r], saved[r][:64], saved[r][64:], w, b)
        R.assert_within("stem gemm sync y rank %d" % r, pooled[r], yref, R.ulp(yref, dt) + e_sel)


# ================================================================================================ controls
def test_rank_order_checker_rejects_staggered_sum():
    g = torch.Generator(device=DEV).manual_seed(1)
    vals = [torch.randn(4096, device=DEV, generator=g) * 2.0 ** float(k % 7) for k in range(7)]
    assert not torch.equal(staggered_sum(vals), rank_order_sum(vals))


# ================================================================================================ public op
def test_public_op_world1_is_the_unsynchronised_op():
    """A one-rank world takes today's path: the handle is dropped and the outputs are the unsynchronised op's bits."""
    from pytorch_distributed_b200.ops.bn_act import bn_act
    from pytorch_distributed_b200.ops.sync_bn import SyncContext

    class _Comm:
        world = 1

    c = 256
    x = act(4, c, 14, BF16, 5).requires_grad_(True)
    w, b = params(c, F32)
    outs = []
    for sync in (None, SyncContext(_Comm(), None, None)):
        xx = x.detach().clone().requires_grad_(True)
        ww, bb = w.clone().requires_grad_(True), b.clone().requires_grad_(True)
        rm, rv = torch.zeros(c, device=DEV), torch.ones(c, device=DEV)
        y = bn_act(xx, ww, bb, rm, rv, relu=True, training=True, sync=sync)
        y.backward(act(4, c, 14, BF16, 6, 0.0))
        outs.append((y, xx.grad, ww.grad, bb.grad, rm, rv))
    assert all(torch.equal(a, b_) for a, b_ in zip(*outs))


class _Comm:
    def __init__(self, world):
        self.world = world


def _sync_layer(c, ctx, relu=True):
    from pytorch_distributed_b200.models.resnet import SyncBNAct
    layer = SyncBNAct(c, relu=relu).to(DEV)
    layer._sync = ctx                        # bound to this emulated rank's handle, as at a first training forward
    return layer


@pytest.mark.parametrize("W", [2, 3, 8])
@pytest.mark.parametrize("op", ["bn_act", "conv1x1_bn_act", "bn_relu_maxpool", "stem_conv_bn_relu_maxpool"])
def test_public_ops_forward_backward(W, op):
    """Each public op with ``sync=`` (or a synchronised layer) under the armed exchange, forward and backward: the
    exchange of the op's own workspace slice is checked bit for bit, the statistics against fp64 over the global batch,
    the input gradient of ``bn_act`` against fp64 and the BatchNorm weight gradients against the rank-local sums."""
    from pytorch_distributed_b200.ops.bn_act import bn_act, workspace
    from pytorch_distributed_b200.ops.conv_bn import conv1x1_bn_act
    from pytorch_distributed_b200.ops.stem import bn_relu_maxpool
    from pytorch_distributed_b200.ops.stem_conv import K_PAD, pack_stem_weight, stem_conv_bn_relu_maxpool
    from pytorch_distributed_b200.ops.sync_bn import SyncContext, sync_work_len
    M = C()
    world = World(W)
    ws = workspace(torch.device(DEV, 0))
    ws.reset()
    ctxs = [SyncContext(_Comm(W), world.handles[r], world.calls[r]) for r in range(W)]
    rows = rank_rows(W, 2)
    g = torch.Generator(device=DEV).manual_seed(21)
    if op == "bn_act":
        c, inputs = 256, [act(n, 256, 14, BF16, 40 + r).requires_grad_(True) for r, n in enumerate(rows)]
    elif op == "conv1x1_bn_act":
        c, inputs = 128, [act(n, 256, 28, BF16, 40 + r, 0.0).requires_grad_(True) for r, n in enumerate(rows)]
        convs = [torch.nn.Conv2d(256, 128, 1, bias=False).to(DEV, BF16).to(memory_format=torch.channels_last) for _ in range(W)]
        for cv in convs:
            cv.weight.data.copy_(convs[0].weight.data)
    elif op == "bn_relu_maxpool":
        c, inputs = 64, [act(n, 64, 56, BF16, 40 + r).requires_grad_(True) for r, n in enumerate(rows)]
    else:
        c, inputs = 64, [act(n, 3, 64, BF16, 40 + r, 0.0) for r, n in enumerate(rows)]
        convs = [torch.nn.Conv2d(3, 64, 7, 2, 3, bias=False).to(DEV, BF16) for _ in range(W)]
        for cv in convs:
            cv.weight.data.copy_(convs[0].weight.data)
    layers = [_sync_layer(c, ctxs[r]) for r in range(W)]
    for ly in layers:
        ly.weight.data.copy_(torch.rand(c, device=DEV, generator=torch.Generator(device=DEV).manual_seed(5)) + 0.5)
    wl = sync_work_len(c)
    offs, outs = {}, {}

    def run(r):
        ly, x = layers[r], inputs[r]
        offs[r] = ws.used
        if op == "bn_act":
            return bn_act(x, ly.weight, ly.bias, ly.running_mean, ly.running_var, relu=True, training=True,
                          num_batches_tracked=ly.num_batches_tracked, sync=ctxs[r])
        if op == "conv1x1_bn_act":
            return conv1x1_bn_act(x, convs[r], ly)
        if op == "bn_relu_maxpool":
            return bn_relu_maxpool(x, ly.weight, ly.bias, ly.running_mean, ly.running_var, training=True,
                                   num_batches_tracked=ly.num_batches_tracked, sync=ctxs[r])
        return stem_conv_bn_relu_maxpool(x, convs[r], ly)

    def bn_input(r):                          # what the op's BatchNorm normalised (its own saved input)
        return outs[r].grad_fn.saved_tensors[0]

    def local_f(r):
        x = inputs[r].detach()
        gs = torch.zeros(2 * c, device=DEV)
        rm, rv = torch.zeros(c, device=DEV), torch.ones(c, device=DEV)
        if op == "bn_act":
            M.bn_act_forward(x, None, layers[r].weight, layers[r].bias, rm, rv, None, True, MOM, EPS, True, False, gs, False)
        elif op == "conv1x1_bn_act":
            M.conv1x1_bnstats(x, convs[r].weight, gs)
        elif op == "bn_relu_maxpool":
            M.stem_forward(x, layers[r].weight, layers[r].bias, rm, rv, None, True, MOM, EPS, False, gs)
        else:
            a = M.stem_im2col(x)
            M.conv1x1_bnstats(a, pack_stem_weight(convs[r].weight).view(64, K_PAD, 1, 1), gs)
        return gs

    def count(r):
        if op in ("bn_act", "bn_relu_maxpool"):
            return inputs[r].numel() // c
        if op == "conv1x1_bn_act":
            return inputs[r].numel() // 256
        return rows[r] * 32 * 32                # 7x7 / 2 over 64 x 64

    def sync_f(r):
        outs[r] = run(r)
        return outs[r], ws.buf[offs[r]:offs[r] + wl]

    world.exchange(lambda r: (local_f(r), count(r)), sync_f)
    saved = [bn_input(r) for r in range(W)]
    sv = [outs[r].grad_fn.saved_tensors[3] for r in range(W)]
    assert_same_bits("saved", sv)
    assert_same_bits("running_var", [ly.running_var for ly in layers])
    assert all(int(ly.num_batches_tracked) == 1 for ly in layers)
    xg = torch.cat([R.rows(t) for t in saved])
    if op == "conv1x1_bn_act":
        d = R.gemm_geometry(max(rows) * 28 * 28, 128, 256, sms())["depth"] + W
    elif op == "stem_conv_bn_relu_maxpool":
        d = R.gemm_geometry(max(rows) * 32 * 32, 64, K_PAD, sms())["depth"] + W
    else:
        d = depth([t.numel() // c for t in saved], c, W)
    R.check_stats(op + " sync", sv[0], xg, d, EPS)

    dys = [(torch.randint(-8, 9, outs[r].shape, device=DEV, generator=g) / 8).to(BF16).contiguous(memory_format=torch.channels_last)
           for r in range(W)]
    locals_b, masks = {}, {}

    def local_b(r):
        t = outs[r].grad_fn.saved_tensors
        masks[r] = t[1]
        gs = torch.zeros(2 * c, device=DEV)
        if op in ("bn_act", "conv1x1_bn_act"):
            locals_b[r] = M.bn_act_backward(dys[r], t[0], t[1], t[2], t[3], True, False, gs)
        else:
            locals_b[r] = M.stem_backward(dys[r], t[0], t[1], t[2], t[3], gs)
        return gs, t[0].numel() // c

    def sync_b(r):
        outs[r].backward(dys[r])
        return None, ws.buf[offs[r] + wl:offs[r] + 2 * wl]

    world.exchange(local_b, sync_b)
    for r in range(W):
        assert torch.equal(layers[r].weight.grad, locals_b[r][-2].to(layers[r].weight.dtype)), "dgamma must be rank-local"
        assert torch.equal(layers[r].bias.grad, locals_b[r][-1].to(layers[r].bias.dtype)), "dbeta must be rank-local"
    if op == "bn_act":                        # input gradient through the global sums
        dzs = [R.rows(dys[r]).double() * R.unpack_mask(masks[r], inputs[r].numel() // c, c) for r in range(W)]
        d = depth([x.numel() // c for x in inputs], c, W)
        ref = R.bn_backward_ref(torch.cat(dzs), xg, sv[0][:c], sv[0][c:], layers[0].weight, d)
        lo = 0
        for r in range(W):
            m = dzs[r].size(0)
            got = R.rows(inputs[r].grad)
            R.assert_within("bn_act public dx rank %d" % r, got, ref["dx"][lo:lo + m], 0.5 * R.ulp(got, BF16) + ref["dx_bound"][lo:lo + m])
            lo += m
