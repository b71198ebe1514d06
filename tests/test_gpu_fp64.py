"""The 1x1-conv wgmma GEMM, the fused BatchNorm and the fused stem kernels against float64 references (tests/_fp64.py)
at ResNet-50 batch-256 training shapes and at the geometry edges of their launch arithmetic.

Every case calls the extension entry points directly.  Shapes that pick a branch of the launch geometry are derived from
the device's SM count, and the branch is asserted through the Python mirrors in _fp64.  Each checker also has a negative
control: a correct kernel result edited after the fact must be rejected.  The reduction kernels write per-CTA partial
rows that combine_partials adds in a fixed order, so a second call with the same inputs must give the same bits.
"""
import os
import subprocess
import sys

import pytest
import torch

TESTS = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, TESTS)
import _fp64 as R  # noqa: E402

pytestmark = pytest.mark.gpu

CL = torch.channels_last
EPS = 1e-5
DEV = "cuda"


def lib():
    from pytorch_distributed_b200 import _ext
    return _ext.lib()


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _equal_all(a, b):
    return all((x is None and y is None) or torch.equal(x, y) for x, y in zip(a, b))


# ================================================================================================ conv1x1_bnstats
def _gemm_inputs(B, K, N, H, W, seed=0):
    g = _gen(seed)
    x = torch.randn(B, K, H, W, device=DEV, generator=g).bfloat16().contiguous(memory_format=CL)
    w = (torch.randn(N, K, 1, 1, device=DEV, generator=g) * K ** -0.5).bfloat16()
    base = torch.randn(2 * N, device=DEV, generator=g) * 64      # gsum accumulates: start from nonzero sums
    base[N:] = base[N:].abs()
    return x, w, base


def _gemm_run(x, w, base):
    gs = base.clone()
    y = lib().conv1x1_bnstats(x, w, gs)
    return y, gs


def _gemm_check(x, w, base, y, gs, geo):
    R.check_conv1x1(y, x, w)
    R.check_sums("gemm_bnstats", gs, R.rows(y), geo["depth"], base)


# (C_in -> C_out, H = W) of every stride-1 1x1 convolution of ResNet-50, and the stem GEMM (im2col K = 192)
RESNET50_1X1 = [(64, 64, 56), (64, 256, 56), (256, 64, 56), (256, 128, 28), (512, 128, 28), (128, 512, 28), (512, 256, 14),
                (1024, 256, 14), (256, 1024, 14), (1024, 512, 7), (2048, 512, 7), (512, 2048, 7), (192, 64, 112)]


@pytest.mark.parametrize("k,n,hw", RESNET50_1X1, ids=["%d-%d@%d" % s for s in RESNET50_1X1])
def test_conv1x1_bnstats_resnet50_batch256(k, n, hw):
    x, w, base = _gemm_inputs(256, k, n, hw, hw)
    M = 256 * hw * hw
    geo = R.gemm_geometry(M, n, k, sms())
    assert geo["max_tiles_per_cta"] > 1            # the TMA ring, the staging tile and the sums run across several m-tiles
    y, gs = _gemm_run(x, w, base)
    _gemm_check(x, w, base, y, gs, geo)
    assert _equal_all((y, gs), _gemm_run(x, w, base))


# (name, K, N, M as a function of the SM count and the n-tile count)
GEMM_EDGES = [
    ("m%%128=%d" % r, 128, 256, (lambda s, nt, r=r: 128 * (2 * s + 3) + r)) for r in (1, 63, 64, 65, 127)
] + [
    # m_tiles = sms / n_tiles + 1: exactly one CTA per n-tile takes a second m-tile (the smallest is the memcheck case)
    ("one_cta_second_tile_n64", 64, 64, lambda s, nt: 128 * s + 1),
    ("one_cta_second_tile_n768", 128, 768, lambda s, nt: 128 * (s // nt) + 64),
] + [
    # several n-tiles of each BLOCK_N; K = 64 gives one k-block per tile, so the stage parity flips on every tile
    ("n%d_k64" % n, 64, n, lambda s, nt: 128 * 4 * s + 65) for n in (192, 320, 384, 768)
]


@pytest.mark.parametrize("name,k,n,m_of", GEMM_EDGES, ids=[e[0] for e in GEMM_EDGES])
def test_conv1x1_bnstats_geometry_edges(name, k, n, m_of):
    nt = R.gemm_geometry(128, n, k, sms())["n_tiles"]
    M = m_of(sms(), nt)
    geo = R.gemm_geometry(M, n, k, sms())
    if name.startswith("m%"):
        assert M % 128 == int(name.split("=")[1]) and geo["max_tiles_per_cta"] > 1
    elif name.startswith("one_cta"):
        assert geo["max_tiles_per_cta"] == 2 and geo["ctas_with_max_tiles"] == 1 and geo["ctas_per_n"] < geo["m_tiles"]
    else:
        assert geo["n_tiles"] > 1 and geo["num_kb"] == 1 and geo["max_tiles_per_cta"] > 1
        assert geo["block_n"] == {192: 64, 320: 64, 384: 128, 768: 256}[n]
    x, w, base = _gemm_inputs(M, k, n, 1, 1, seed=M)
    y, gs = _gemm_run(x, w, base)
    _gemm_check(x, w, base, y, gs, geo)


def test_conv1x1_bnstats_weight_layouts():
    x, w, base = _gemm_inputs(8, 256, 512, 28, 28)
    y, gs = _gemm_run(x, w, base)
    y2, gs2 = _gemm_run(x, w.contiguous(memory_format=CL), base)
    assert torch.equal(y, y2) and torch.equal(gs, gs2)
    _gemm_check(x, w, base, y, gs, R.gemm_geometry(8 * 28 * 28, 512, 256, sms()))


_FORCED = """
import sys, torch
sys.path[:0] = [%r, %r]
import _fp64 as R
from test_gpu_fp64 import _gemm_inputs, _gemm_run, _gemm_check, sms
x, w, base = _gemm_inputs(2, 256, 512, 56, 56)
geo = R.gemm_geometry(2 * 56 * 56, 512, 256, sms(), max_block_n=%d)
assert geo["block_n"] == %d and geo["n_tiles"] > 1 and geo["max_tiles_per_cta"] > 1, geo
y, gs = _gemm_run(x, w, base)
_gemm_check(x, w, base, y, gs, geo)
print("ok", geo)
"""


@pytest.mark.parametrize("block_n", [64, 128])
def test_conv1x1_bnstats_forced_block_n(block_n):
    """PTD_GEMM_BLOCK_N caps BLOCK_N; it is read once per process, so each width runs in its own interpreter."""
    env = dict(os.environ, PTD_GEMM_BLOCK_N=str(block_n))
    p = subprocess.run([sys.executable, "-c", _FORCED % (os.path.dirname(TESTS), TESTS, block_n, block_n)], env=env,
                       capture_output=True, text=True, timeout=600)
    assert p.returncode == 0 and "ok" in p.stdout, p.stdout[-2000:] + p.stderr[-4000:]


def test_conv1x1_checkers_reject_edited_results():
    x, w, base = _gemm_inputs(8, 256, 512, 28, 28)
    geo = R.gemm_geometry(8 * 28 * 28, 512, 256, sms())
    y, gs = _gemm_run(x, w, base)
    _gemm_check(x, w, base, y, gs, geo)
    bad = y.clone()
    v = bad[3, 100, 5, 7].double()
    bad[3, 100, 5, 7] = (v + 2 * R.ulp(v, torch.bfloat16)).bfloat16()        # one element moved by 2 ulp
    with pytest.raises(AssertionError, match="conv1x1 y"):
        R.check_conv1x1(bad, x, w)
    tile = R.rows(y)[128:256].double()                                          # one 128-row tile left out of the sums
    gbad = gs.clone()
    gbad[:512] -= tile.sum(0).float()
    gbad[512:] -= (tile * tile).sum(0).float()
    with pytest.raises(AssertionError, match="gemm_bnstats"):
        R.check_sums("gemm_bnstats", gbad, R.rows(y), geo["depth"], base)


# ================================================================================================ fused BatchNorm
def _bn_params(C, wdt, seed):
    g = _gen(seed)
    w = (torch.rand(C, device=DEV, generator=g) + 0.5).to(wdt)
    b = torch.randn(C, device=DEV, generator=g).to(wdt)
    rm0 = torch.randn(C, device=DEV, generator=g) * 0.1
    rv0 = torch.rand(C, device=DEV, generator=g) + 0.5
    return w, b, rm0, rv0


def _bn_forward(x, res, w, b, rm0, rv0, relu, work=None, stats_ready=False):
    C = x.size(1)
    rm, rv = rm0.clone(), rv0.clone()
    nbt = torch.zeros((), dtype=torch.long, device=DEV)
    work = torch.zeros(2 * C, device=DEV) if work is None else work.clone()
    y, saved, mask = lib().bn_act_forward(x, res, w, b, rm, rv, nbt, True, 0.1, EPS, relu, True, work, stats_ready)
    return y, saved, mask, rm, rv, nbt


def _check_bn_forward(name, x, res, w, b, rm0, rv0, relu, out, depth, max_rel_invstd=None):
    y, saved, mask, rm, rv, nbt = out
    C = x.size(1)
    x2 = R.rows(x)
    st = R.check_stats(name, saved, x2, depth, EPS, max_rel_invstd)
    R.check_running(name, rm, rv, rm0, rv0, st, 0.1)
    assert nbt.item() == 1
    R.check_bn_forward(name, y, mask, x2, saved[:C], saved[C:], w, b, None if res is None else R.rows(res), relu)
    return st


def _check_bn_backward(name, x, w, saved, mask, relu, dz2d, depth, out):
    C = x.size(1)
    ref = R.bn_backward_ref(dz2d, R.rows(x), saved[:C], saved[C:], w, depth)
    dx, dw, db = out
    R.check_bn_backward(name, dx, dw, db, ref)


def _bn_full(name, x, res, w, b, rm0, rv0, relu, dt, twice=False, seed=0):
    """Forward, bn_act_backward and bn_act_backward2 of one case against fp64; with `twice`, each entry point is called a
    second time with the same inputs and must return the same bits."""
    C = x.size(1)
    M = x.numel() // C
    depth = R.bn_depth(M, C, sms())
    fwd = _bn_forward(x, res, w, b, rm0, rv0, relu)
    _check_bn_forward(name, x, res, w, b, rm0, rv0, relu, fwd, depth)
    y, saved, mask = fwd[:3]
    if twice:
        assert _equal_all(fwd, _bn_forward(x, res, w, b, rm0, rv0, relu)), name + ": forward is not reproducible"
    keep = R.unpack_mask(mask, M, C).double() if relu else 1.0
    g = _gen(seed + 1)
    dy = torch.randn(x.shape, device=DEV, generator=g).to(dt).contiguous(memory_format=CL)

    def bwd():
        return lib().bn_act_backward(dy, x, mask, w, saved, relu, res is not None, torch.zeros(2 * C, device=DEV))
    dx, dres, dw, db = bwd()
    dz = R.rows(dy).double() * keep
    _check_bn_backward(name + " backward", x, w, saved, mask, relu, dz, depth, (dx, dw, db))
    if res is not None:
        assert torch.equal(R.rows(dres).double(), dz)
    if twice:
        assert _equal_all((dx, dres, dw, db), bwd()), name + ": backward is not reproducible"
    dya = dy
    dyb = torch.randn(x.shape, device=DEV, generator=g).to(dt).contiguous(memory_format=CL)

    def bwd2():
        return lib().bn_act_backward2(dya, dyb, x, mask, w, saved, relu, torch.zeros(2 * C, device=DEV))
    dx2, gsum, dw2, db2 = bwd2()
    gz = (R.rows(dya).float() + R.rows(dyb).float()).to(dt).double() * keep     # the sum is rounded to the activation type
    assert torch.equal(R.rows(gsum).double(), gz)
    _check_bn_backward(name + " backward2", x, w, saved, mask, relu, gz, depth, (dx2, dw2, db2))
    if twice:
        assert _equal_all((dx2, gsum, dw2, db2), bwd2()), name + ": backward2 is not reproducible"


# (C, H = W, residual): BN after each 1x1 / 3x3 convolution of ResNet-50; the residual cases end a Bottleneck
RESNET50_BN = [(64, 56, False), (256, 56, True), (128, 56, False), (128, 28, False), (512, 28, True), (256, 28, False),
               (256, 14, False), (1024, 14, True), (512, 14, False), (512, 7, False), (2048, 7, True)]


@pytest.mark.parametrize("c,hw,res", RESNET50_BN, ids=["%d@%d%s" % (c, hw, "+res" if r else "") for c, hw, r in RESNET50_BN])
def test_bn_act_resnet50_batch256(c, hw, res):
    g = _gen(c + hw)
    x = torch.randn(256, c, hw, hw, device=DEV, generator=g).bfloat16().contiguous(memory_format=CL)
    r = torch.randn(256, c, hw, hw, device=DEV, generator=g).bfloat16().contiguous(memory_format=CL) if res else None
    w, b, rm0, rv0 = _bn_params(c, torch.float32, c)
    _bn_full("bn %d@%d" % (c, hw), x, r, w, b, rm0, rv0, True, torch.bfloat16, twice=True)


BN_C = [8, 24, 264, 2056, 4096]


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16, torch.float32], ids=["bf16", "fp16", "fp32"])
@pytest.mark.parametrize("c", BN_C)
@pytest.mark.parametrize("mkind", ["2", "8rpp-1", "8rpp+1"])
def test_bn_act_geometry_edges(dt, c, mkind):
    geo = R.bn_reduce_geometry(8, c, sms(), 4)
    M = {"2": 2, "8rpp-1": 8 * geo["rpp"] - 1, "8rpp+1": 8 * geo["rpp"] + 1}[mkind]
    geo = R.bn_reduce_geometry(M, c, sms(), 4)
    # C = 24: 3 threads per row; 264: 33 (not a power of two); 2056: a ragged second 256-thread chunk; 4096: two chunks
    assert geo["tpr"] == {8: 1, 24: 3, 264: 33, 2056: 256, 4096: 256}[c]
    assert geo["chunks"] == (2 if c > 2048 else 1) and geo["ragged"] == (c == 2056)
    res = c in (24, 2056)
    relu = not (c == 264 and mkind == "2")
    wdt = torch.bfloat16 if mkind == "8rpp+1" else torch.float32        # the ld_w / st_w paths of both parameter types
    g = _gen(c * 7 + M)
    x = torch.randint(-40, 41, (M, c, 1, 1), device=DEV, generator=g).to(dt).contiguous(memory_format=CL)
    r = torch.randint(-8, 9, (M, c, 1, 1), device=DEV, generator=g).to(dt).contiguous(memory_format=CL) if res else None
    w, b, rm0, rv0 = _bn_params(c, wdt, c + M)
    _bn_full("bn C=%d M=%d" % (c, M), x, r, w, b, rm0, rv0, relu, dt)


def test_bn_stats_two_wave_grid():
    """reduce_grid's two-wave branch at every occupancy up to 8 resident CTAs per SM."""
    c, hw = 64, 56
    M = 2 * 8 * sms() * 32 * 64                          # M / (2 waves) >= 64 row passes of 32 rows at 8 CTAs / SM
    n = R.cdiv(M, hw * hw)
    assert all(R.bn_reduce_geometry(n * hw * hw, c, sms(), r)["two_wave"] for r in range(1, 9))
    x = torch.randn(n, c, hw, hw, device=DEV, generator=_gen(5)).bfloat16().contiguous(memory_format=CL)
    w, b, rm0, rv0 = _bn_params(c, torch.float32, 5)
    y, saved, mask, rm, rv, nbt = _bn_forward(x, None, w, b, rm0, rv0, True)
    del y, mask
    st = R.check_stats("bn two-wave", saved, R.rows(x), R.bn_depth(n * hw * hw, c, sms()), EPS)
    R.check_running("bn two-wave", rm, rv, rm0, rv0, st, 0.1)


@pytest.mark.parametrize("ratio", [0, 4, 8])
def test_bn_stats_offset_mean(ratio):
    """x = mu + sigma z with mu / sigma = ratio: the one-pass variance E[x^2] - mean^2 loses about log2(1 + ratio^2)
    bits to cancellation; invstd must stay within 1e-3 of fp64."""
    g = _gen(ratio)
    s = 2.0 ** -3
    z = torch.round(torch.randn(256, 64, 56, 56, device=DEV, generator=g) * 4).clamp_(-60, 60)
    x = (s * (4 * ratio + z)).bfloat16().contiguous(memory_format=CL)          # |4 ratio + z| <= 92: exact in bf16
    w, b, rm0, rv0 = _bn_params(64, torch.float32, ratio)
    out = _bn_forward(x, None, w, b, rm0, rv0, True)
    st = _check_bn_forward("bn mu/sigma=%d" % ratio, x, None, w, b, rm0, rv0, True, out, R.bn_depth(x.numel() // 64, 64, sms()),
                           max_rel_invstd=1e-3)
    print("mu/sigma %d: max relative invstd error %.3g" % (ratio, st["rel_invstd"]))


def test_bn_stats_ready_from_conv1x1():
    """bn_act_forward(stats_ready=True) normalising with the sums the GEMM epilogue reduced; the GEMM output has a mean
    offset of about 4 standard deviations (a constant input channel)."""
    k, n, hw = 256, 128, 28
    x, w, _ = _gemm_inputs(64, k, n, hw, hw, seed=9)
    x[:, 0] = 1.0
    w[:, 0] = 4.0
    gs = torch.zeros(2 * n, device=DEV)
    y = lib().conv1x1_bnstats(x, w, gs)
    geo = R.gemm_geometry(64 * hw * hw, n, k, sms())
    wt, b, rm0, rv0 = _bn_params(n, torch.float32, 9)
    out = _bn_forward(y, None, wt, b, rm0, rv0, True, work=gs, stats_ready=True)
    _check_bn_forward("bn stats_ready", y, None, wt, b, rm0, rv0, True, out, geo["depth"], max_rel_invstd=1e-3)


@pytest.mark.parametrize("wdt", [torch.float32, torch.bfloat16], ids=["w_fp32", "w_bf16"])
def test_bn_act_eval_mode(wdt):
    c = 256
    x = torch.randn(64, c, 14, 14, device=DEV, generator=_gen(11)).bfloat16().contiguous(memory_format=CL)
    r = torch.randn(64, c, 14, 14, device=DEV, generator=_gen(12)).bfloat16().contiguous(memory_format=CL)
    w, b, rm, rv = _bn_params(c, wdt, 13)
    rm0, rv0 = rm.clone(), rv.clone()
    y, saved, mask = lib().bn_act_forward(x, r, w, b, rm, rv, None, False, 0.1, EPS, True, True, torch.zeros(2 * c, device=DEV), False)
    assert torch.equal(rm, rm0) and torch.equal(rv, rv0)
    invstd = 1.0 / torch.sqrt(rv.double() + EPS)
    pre, e = R.bn_apply_ref(R.rows(x), rm, invstd, w, b, R.rows(r))
    e = e + 2.0 ** -20 * (pre - R.rows(r).double() - b.double()).abs()      # rsqrtf
    R.assert_within("bn eval y", R.rows(y), pre.clamp_min(0), 0.5 * R.ulp(R.rows(y), torch.bfloat16) + e)
    bits = R.unpack_mask(mask, x.numel() // c, c)
    assert not ((bits != (pre > 0)) & (pre.abs() > e)).any()


def test_bn_checkers_reject_edited_results():
    c = 64
    x = torch.randint(-40, 41, (4, c, 9, 9), device=DEV, generator=_gen(20)).bfloat16().contiguous(memory_format=CL)
    w, b, rm0, rv0 = _bn_params(c, torch.float32, 20)
    out = _bn_forward(x, None, w, b, rm0, rv0, True)
    depth = R.bn_depth(x.numel() // c, c, sms())
    _check_bn_forward("bn", x, None, w, b, rm0, rv0, True, out, depth)
    y, saved, mask, rm, rv, nbt = out
    x2 = R.rows(x)
    bad = y.clone()
    flat = R.rows(bad).view(-1)                                     # a view: channels_last rows are contiguous
    i = (flat > 0).int().argmax()
    flat[i] = (flat[i].double() + 2 * R.ulp(flat[i], torch.bfloat16)).bfloat16()
    with pytest.raises(AssertionError, match="bn y"):
        R.check_bn_forward("bn", bad, mask, x2, saved[:c], saved[c:], w, b)
    mbad = mask.clone()
    mbad[7] ^= 1
    with pytest.raises(AssertionError, match="bn mask"):
        R.check_bn_forward("bn", y, mbad, x2, saved[:c], saved[c:], w, b)
    sbad = saved.clone()
    sbad[c + 3] *= 1 + 2e-3
    with pytest.raises(AssertionError, match="bn invstd"):
        R.check_stats("bn", sbad, x2, depth, EPS)
    dy = torch.randn(x.shape, device=DEV, generator=_gen(21)).bfloat16().contiguous(memory_format=CL)
    dx, _, dw, db = lib().bn_act_backward(dy, x, mask, w, saved, True, False, torch.zeros(2 * c, device=DEV))
    dz = R.rows(dy).double() * R.unpack_mask(mask, x2.size(0), c).double()
    ref = R.bn_backward_ref(dz, x2, saved[:c], saved[c:], w, depth)
    R.check_bn_backward("bn", dx, dw, db, ref)
    dxb = dx.clone()
    v = dxb[1, 2, 3, 4].double()
    dxb[1, 2, 3, 4] = (v + 2 * R.ulp(v, torch.bfloat16)).bfloat16()
    with pytest.raises(AssertionError, match="bn dx"):
        R.check_bn_backward("bn", dxb, dw, db, ref)
    dwb = dw.clone()
    dwb[5] += 1e-3 * dw.abs().max()
    with pytest.raises(AssertionError, match="bn dgamma"):
        R.check_bn_backward("bn", dx, dwb, db, ref)


# ================================================================================================ fused stem
def _stem_inputs(N, C, H, W, dt, wdt=torch.float32, seed=0):
    x64, s = R.tie_free_stem_input(N, C, H, W, device=DEV, seed=seed)
    x = x64.to(dt).contiguous(memory_format=CL)                 # exact: |x| / s_c <= 134
    g = _gen(seed + 1)
    w = (torch.rand(C, device=DEV, generator=g) + 0.5).to(wdt)
    b = R.stem_bias_between_levels(x64, s, w, EPS).to(wdt)      # rounding moves the ReLU threshold by < s_c / 8
    del x64
    rm0 = torch.randn(C, device=DEV, generator=g) * 0.1
    rv0 = torch.rand(C, device=DEV, generator=g) + 0.5
    OH, OW = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    dp = (torch.randint(-8, 9, (N, C, OH, OW), device=DEV, generator=g) / 8).to(dt).contiguous(memory_format=CL)
    return x, w, b, rm0, rv0, dp                                # dp: sums of up to 4 are exact in every dtype


def _stem_forward(x, w, b, rm0, rv0, work=None, pre=False):
    C = x.size(1)
    rm, rv = rm0.clone(), rv0.clone()
    nbt = torch.zeros((), dtype=torch.long, device=DEV)
    work = torch.zeros(2 * C, device=DEV) if work is None else work.clone()
    fn = lib().stem_forward_pre if pre else lib().stem_forward
    y, saved, code = fn(x, w, b, rm, rv, nbt, True, 0.1, EPS, True, work)
    return y, saved, code, rm, rv, nbt


def check_stem_forward(name, x, w, b, y, saved, code):
    """4-bit codes exactly, pooled y within 1 ulp (16-bit) or the derived bound (fp32), from the kernel's statistics."""
    N, C, H, W = x.shape
    yref, cref, e_sel, margin = R.stem_forward_ref(x, saved[:C], saved[C:], w, b)
    assert margin > 100, "%s: a pre-activation lies within 100x the rounding bound of 0 (margin %.3g)" % (name, margin)
    got = R.code_nchw(code, N, C, *yref.shape[2:])
    wrong = got != cref
    assert not wrong.any(), "%s codes: %d differ" % (name, int(wrong.sum()))
    R.assert_within(name + " y", y, yref, 0.5 * R.ulp(y, y.dtype) + e_sel)
    if y.dtype != torch.float32:
        R.assert_within(name + " y (1 ulp)", y, yref, R.ulp(yref, y.dtype))
    return cref


def _stem_full(name, N, C, H, W, dt, wdt=torch.float32, twice=False):
    x, w, b, rm0, rv0, dp = _stem_inputs(N, C, H, W, dt, wdt, seed=N + C + H + W)
    fwd = _stem_forward(x, w, b, rm0, rv0)
    y, saved, code, rm, rv, nbt = fwd
    st = R.check_stats(name, saved, R.rows(x), R.bn_depth(N * H * W, C, sms()), EPS)
    R.check_running(name, rm, rv, rm0, rv0, st, 0.1)
    cref = check_stem_forward(name, x, w, b, y, saved, code)
    if twice:
        assert _equal_all(fwd, _stem_forward(x, w, b, rm0, rv0)), name + ": forward is not reproducible"
    geo = R.stem_bwd_geometry(N, C, H, W, sms())

    def bwd():
        return lib().stem_backward(dp, x, code, w, saved, torch.zeros(2 * C, device=DEV))
    dx, dw, db = bwd()
    dz = R.stem_dz_ref(dp, cref, H, W)
    ref = R.bn_backward_ref(R.rows(dz), R.rows(x), saved[:C], saved[C:], w, geo["depth"])
    R.check_bn_backward(name, dx, dw, db, ref)
    if twice:
        assert _equal_all((dx, dw, db), bwd()), name + ": backward is not reproducible"
    return geo


# (name, N as a function of the SM count, C, H, W, dtype, quad rows per CTA it must reach, rows cross images)
_Q = lambda rpb, qh: (lambda s: R.cdiv(rpb * s * 8, qh))    # noqa: E731  smallest N with N * ceil(H/2) >= rpb * sms * 8
STEM_CASES = [
    ("small_odd_15x13_bf16", lambda s: 2, 64, 15, 13, torch.bfloat16, 1, False),
    ("small_odd_9x9_fp16_c32", lambda s: 3, 32, 9, 9, torch.float16, 1, False),
    ("small_even_8x10_fp32_c128", lambda s: 2, 128, 8, 10, torch.float32, 1, False),
    ("small_even_16x16_fp16", lambda s: 4, 64, 16, 16, torch.float16, 1, False),
    ("rpb2_odd_13x13_bf16", _Q(2, 7), 64, 13, 13, torch.bfloat16, 2, True),
    ("rpb3_odd_13x14_fp16_c32", _Q(3, 7), 32, 13, 14, torch.float16, 3, True),
    ("rpb2_even_14x12_fp32_c128", _Q(2, 7), 128, 14, 12, torch.float32, 2, True),
    ("rpb3_odd_13x13_fp32", _Q(3, 7), 64, 13, 13, torch.float32, 3, True),
    ("rpb2_even_16x16_bf16_c128", _Q(2, 8), 128, 16, 16, torch.bfloat16, 2, False),
    ("rpb4_production_bf16", lambda s: 256, 64, 112, 112, torch.bfloat16, 4, False),
]


@pytest.mark.parametrize("name,n_of,c,h,w,dt,rpb,cross", STEM_CASES, ids=[s[0] for s in STEM_CASES])
def test_stem_forward_backward_fp64(name, n_of, c, h, w, dt, rpb, cross):
    N = n_of(sms())
    geo = R.stem_bwd_geometry(N, c, h, w, sms())
    assert geo["rows_per_block"] == rpb and geo["crosses_images"] == cross, geo
    _stem_full(name, N, c, h, w, dt, wdt=torch.bfloat16 if "fp16" in name else torch.float32, twice=name.startswith("rpb4"))


def test_stem_forward_pre_from_stem_gemm():
    """stem_forward_pre normalising with the sums of the stem GEMM (im2col + conv1x1_bnstats), as the stem-GEMM path runs
    it.  The GEMM output is not tie-free, so the codes are only checked for consistency with y (15 <=> y == 0)."""
    from pytorch_distributed_b200.ops.stem_conv import K_PAD, pack_stem_weight
    img = torch.randn(32, 3, 224, 224, device=DEV, generator=_gen(30)).bfloat16().contiguous(memory_format=CL)
    wconv = (torch.randn(64, 3, 7, 7, device=DEV, generator=_gen(31)) * 0.1).bfloat16()
    a = lib().stem_im2col(img)
    gs = torch.zeros(2 * 64, device=DEV)
    yc = lib().conv1x1_bnstats(a, pack_stem_weight(wconv).view(64, K_PAD, 1, 1), gs)
    geo = R.gemm_geometry(yc.numel() // 64, 64, K_PAD, sms())
    w, b, rm0, rv0 = _bn_params(64, torch.float32, 32)
    y, saved, code, rm, rv, nbt = _stem_forward(yc, w, b, rm0, rv0, work=gs, pre=True)
    st = R.check_stats("stem_pre", saved, R.rows(yc), geo["depth"], EPS)
    R.check_running("stem_pre", rm, rv, rm0, rv0, st, 0.1)
    assert nbt.item() == 1
    yref, _, e_sel, _ = R.stem_forward_ref(yc, saved[:64], saved[64:], w, b)
    R.assert_within("stem_pre y", y, yref, 0.5 * R.ulp(y, y.dtype) + e_sel)
    assert torch.equal(R.code_nchw(code, *y.shape) == 15, y == 0)


def test_stem_checkers_reject_edited_results():
    N, C, H, W = 3, 64, 13, 13
    x, w, b, rm0, rv0, dp = _stem_inputs(N, C, H, W, torch.bfloat16, seed=40)
    y, saved, code, *_ = _stem_forward(x, w, b, rm0, rv0)
    cref = check_stem_forward("stem", x, w, b, y, saved, code)
    cbad = code.clone()
    cbad[100] = (int(cbad[100]) + 1) % 9
    with pytest.raises(AssertionError, match="stem codes"):
        check_stem_forward("stem", x, w, b, y, saved, cbad)
    ybad = y.clone()
    flat = R.rows(ybad).view(-1)
    i = (flat > 0).int().argmax()
    flat[i] = (flat[i].double() + 2 * R.ulp(flat[i], torch.bfloat16)).bfloat16()
    with pytest.raises(AssertionError, match="stem y"):
        check_stem_forward("stem", x, w, b, ybad, saved, code)
    dx, dw, db = lib().stem_backward(dp, x, code, w, saved, torch.zeros(2 * C, device=DEV))
    ref = R.bn_backward_ref(R.rows(R.stem_dz_ref(dp, cref, H, W)), R.rows(x), saved[:C], saved[C:], w,
                            R.stem_bwd_geometry(N, C, H, W, sms())["depth"])
    R.check_bn_backward("stem", dx, dw, db, ref)
    dxb = dx.clone()
    dxb[N - 1, :, H - 1, W - 1] = 0                                   # one corner of the input gradient zeroed
    with pytest.raises(AssertionError, match="stem dx"):
        R.check_bn_backward("stem", dxb, dw, db, ref)
