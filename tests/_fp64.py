"""Float64 references of the hand-written GEMM, BatchNorm and stem kernels, with error bounds taken from how each kernel
computes.

Each reference takes the exact (bf16 / fp16 / fp32) inputs the kernel was given and computes in float64.  Each checker
raises AssertionError naming the worst offending element.  The ``*_geometry`` functions repeat the launch arithmetic of
``csrc/gemm_bnstats.cu`` (``launch_gemm``) and ``csrc/bn_act.cu`` (``reduce_grid``, ``stem_bwd_impl``), so a test can
state which branch a case reaches and how many fp32 additions lie on the longest path of each reduction ("depth").

Rounding-error bounds: a sum of fp32 values computed by any tree of additions whose longest leaf-to-root path has d
additions is within d * u * sum|terms| of the exact sum (u = 2^-24, round to nearest; the d u / (1 - d u) form differs
by less than 1 % for every depth used here, covered by the factor 1.01).
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

U32 = 2.0 ** -24
_MANT = {torch.bfloat16: 7, torch.float16: 10, torch.float32: 23}
_TINY = {torch.bfloat16: 2.0 ** -133, torch.float16: 2.0 ** -24, torch.float32: 2.0 ** -149}


def cdiv(a: int, b: int) -> int:
    return -(-a // b)


def ulp(v: torch.Tensor, dtype) -> torch.Tensor:
    """Spacing of ``dtype`` numbers at |v| (float64), i.e. 2^(floor(log2|v|) - mantissa bits), subnormal spacing near 0."""
    a = v.double().abs()
    _, e = torch.frexp(a)                      # a = m * 2^e, m in [0.5, 1)
    u = torch.ldexp(torch.ones_like(a), (e - 1 - _MANT[dtype]).double())
    return torch.where(a > 0, u, torch.zeros_like(u)).clamp_min(_TINY[dtype])


def assert_within(name: str, got: torch.Tensor, ref: torch.Tensor, tol) -> None:
    err = (got.double() - ref).abs()
    tol = torch.as_tensor(tol, dtype=torch.float64, device=err.device).expand_as(err)
    bad = err > tol
    nbad = int(bad.sum())
    if nbad:
        i = int(bad.flatten().to(torch.int8).argmax())
        raise AssertionError("%s: %d of %d elements outside the bound; first at flat index %d: got %r, fp64 %r, |err| %.3g > bound %.3g"
                             % (name, nbad, err.numel(), i, got.flatten()[i].item(), ref.flatten()[i].item(),
                                err.flatten()[i].item(), tol.flatten()[i].item()))


def rows(t: torch.Tensor) -> torch.Tensor:
    """[N, C, H, W] (channels_last or not) -> [N*H*W, C]."""
    return t.permute(0, 2, 3, 1).reshape(-1, t.size(1))


# ---------------------------------------------------------------------------------------------------------- geometry
def gemm_geometry(M: int, N: int, K: int, sms: int, max_block_n: int = 256) -> dict:
    """launch_gemm: BLOCK_N choice, persistent grid, tiles per CTA and the depth of the epilogue statistics sums."""
    bn = 256 if N % 256 == 0 and max_block_n >= 256 else 128 if N % 128 == 0 and max_block_n >= 128 else 64
    m_tiles, n_tiles = cdiv(M, 128), N // bn
    ctas_per_n = max(1, min(m_tiles, sms // n_tiles))
    tiles = cdiv(m_tiles, ctas_per_n)
    pairs = bn // 2
    parts = 128 // pairs
    # per thread: `64 / parts` staged rows per tile, then 2 warpgroups x `parts` row parts in order, then
    # combine_partials (ctas_per_n rows in 32 slices, the 32 slice sums) and the add into gsum
    depth = tiles * (64 // parts) + 2 * parts + cdiv(ctas_per_n, 32) + 32 + 1
    return dict(block_n=bn, m_tiles=m_tiles, n_tiles=n_tiles, ctas_per_n=ctas_per_n, max_tiles_per_cta=tiles,
                ctas_with_max_tiles=m_tiles - (tiles - 1) * ctas_per_n, num_kb=K // 64, depth=depth)


def bn_reduce_geometry(M: int, C: int, sms: int, resident: int) -> dict:
    """reduce_grid + cta_combine of bn_stats / bn_bwd_reduce / bn_bwd_reduce_sum at `resident` CTAs per SM."""
    tpr = min(C // 8, 256)
    rpp = 256 // tpr
    blocks = cdiv(M, rpp * 8)
    wave = sms * resident
    two_wave = False
    if blocks > wave:
        two_wave = blocks >= 2 * wave and M // (2 * wave) >= rpp * 64
        blocks = 2 * wave if two_wave else wave
    blocks = max(blocks, 1)
    rpb = cdiv(cdiv(M, blocks), rpp) * rpp
    grid = cdiv(M, rpb)
    fold = (tpr & (tpr - 1)) == 0 and tpr < 32
    depth = rpb // rpp + (int(math.log2(32 // tpr)) if fold else 0) + (8 if fold else rpp) + cdiv(grid, 32) + 32 + 1
    return dict(tpr=tpr, rpp=rpp, rows_per_block=rpb, grid=grid, two_wave=two_wave, chunks=cdiv(C // 8, tpr),
                ragged=(C // 8) % tpr != 0, depth=depth)


def bn_depth(M: int, C: int, sms: int) -> int:
    """Reduction depth whatever the occupancy (1..8 resident CTAs of 256 threads per SM)."""
    return max(bn_reduce_geometry(M, C, sms, r)["depth"] for r in range(1, 9))


def stem_bwd_geometry(N: int, C: int, H: int, W: int, sms: int) -> dict:
    """stem_bwd_impl: quad rows per CTA, whether a CTA's quad rows cross an image boundary, reduction depth."""
    qh, qw = (H + 1) // 2, (W + 1) // 2
    nrows = N * qh
    rpb = max(1, min(4, nrows // (sms * 8)))
    grid = cdiv(nrows, rpb)
    tpr = C // 8
    rpp = 256 // tpr
    fold = tpr < 32
    depth = rpb * cdiv(qw, rpp) * 4 + (int(math.log2(32 // tpr)) if fold else 0) + (8 if fold else rpp) + cdiv(grid, 32) + 32 + 1
    return dict(rows_per_block=rpb, quad_rows=nrows, grid=grid, crosses_images=rpb > 1 and qh % rpb != 0, depth=depth)


# ---------------------------------------------------------------------------------------------------------- GEMM
def check_conv1x1(y: torch.Tensor, x: torch.Tensor, w: torch.Tensor, max_changed: float | None = None) -> None:
    """y = conv1x1(x, w) in bf16 against the fp64 product of the same bf16 operands.

    The products of two bf16 values are exact in fp32 (8 + 8 significant bits), so the only fp32 error is in the K - 1
    additions of the accumulation: at most (K - 1) u sum_k |a_k b_k| / (1 - (K - 1) u) < K u sum_k |a_k b_k|.  Rounding
    the fp32 result to bf16 adds at most half a bf16 ulp of the stored value (rounding is monotone, so ulp(y) >= ulp of
    the fp32 value).  Apart from that bound, at most `max_changed` of the elements may differ from bf16(fp64) at all:
    only elements whose exact value lies within the accumulation error of a bf16 rounding boundary can.  That error grows
    with K, so the default allowance does too: 1e-3 up to K = 1024 (1.2e-3 was measured at K = 2048 on an H100)."""
    K, N = x.size(1), w.size(0)
    if max_changed is None:
        max_changed = 1e-3 * max(1.0, K / 1024)
    a = rows(x).double()
    b = w.reshape(N, K).double()
    ref = a @ b.t()
    mag = a.abs() @ b.abs().t()
    del a, b
    got = rows(y)
    assert_within("conv1x1 y", got, ref, 0.5 * ulp(got, torch.bfloat16) + K * U32 * mag)
    changed = (got != ref.to(torch.bfloat16)).double().mean().item()
    assert changed <= max_changed, "conv1x1 y: %.3g of the elements differ from bf16(fp64) (limit %.3g)" % (changed, max_changed)


def check_sums(name: str, gsum: torch.Tensor, vals2d: torch.Tensor, depth: int, base: torch.Tensor | None = None) -> None:
    """gsum[0:C] = base + sum of vals, gsum[C:2C] = base + sum of vals^2 (squares of 16-bit values are exact in fp32)."""
    v = vals2d.double()
    C = v.size(1)
    s, q, sa = v.sum(0), (v * v).sum(0), v.abs().sum(0)
    if base is not None:
        s, q = s + base[:C].double(), q + base[C:2 * C].double()
        sa = sa + base[:C].double().abs()
        qa = (v * v).sum(0) + base[C:2 * C].double().abs()
    else:
        qa = q
    assert_within(name + " sum", gsum[:C], s, 1.01 * depth * U32 * sa)
    assert_within(name + " sum of squares", gsum[C:2 * C], q, 1.01 * depth * U32 * qa)


# ---------------------------------------------------------------------------------------------------------- BatchNorm
def batch_stats(x2d: torch.Tensor, eps: float) -> dict:
    x = x2d.double()
    M = x.size(0)
    mean = x.mean(0)
    var = ((x - mean) ** 2).mean(0)
    return dict(M=M, mean=mean, var=var, invstd=1.0 / torch.sqrt(var + eps), s1=x.abs().sum(0), s2=(x * x).sum(0))


def stats_bounds(st: dict, depth: int, eps: float) -> tuple:
    """Error bounds of the kernels' mean and invstd: sums of depth `depth` (check_sums), mean = sum * (1/M), the one-pass
    variance E[x^2] - mean^2 in fp32, rsqrtf (relative error < 2^-21 with fast math)."""
    M, mean = st["M"], st["mean"]
    e2 = st["s2"] / M
    dmean = 1.01 * depth * U32 * st["s1"] / M + 4 * U32 * mean.abs()
    de2 = 1.01 * depth * U32 * st["s2"] / M + 4 * U32 * e2
    dvar = de2 + (2 * mean.abs() + dmean) * dmean + 2 * U32 * (e2 + mean * mean)
    r = dvar / (st["var"] + eps)
    rel_inv = torch.where(r < 1, 0.5 * r / (1 - r).clamp_min(1e-300), torch.full_like(r, math.inf)) + 2.0 ** -21 + U32
    return dmean, dvar, rel_inv


def check_stats(name: str, saved: torch.Tensor, x2d: torch.Tensor, depth: int, eps: float, max_rel_invstd: float | None = None) -> dict:
    """saved = [mean | invstd] (fp32) against the fp64 batch statistics of x."""
    C = x2d.size(1)
    st = batch_stats(x2d, eps)
    dmean, dvar, rel_inv = stats_bounds(st, depth, eps)
    assert_within(name + " mean", saved[:C], st["mean"], dmean)
    assert_within(name + " invstd", saved[C:2 * C], st["invstd"], rel_inv * st["invstd"])
    rel = ((saved[C:2 * C].double() - st["invstd"]).abs() / st["invstd"]).max().item()
    if max_rel_invstd is not None:
        assert rel <= max_rel_invstd, "%s invstd: relative error %.3g > %.3g" % (name, rel, max_rel_invstd)
    st.update(dmean=dmean, dvar=dvar, rel_invstd=rel)
    return st


def check_running(name: str, rm: torch.Tensor, rv: torch.Tensor, rm0: torch.Tensor, rv0: torch.Tensor, st: dict, momentum: float) -> None:
    """running_mean / running_var (unbiased, M / (M - 1)) after one training step from rm0 / rv0."""
    m = float(torch.tensor(momentum, dtype=torch.float32))     # the kernel blends with the fp32 momentum
    M = st["M"]
    f = M / (M - 1) if M > 1 else 1.0
    erm = (1 - m) * rm0.double() + m * st["mean"]
    erv = (1 - m) * rv0.double() + m * st["var"] * f
    assert_within(name + " running_mean", rm, erm, m * st["dmean"] + 4 * U32 * ((1 - m) * rm0.double().abs() + m * st["mean"].abs()))
    assert_within(name + " running_var", rv, erv, m * f * st["dvar"] + 6 * U32 * ((1 - m) * rv0.double().abs() + m * f * st["var"]))


def unpack_mask(mask: torch.Tensor, M: int, C: int) -> torch.Tensor:
    """The ReLU bit mask (byte [row * C/8 + c/8], bit c % 8) -> bool [M, C]."""
    bits = torch.arange(8, device=mask.device, dtype=torch.uint8)
    return ((mask.view(M, C // 8, 1) >> bits) & 1).bool().reshape(M, C)


def bn_apply_ref(x2d, mean, invstd, w, b, res2d=None, relu=True):
    """pre = (x - mean) * invstd * w + b (+ res) in fp64, from the given statistics; returns (pre, bound of the kernel's
    fp32 pre-activation: sc = w*invstd, sh = b - mean*sc, v = x*sc + sh (+ res), a few roundings of each term)."""
    sc = w.double() * invstd.double()
    x = x2d.double()
    pre = x * sc + (b.double() - mean.double() * sc)
    e = (x * sc).abs() + (mean.double() * sc).abs() + b.double().abs()
    if res2d is not None:
        pre = pre + res2d.double()
        e = e + res2d.double().abs()
    return pre, 4 * U32 * e + 2 * U32 * pre.abs()


def check_bn_forward(name, y, mask, x2d, mean, invstd, w, b, res2d=None, relu=True, max_band=1e-3) -> None:
    """y and the ReLU mask against fp64 applied with the kernel's own statistics (checked separately by check_stats).
    The mask must be exact wherever the fp64 pre-activation is farther from 0 than the fp32 error bound."""
    pre, e = bn_apply_ref(x2d, mean, invstd, w, b, res2d, relu)
    ref = pre.clamp_min(0) if relu else pre
    got = rows(y)
    assert_within(name + " y", got, ref, 0.5 * ulp(got, y.dtype) + e)
    if relu and mask is not None:
        M, C = got.shape
        bits = unpack_mask(mask, M, C)
        band = pre.abs() <= e
        wrong = (bits != (pre > 0)) & ~band
        assert not wrong.any(), "%s mask: %d bits differ outside the |pre| <= bound band" % (name, int(wrong.sum()))
        frac = band.double().mean().item()
        assert frac <= max_band, "%s mask: %.3g of the pre-activations lie in the unchecked band" % (name, frac)


def bn_backward_ref(dz2d, x2d, mean, invstd, w, depth):
    """dx, dgamma = sum dz*xhat, dbeta = sum dz from the exact masked gradient dz and the statistics the kernel saved, with
    bounds: sums of depth `depth` (+3 roundings in dz * (x - mean) * invstd), then dx = ka dz + kb x + kd with
    ka = w invstd, kb = -ka invstd sdzx / M, kd = -ka sdz / M - kb mean, each formed with a few fp32 roundings."""
    dz, x = dz2d.double(), x2d.double()
    M = dz.size(0)
    mean, invstd = mean.double(), invstd.double()
    xhat = (x - mean) * invstd
    sdz, sdzx = dz.sum(0), (dz * xhat).sum(0)
    d_sdz = 1.01 * depth * U32 * dz.abs().sum(0)
    d_sdzx = 1.01 * (depth + 3) * U32 * (dz * xhat).abs().sum(0)
    ka = w.double() * invstd
    kb = -ka * invstd * sdzx / M
    kd = -ka * sdz / M - kb * mean
    dx = ka * (dz - sdz / M - xhat * sdzx / M)
    e = (ka.abs() * d_sdz / M + (ka * xhat).abs() * d_sdzx / M
         + 6 * U32 * ((ka * dz).abs() + (kb * x).abs() + kd.abs() + (ka * sdz / M).abs() + (kb * mean).abs()))
    return dict(dx=dx, dx_bound=e, dgamma=sdzx, dbeta=sdz, dgamma_bound=d_sdzx, dbeta_bound=d_sdz)


def check_bn_backward(name, dx, dw, db, ref) -> None:
    got = rows(dx)
    assert_within(name + " dx", got, ref["dx"], 0.5 * ulp(got, dx.dtype) + ref["dx_bound"])
    assert_within(name + " dgamma", dw, ref["dgamma"], 0.5 * ulp(dw, dw.dtype) + ref["dgamma_bound"])
    assert_within(name + " dbeta", db, ref["dbeta"], 0.5 * ulp(db, db.dtype) + ref["dbeta_bound"])


# ---------------------------------------------------------------------------------------------------------- stem
def tie_free_stem_input(N, C, H, W, device="cpu", seed=0):
    """x[n,c,h,w] = s_c (9 q + 3 (h mod 3) + (w mod 3)), q in [-14, 14], s_c a power of two: every 3x3 window holds
    nine distinct residues mod 9, so no window has two equal values, and |x| / s_c <= 134 is exact in bf16 and fp16.
    Returned as float64 (NCHW), together with s."""
    gen = torch.Generator(device=device).manual_seed(seed)
    q = torch.randint(-14, 15, (N, C, H, W), generator=gen, device=device).double()
    s = torch.ldexp(torch.ones(C, dtype=torch.float64, device=device),
                    torch.randint(-2, 3, (C,), generator=gen, device=device).double())
    r = 3 * (torch.arange(H, device=device) % 3).double()[:, None] + (torch.arange(W, device=device) % 3).double()[None, :]
    return s[:, None, None] * (9 * q + r), s


def stem_bias_between_levels(x64, s, w, eps):
    """A BN bias that puts the ReLU threshold halfway between two neighbouring levels s_c * k of each channel (a quarter
    of a standard deviation below the mean), so no pre-activation lies near 0 and every 4-bit code is decided far from
    rounding noise."""
    st = batch_stats(rows(x64), eps)
    thr = (torch.floor((st["mean"] - 0.25 * st["var"].sqrt()) / s) + 0.5) * s
    return w.double() * st["invstd"] * (st["mean"] - thr)


def stem_forward_ref(x, mean, invstd, w, b):
    """relu(bn(x)) -> maxpool 3x3/2/1 in fp64 with the given statistics: returns (y, code, bound at the selected input,
    min |pre-activation| / bound) where code = kh*3 + kw of the window's arg-max, or 15 when every candidate is <= 0."""
    N, C, H, W = x.shape
    sc = (w.double() * invstd.double())[:, None, None]
    xd = x.double()
    pre = xd * sc + (b.double()[:, None, None] - (mean.double()[:, None, None] * sc))
    e = 4 * U32 * ((xd * sc).abs() + (mean.double()[:, None, None] * sc).abs() + b.double().abs()[:, None, None]) + 2 * U32 * pre.abs()
    margin = (pre.abs() / e).min().item()
    del xd
    pooled, idx = F.max_pool2d(pre.contiguous(), 3, 2, 1, return_indices=True)
    OH, OW = pooled.shape[2:]
    ih, iw = idx // W, idx % W
    kh = ih - (2 * torch.arange(OH, device=x.device)[:, None] - 1)
    kw = iw - (2 * torch.arange(OW, device=x.device)[None, :] - 1)
    code = torch.where(pooled > 0, kh * 3 + kw, torch.full_like(kh, 15)).to(torch.uint8)
    e_sel = torch.gather(e.reshape(N, C, -1), 2, idx.reshape(N, C, -1)).reshape(pooled.shape)
    return pooled.clamp_min(0), code, e_sel, margin


def code_nchw(code: torch.Tensor, N, C, OH, OW) -> torch.Tensor:
    """The kernel's code bytes ([pooled pixel][channel]) as [N, C, OH, OW]."""
    return code.view(N, OH, OW, C).permute(0, 3, 1, 2)


def stem_dz_ref(dp, code, H, W):
    """Gradient at the BN+ReLU output: each pooled gradient goes to the input its code selected (none for code 15)."""
    N, C, OH, OW = dp.shape
    dzp = torch.zeros(N, C, 2 * OH + 1, 2 * OW + 1, dtype=torch.float64, device=dp.device)
    d = dp.double()
    for k in range(9):
        kh, kw = divmod(k, 3)
        dzp[:, :, kh:kh + 2 * OH:2, kw:kw + 2 * OW:2] += torch.where(code == k, d, torch.zeros_like(d))
    return dzp[:, :, 1:H + 1, 1:W + 1]


# ---------------------------------------------------------------------------------------------------------- optimizer
# csrc/optim.cu: chunked multi-tensor apply (mta_for_each) and the flat SGD launch
MTA_TENSORS, MTA_BLOCKS, MTA_CHUNK = 30, 320, 8192


def sgd_step_fp64(p, m, g, hyper, nesterov: bool, first: bool) -> dict:
    """One step of ``sgd_update`` (csrc/optim.cu) in float64 from the fp32 state the kernel started with: returns the new
    master ``p``, momentum ``m``, and a bound on the kernel's error in each.

    ``hyper`` = (lr, momentum, weight_decay, dampening, gmul) as the kernel read them (fp32 values).  The kernel computes
        a = g*gmul + wd*p;  m' = first ? a : mom*m + (1 - d)*a;  b = nesterov ? a + mom*m' : m';  p' = p - lr*b
    (momentum 0: b = a, m unchanged) with fp32 roundings of every product, sum and of (1 - d).  Each rounding adds at
    most u |value rounded| (u = 2^-24); the errors carried into a later operation are scaled by its coefficient:
        e_a  = u (|g gmul| + |wd p| + |a|)
        e_m' = e_a                                              (first)
             = u |mom m| + |1-d| e_a + 2 u |(1-d) a| + u |m'|   (otherwise)
        e_b  = e_a + |mom| e_m' + u |mom m'| + u |b|            (nesterov),  e_m'  (plain),  e_a  (momentum 0)
        e_p' = |lr| e_b + u |lr b| + u |p'|
    An FMA contraction by nvcc removes roundings, so it only tightens this.  First-order terms only: the factor 1.01
    covers the products of u, and 8 * 2^-126 covers results flushed to zero (the extension is built with --use_fast_math,
    so subnormal fp32 results are flushed).  Compare one step at a time from the
    kernel's own previous state, so that errors do not compound."""
    lr, mom, wd, d, gmul = (float(x) for x in hyper[:5])
    p, m, g = p.double(), m.double(), g.double()
    tiny = 8 * 2.0 ** -126
    a = g * gmul + wd * p
    e_a = U32 * ((g * gmul).abs() + (wd * p).abs() + a.abs())
    if mom != 0.0:
        if first:
            m1, e_m = a, e_a
        else:
            m1 = mom * m + (1.0 - d) * a
            e_m = U32 * (mom * m).abs() + abs(1.0 - d) * e_a + 2 * U32 * ((1.0 - d) * a).abs() + U32 * m1.abs()
        if nesterov:
            b = a + mom * m1
            e_b = e_a + abs(mom) * e_m + U32 * (mom * m1).abs() + U32 * b.abs()
        else:
            b, e_b = m1, e_m
    else:
        m1, e_m = m, torch.zeros_like(m)
        b, e_b = a, e_a
    p1 = p - lr * b
    e_p = abs(lr) * e_b + U32 * (lr * b).abs() + U32 * p1.abs()
    return dict(p=p1, m=m1, p_bound=1.01 * e_p + tiny, m_bound=1.01 * e_m + tiny)


def check_sgd(name: str, p, m, ref: dict) -> float:
    """Master and momentum against sgd_step_fp64; returns the largest error / bound ratio."""
    assert_within(name + " master", p, ref["p"], ref["p_bound"])
    assert_within(name + " momentum", m, ref["m"], ref["m_bound"])
    rp = ((p.double() - ref["p"]).abs() / ref["p_bound"]).max().item()
    rm = ((m.double() - ref["m"]).abs() / ref["m_bound"]).max().item()
    return max(rp, rm)


def mta_geometry(numels) -> list:
    """mta_for_each (csrc/optim.cu): the launches of a multi-tensor kernel over tensors of the given sizes.

    Each launch is a dict: ``tensors`` (indices registered, in order; a tensor split across launches is registered again
    in the next one), ``ranges`` (tensor -> [first chunk, last chunk + 1) of MTA_CHUNK elements handled in this launch),
    ``blocks`` (CTAs) and ``reason`` - why the launch was flushed: "tensors" (MTA_TENSORS registered), "blocks"
    (MTA_BLOCKS CTAs) or "end" (the list ran out).  Zero-size tensors are skipped."""
    launches = []
    cur = dict(tensors=[], ranges={}, blocks=0)

    def flush(reason):
        nonlocal cur
        if cur["blocks"] > 0:
            cur["reason"] = reason
            launches.append(cur)
        cur = dict(tensors=[], ranges={}, blocks=0)

    for i, n in enumerate(int(x) for x in numels):
        if n == 0:
            continue
        chunks = cdiv(n, MTA_CHUNK)
        c = 0
        while c < chunks:
            if len(cur["tensors"]) == MTA_TENSORS or cur["blocks"] == MTA_BLOCKS:
                flush("tensors" if len(cur["tensors"]) == MTA_TENSORS else "blocks")
            take = min(chunks - c, MTA_BLOCKS - cur["blocks"])
            cur["tensors"].append(i)
            cur["ranges"][i] = (c, c + take)
            cur["blocks"] += take
            c += take
    flush("end")
    return launches


def sgd_flat_geometry(n: int, sms: int) -> dict:
    """fused_sgd_flat: 8 elements per thread-iteration, 256 threads, grid = min(ceil(n/8 / 256), 8 * SMs); a thread takes
    up to ``iters`` grid-stride iterations."""
    nvec = n // 8
    grid = min(cdiv(nvec, 256), sms * 8)
    return dict(grid=grid, iters=cdiv(nvec, grid * 256), nvec=nvec)


def wire_round(src: torch.Tensor, scale: float, wire) -> torch.Tensor:
    """What pack writes for ``src``: fp32(src) * fp32(scale), rounded to nearest even into the wire dtype (torch's casts
    round like __float2bfloat16_rn / __float2half_rn, including fp16 overflow to +-inf and fp16 subnormals)."""
    return (src.float() * float(scale)).to(wire)


def assert_bits_equal(name: str, got: torch.Tensor, ref: torch.Tensor) -> None:
    """Bitwise equality of two tensors of the same floating dtype (any NaN equals any NaN)."""
    assert got.dtype == ref.dtype, "%s: dtype %s != %s" % (name, got.dtype, ref.dtype)
    g, r = got.reshape(-1), ref.reshape(-1)
    ib = {2: torch.int16, 4: torch.int32, 8: torch.int64}[g.element_size()]
    diff = (g.view(ib) != r.view(ib)) & ~(torch.isnan(g) & torch.isnan(r))
    n = int(diff.sum())
    if n:
        i = int(diff.to(torch.int8).argmax())
        raise AssertionError("%s: %d of %d elements differ bitwise; first at flat index %d: got %r, expected %r"
                             % (name, n, g.numel(), i, g[i].item(), r[i].item()))


# ---------------------------------------------------------------------------------------------------------- collectives
# csrc/collectives.cu: 512 threads per CTA, 16-byte units; one-shot and reduce-to-caller keep 8 units in flight per thread,
# push_range 4; the two-shot P2P reduce is a single grid-stride loop.
COLL_THREADS = 512
ONESHOT_U, REDUCE_U, PUSH_U = 8, 8, 4


def allreduce_ref(per_rank_wire, wire=None, scale: float = 1.0, prepacked: bool = False) -> torch.Tensor:
    """The P2P reduce contract of every rank: the fp32 sum, in rank order 0..W-1 starting from +0.0, of the values each
    rank put on the wire; with ``prepacked`` (the scale was not applied by a pack pass) the fp32 product with fp32(scale);
    then one rounding to the wire dtype.  Inputs are the per-rank wire tensors (same shape and dtype)."""
    wire = per_rank_wire[0].dtype if wire is None else wire
    acc = torch.zeros(per_rank_wire[0].shape, dtype=torch.float32, device=per_rank_wire[0].device)
    for v in per_rank_wire:
        acc = acc + v.float()
    if prepacked:
        acc = acc * torch.tensor(scale, dtype=torch.float32, device=acc.device)
    return acc.to(wire)


def staggered_ref(per_rank_wire, rank: int) -> torch.Tensor:
    """Host model of a reduction that starts at the caller's own rank, p = (rank + i) mod W: the order the P2P reduce
    used before it summed in rank order.  Kept to show that the bitwise checks can tell the two orders apart."""
    W = len(per_rank_wire)
    acc = torch.zeros(per_rank_wire[0].shape, dtype=torch.float32, device=per_rank_wire[0].device)
    for i in range(W):
        acc = acc + per_rank_wire[(rank + i) % W].float()
    return acc.to(per_rank_wire[0].dtype)


def slice_owner(layout, pos):
    """Rank that reduces arena element ``pos`` (int or int64 tensor) in the two-shot kernel: CTA b = pos // block_elems
    owns [b * block_elems, (b + 1) * block_elems) and rank r owns the r-th of its ``world`` equal slices."""
    slice_elems = layout.block_elems // layout.world
    return (pos % layout.block_elems) // slice_elems


def loop_units(units: int, U: int, threads: int = COLL_THREADS) -> dict:
    """How a CTA's ``units`` 16-byte units split between an unrolled main loop (``for (u = tid; u + (U-1)*T < units;
    u += U*T)``) and the single-unit tail loop that follows it."""
    main = tail = 0
    for t in range(min(threads, units)):
        n = 0 if t + (U - 1) * threads >= units else (units - (U - 1) * threads - 1 - t) // (U * threads) + 1
        main += n * U
        tail += len(range(t + n * U * threads, units, threads))
    assert main + tail == units
    return dict(units=units, main_units=main, tail_units=tail)


def oneshot_units(layout, wire_bytes: int) -> dict:
    """oneshot_allreduce_kernel (and reduce_to_caller_kernel, same U): every rank reduces the whole CTA range."""
    return loop_units(layout.block_elems * wire_bytes // 16, ONESHOT_U)


def push_units(layout, wire_bytes: int) -> dict:
    """push_range of fused_broadcast_kernel / push_kernel."""
    return loop_units(layout.block_elems * wire_bytes // 16, PUSH_U)


def twoshot_units(layout, wire_bytes: int) -> dict:
    """fused_allreduce_kernel (P2P): each rank reduces its slice of every CTA range, one unit per loop iteration."""
    units = layout.block_elems // layout.world * wire_bytes // 16
    return dict(units=units, main_units=units, tail_units=0, iters=cdiv(units, COLL_THREADS))


def ll_allreduce_ref(per_rank_in, scale: float) -> torch.Tensor:
    """ll_allreduce_kernel: slot s is the fp32 sum over sources in rank order (from +0.0) times fp32(scale)."""
    acc = torch.zeros_like(per_rank_in[0], dtype=torch.float32)
    for v in per_rank_in:
        acc = acc + v.float()
    return acc * torch.tensor(scale, dtype=torch.float32, device=acc.device)


def metrics_mean_bound(vals: torch.Tensor, world: int, got: torch.Tensor) -> tuple:
    """metrics_kernel's cross-rank mean of ``vals`` [world, 3] (fp32 values the ranks sent): returns the fp64 mean and
    a bound.  Lane l < 3W of warp 0 takes term l, and l + 32 when 3W > 32, then a 5-level xor-shuffle tree: depth
    cdiv(3W, 32) + 5 additions.  The division by ``world`` is a --use_fast_math '/', within 2 ulp of the result."""
    v = vals.double()
    depth = cdiv(3 * world, 32) + 5
    ref = v.sum(0) / world
    return ref, 1.01 * depth * U32 * v.abs().sum(0) / world + 2 * ulp(got, torch.float32)


def topk_correct_ref(logits: torch.Tensor, target: torch.Tensor, ks=(1, 5)) -> list:
    """utils/meters.accuracy's rule as exact integers: sample i is top-k correct iff its target lies in [0, classes) and
    fewer than k logits are strictly greater than the target logit (16-bit and fp32 logits are exact in float64)."""
    x = logits.double()
    C = x.size(1)
    valid = (target >= 0) & (target < C)
    tv = x.gather(1, target.clamp(0, max(C - 1, 0)).view(-1, 1))
    rank = (x > tv).sum(1)
    return [int((valid & (rank < k)).sum()) for k in ks]
