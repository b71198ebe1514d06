"""The fused optimizer step, loss scaling, gradient wire and metric kernels against float64 / exact references at ResNet-50
parameter shapes (161 tensors, 25,557,032 elements), with launch-geometry assertions and negative controls.

Covers every kernel between "autograd produced a gradient" and "the weights changed": pack / unpack and the non-finite
test of ``fused_allreduce_kernel`` (``csrc/collectives.cu``), ``fused_sgd_flat``, ``fused_sgd_multi``,
``multi_tensor_scale``, ``multi_tensor_axpby``, ``amp_update_scale`` (``csrc/optim.cu``) and ``metrics_kernel``.
References and bounds live in tests/_fp64.py; run with ``-s`` to see the largest error / bound ratio of each checker."""
import functools
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _fp64 as R  # noqa: E402

pytestmark = pytest.mark.gpu

DEV = "cuda"
F32, BF16, F16 = torch.float32, torch.bfloat16, torch.float16
CL = torch.channels_last
WIRE_DT = {"fp32": F32, "bf16": BF16, "fp16": F16}
RATIOS = {}


def C():
    from pytorch_distributed_b200 import _ext
    return _ext.lib()


def _ratio(name, r):
    RATIOS[name] = max(RATIOS.get(name, 0.0), r)


@pytest.fixture(scope="module", autouse=True)
def _report_ratios():
    yield
    for k in sorted(RATIOS):
        print("max error / bound  %-28s %.3f" % (k, RATIOS[k]))


@functools.lru_cache(maxsize=1)
def r50_shapes():
    from pytorch_distributed_b200.models import create_model
    shapes = [tuple(p.shape) for p in create_model("resnet50").parameters()]
    assert len(shapes) == 161 and sum(math.prod(s) for s in shapes) == 25_557_032
    return shapes


def r50_flat_size():
    from pytorch_distributed_b200.parallel import plan as P
    return P.tensor_layout([math.prod(s) for s in r50_shapes()])[1]


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def hyper_t(lr=0.1, mom=0.9, wd=1e-4, damp=0.0, gmul=1.0, pending=0.0):
    return torch.tensor([lr, mom, wd, damp, gmul, pending, 0, 0], dtype=F32, device=DEV)


def reduced(w: torch.Tensor) -> torch.Tensor:
    """The world-1 reduce phase sums 0 + v in fp32: every value is kept exactly except -0, which becomes +0."""
    return torch.where(w == 0, torch.zeros_like(w), w)


# ================================================================================================ fused_sgd_flat
BIG = [70000.0, -70000.0, 65504.0, -65504.0, 65519.0, 65520.0, -65520.0, 1.0e5, 3.0e38, -3.0e38]


def _flat_state(n, gdt, gmul, seed=0, steps=2):
    g = torch.Generator(device=DEV).manual_seed(seed)
    master = torch.randn(n, device=DEV, generator=g)
    master[:len(BIG)] = torch.tensor(BIG, device=DEV)        # fp16 copies of these are +-inf / the largest finite values
    mom = torch.randn(n, device=DEV, generator=g) * 0.1
    grads = [(torch.randn(n, device=DEV, generator=g) * (0.01 / gmul)).to(gdt) for _ in range(steps)]
    return master, mom, grads


def _flat_steps(name, gdt, cdt, hyper, nesterov, n=None):
    n = n or r50_flat_size()
    hv = hyper[:5].tolist()
    master, mom, grads = _flat_state(n, gdt, hv[4])
    copy = torch.zeros(n, dtype=cdt, device=DEV) if cdt is not None else None
    for step, g in enumerate(grads):
        p0, m0 = master.clone(), mom.clone()
        C().fused_sgd_flat(g, master, mom, copy, hyper, None, nesterov, step == 0)
        ref = R.sgd_step_fp64(p0, m0, g, hv, nesterov, step == 0)
        _ratio(name, R.check_sgd("%s step %d" % (name, step), master, mom, ref))
        if copy is not None:
            R.assert_bits_equal("%s copy" % name, copy, master.to(cdt))
    return master, mom, copy


FLAT_PAIRS = [(g, c) for g in (F32, BF16, F16) for c in (None, BF16, F16)]


@pytest.mark.parametrize("gdt,cdt", FLAT_PAIRS, ids=lambda d: str(d).replace("torch.", ""))
def test_fused_sgd_flat_dtype_pairs_resnet50(gdt, cdt):
    n = r50_flat_size()
    geo = R.sgd_flat_geometry(n, sms())
    assert geo["iters"] > 1, geo          # every thread takes several grid-stride iterations
    master, _, copy = _flat_steps("sgd_flat", gdt, cdt, hyper_t(), False, n)
    if cdt == F16:
        assert torch.isinf(copy[:len(BIG)].float()).sum() >= 4          # masters beyond 65504 give +-inf copies


HYPER_CASES = {
    "nesterov": (dict(), True),
    "dampening": (dict(damp=0.1), False),
    "momentum0": (dict(mom=0.0), False),
    "wd0": (dict(wd=0.0), False),
    "gmul_2^-16": (dict(gmul=2.0 ** -16), False),
    "nesterov_gmul_2^-16_wd0": (dict(gmul=2.0 ** -16, wd=0.0), True),
}


@pytest.mark.parametrize("case", list(HYPER_CASES))
def test_fused_sgd_flat_hyper_cases(case):
    kw, nesterov = HYPER_CASES[case]
    _flat_steps("sgd_flat", F16 if "gmul" in case else BF16, F16 if "gmul" in case else BF16, hyper_t(**kw), nesterov)


@pytest.mark.parametrize("cdt", [F16, BF16])
def test_fused_sgd_flat_found_inf_leaves_state_bitwise(cdt):
    n = r50_flat_size()
    master, mom, grads = _flat_state(n, F16, 1.0)
    copy = master.to(cdt)
    before = [t.clone() for t in (master, mom, copy)]
    flag = torch.ones(1, dtype=torch.int32, device=DEV)
    for first in (True, False):
        C().fused_sgd_flat(grads[0], master, mom, copy, hyper_t(pending=1.0), flag, False, first)
    for nm, a, b in zip(("master", "momentum", "copy"), (master, mom, copy), before):
        R.assert_bits_equal("skipped step " + nm, a, b)


def test_fused_sgd_flat_bucket_slices_match_one_launch():
    """The overlap path applies the update slice by slice (FusedSGD._apply_slice) at bucket offsets: same bits."""
    from pytorch_distributed_b200.parallel import plan as P
    offs, n = P.tensor_layout([math.prod(s) for s in r50_shapes()])
    master, mom, grads = _flat_state(n, BF16, 1.0)
    copy = master.to(BF16)
    whole = [t.clone() for t in (master, mom, copy)]
    hyper = hyper_t()
    cuts = [0, offs[3], offs[40], offs[90], offs[150], offs[160], n]
    for first, g in zip((True, False), grads):
        C().fused_sgd_flat(g, whole[0], whole[1], whole[2], hyper, None, False, first)
        for a, b in zip(cuts, cuts[1:]):
            assert a % 8 == 0 and (b - a) % 8 == 0
            C().fused_sgd_flat(g[a:b], master[a:b], mom[a:b], copy[a:b], hyper, None, False, first)
    for nm, x, y in zip(("master", "momentum", "copy"), (master, mom, copy), whole):
        R.assert_bits_equal("sliced " + nm, x, y)


def test_fused_sgd_flat_graph_replay_reads_edited_hyper():
    """Captured once; lr and gmul edited in place between replays: each replay matches fp64 with the new values."""
    n = r50_flat_size()
    master, mom, grads = _flat_state(n, F16, 1.0, steps=1)
    copy = master.to(F16)
    hyper = hyper_t()
    C().fused_sgd_flat(grads[0], master, mom, copy, hyper, None, False, True)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        C().fused_sgd_flat(grads[0], master, mom, copy, hyper, None, False, False)
    for lr, gmul in ((0.1, 1.0), (0.025, 0.5), (0.3, 2.0 ** -16), (0.0, 1.0)):
        hyper[0].fill_(lr)
        hyper[4].fill_(gmul)
        p0, m0 = master.clone(), mom.clone()
        graph.replay()
        ref = R.sgd_step_fp64(p0, m0, grads[0], hyper[:5].tolist(), False, False)
        _ratio("sgd_flat graph", R.check_sgd("graph lr=%g gmul=%g" % (lr, gmul), master, mom, ref))
        R.assert_bits_equal("graph copy", copy, master.to(F16))
    R.assert_bits_equal("lr 0 leaves the master", master, p0)


def test_sgd_checkers_reject_edited_results():
    n = 1 << 16
    master, mom, grads = _flat_state(n, BF16, 1.0, steps=1)
    p0, m0 = master.clone(), mom.clone()
    copy = torch.zeros(n, dtype=F16, device=DEV)
    hyper = hyper_t()
    C().fused_sgd_flat(grads[0], master, mom, copy, hyper, None, False, False)
    ref = R.sgd_step_fp64(p0, m0, grads[0], hyper[:5].tolist(), False, False)
    R.check_sgd("ok", master, mom, ref)
    bad = master.clone()
    i = 1234
    bad[i] = bad[i] + 2 * R.ulp(bad[i:i + 1], F32)[0].float()
    with pytest.raises(AssertionError, match="master"):
        R.check_sgd("master + 2 ulp", bad, mom, ref)
    badc = copy.clone()
    cf = copy.float()
    # an element whose copy was rounded, finite and non-zero: move it to the other rounding candidate
    j = int(((cf != master) & torch.isfinite(cf) & (cf != 0) & (master.abs() < 6e4)).nonzero()[0])
    up = bool(cf[j] < master[j])                            # the other candidate lies above the copy
    badc.view(torch.int16)[j] += 1 if up == bool(cf[j] > 0) else -1
    assert (badc[j].float() - master[j]).sign() == -(cf[j] - master[j]).sign()
    with pytest.raises(AssertionError, match="bitwise"):
        R.assert_bits_equal("copy rounded the other way", badc, master.to(F16))


# ================================================================================================ fused_sgd_multi
def _r50_lists(gdt, seed=0, gscale=0.01):
    g = torch.Generator(device=DEV).manual_seed(seed)
    ps = [torch.randn(s, device=DEV, generator=g) for s in r50_shapes()]
    ms = [torch.randn(s, device=DEV, generator=g) * 0.1 for s in r50_shapes()]
    gs = [[(torch.randn(s, device=DEV, generator=g) * gscale).to(gdt) for s in r50_shapes()] for _ in range(2)]
    return ps, ms, gs


def _cat(ts):
    return torch.cat([t.reshape(-1) for t in ts])


def test_mta_geometry_reaches_split_and_both_flushes_at_resnet50():
    L = R.mta_geometry([math.prod(s) for s in r50_shapes()])
    reasons = [x["reason"] for x in L]
    assert "tensors" in reasons and "blocks" in reasons
    seen = {}
    for x in L:
        for t in x["tensors"]:
            seen[t] = seen.get(t, 0) + 1
    assert any(v > 1 for v in seen.values())               # a tensor split across two launches
    assert len(L) > 2


@pytest.mark.parametrize("gdt,cdt", [(F32, None), (BF16, None), (F16, None), (F32, BF16), (BF16, BF16), (F16, F16)],
                         ids=lambda d: str(d).replace("torch.", ""))
def test_fused_sgd_multi_resnet50(gdt, cdt):
    """The ResNet-50 list through mta_for_each: 12 launches, a tensor split across launches, flushes by both the 30-tensor
    and the 320-block limit (asserted in the geometry test above).  `cdt` set: fp32 masters with a low-precision model
    copy (FusedSGD._step_group's `low` path)."""
    ps, ms, gs = _r50_lists(gdt)
    copies = [p.to(cdt) for p in ps] if cdt is not None else []
    hyper = hyper_t(lr=0.1, mom=0.9, wd=1e-4, damp=0.1, gmul=0.5)
    hv = hyper[:5].tolist()
    for step, grads in enumerate(gs):
        p0, m0 = _cat(ps), _cat(ms)
        C().fused_sgd_multi(grads, ps, ms, copies, hyper, None, False, step == 0)
        ref = R.sgd_step_fp64(p0, m0, _cat(grads), hv, False, step == 0)
        _ratio("sgd_multi", R.check_sgd("multi step %d" % step, _cat(ps), _cat(ms), ref))
        if cdt is not None:
            R.assert_bits_equal("multi copy", _cat(copies), _cat(ps).to(cdt))


# ================================================================================================ multi_tensor_scale / axpby
SCALE_PAIRS = [(F32, F32), (F16, F32), (BF16, F32), (F32, F16), (F16, F16), (F32, BF16)]


@pytest.mark.parametrize("sdt,ddt", SCALE_PAIRS, ids=lambda d: str(d).replace("torch.", ""))
def test_multi_tensor_scale_resnet50(sdt, ddt):
    g = torch.Generator(device=DEV).manual_seed(3)
    src = [(torch.randn(s, device=DEV, generator=g) * 100).to(sdt) for s in r50_shapes()]
    dst = [torch.empty(s, device=DEV, dtype=ddt) for s in r50_shapes()]
    flag = torch.zeros(1, dtype=torch.int32, device=DEV)
    scale = 0.37
    C().multi_tensor_scale(src, dst, scale, flag)
    assert int(flag.item()) == 0
    x, got = _cat(src), _cat(dst)
    exact = x.double() * float(np.float32(scale))
    tol = R.U32 * exact.abs() + (0.5 * R.ulp(got, ddt) if ddt != F32 else 0) + 2.0 ** -126
    R.assert_within("multi_tensor_scale", got, exact, tol)
    _ratio("multi_tensor_scale", ((got.double() - exact).abs() / tol).max().item())
    R.assert_bits_equal("multi_tensor_scale", got, (x.float() * scale).to(ddt))       # fp32 product, then one cast


@pytest.mark.parametrize("xdt,ydt,odt", [(F32, F32, F32), (F16, F32, F32), (BF16, BF16, F32), (F32, F16, F16)],
                         ids=lambda d: str(d).replace("torch.", ""))
def test_multi_tensor_axpby_resnet50(xdt, ydt, odt):
    g = torch.Generator(device=DEV).manual_seed(4)
    xs = [(torch.randn(s, device=DEV, generator=g) * 10).to(xdt) for s in r50_shapes()]
    ys = [(torch.randn(s, device=DEV, generator=g) * 10).to(ydt) for s in r50_shapes()]
    out = [torch.empty(s, device=DEV, dtype=odt) for s in r50_shapes()]
    flag = torch.zeros(1, dtype=torch.int32, device=DEV)
    a, b = 0.75, -1.3
    C().multi_tensor_axpby(xs, ys, out, a, b, flag)
    assert int(flag.item()) == 0
    ax, by = _cat(xs).double() * float(np.float32(a)), _cat(ys).double() * float(np.float32(b))
    got = _cat(out)
    # a*x and b*y rounded (unless contracted into an FMA), their sum rounded, then one rounding into the output dtype
    tol = 2 * R.U32 * (ax.abs() + by.abs()) + R.U32 * (ax + by).abs() + (0.5 * R.ulp(got, odt) if odt != F32 else 0) + 2.0 ** -126
    R.assert_within("multi_tensor_axpby", got, ax + by, tol)
    _ratio("multi_tensor_axpby", ((got.double() - (ax + by)).abs() / tol).max().item())


def _bad_positions():
    """(tensor, flat element) where one non-finite value is planted: the first element of a tensor, the last element of a
    chunk, and the last element of a tensor registered only in a later launch."""
    numels = [math.prod(s) for s in r50_shapes()]
    L = R.mta_geometry(numels)
    first_launch = L[0]["tensors"]
    multi_chunk = next(t for t in range(len(numels)) if numels[t] > 2 * R.MTA_CHUNK)
    late = next(t for t in L[-1]["tensors"] if all(t not in x["tensors"] for x in L[:-1]))
    assert late not in first_launch
    return [(first_launch[5], 0), (multi_chunk, R.MTA_CHUNK - 1), (late, numels[late] - 1)]


def check_found_inf(name: str, flag: torch.Tensor, want: int) -> None:
    """The overflow flag word holds exactly `want` (1: some tested value was non-finite, 0: none was)."""
    got = int(flag.item())
    assert got == want, "%s: found_inf is %d, expected %d" % (name, got, want)


@pytest.mark.parametrize("value", [math.inf, -math.inf, math.nan])
@pytest.mark.parametrize("op", ["scale", "axpby_x", "axpby_y"])
def test_found_inf_is_set_and_sticky(op, value):
    g = torch.Generator(device=DEV).manual_seed(5)
    clean = [torch.randn(s, device=DEV, generator=g).half() for s in r50_shapes()]
    other = [torch.randn(s, device=DEV, generator=g) for s in r50_shapes()]
    out = [torch.empty(s, device=DEV) for s in r50_shapes()]
    flag = torch.zeros(1, dtype=torch.int32, device=DEV)

    def run(src):
        if op == "scale":
            C().multi_tensor_scale(src, out, 0.5, flag)
        elif op == "axpby_x":
            C().multi_tensor_axpby(src, other, out, 1.0, 1.0, flag)
        else:
            C().multi_tensor_axpby(other, src, out, 1.0, 1.0, flag)

    run(clean)
    check_found_inf("clean", flag, 0)
    for t, i in _bad_positions():
        flag.zero_()
        bad = [x.clone() if k == t else x for k, x in enumerate(clean)]
        bad[t].view(-1)[i] = value
        run(bad)
        check_found_inf("%s %r at tensor %d element %d" % (op, value, t, i), flag, 1)
        run(clean)                                      # a later clean call never clears the flag (sticky OR)
        check_found_inf("%s %r at tensor %d element %d, then clean" % (op, value, t, i), flag, 1)


def test_multi_tensor_scale_tests_inputs_only():
    """Contract: only the INPUTS are tested for non-finite values.  A finite fp32 input whose scaled fp16 output
    overflows is stored as +-inf and does not set found_inf (the unscale pass of amp divides, so it cannot overflow;
    an overflowing cast is the caller's concern)."""
    src = [torch.tensor([1.0, 70000.0, -65520.0, 65504.0], device=DEV)]
    dst = [torch.empty(4, device=DEV, dtype=F16)]
    flag = torch.zeros(1, dtype=torch.int32, device=DEV)
    C().multi_tensor_scale(src, dst, 1.0, flag)
    assert int(flag.item()) == 0
    R.assert_bits_equal("overflowing cast", dst[0], src[0].to(F16))
    assert torch.isinf(dst[0][1:3]).all()


def test_found_inf_checker_rejects_cleared_flag():
    """Negative control of check_found_inf: the flag a real overflow set, cleared after the fact, is rejected."""
    flag = torch.zeros(1, dtype=torch.int32, device=DEV)
    x = [torch.tensor([1.0, math.inf], device=DEV)]
    C().multi_tensor_scale(x, [torch.empty(2, device=DEV)], 1.0, flag)
    check_found_inf("inf input", flag, 1)
    flag.zero_()                                         # edited after the fact
    with pytest.raises(AssertionError, match="found_inf is 0, expected 1"):
        check_found_inf("cleared", flag, 1)


# ================================================================================================ amp_update_scale
def _amp_model(scale, tracker, bad, growth, backoff, interval):
    f = np.float32
    if bad:
        return max(f(scale * f(backoff)), f(1.0)), 0
    t = tracker + 1
    if t >= interval:
        with np.errstate(over="ignore"):
            s = f(scale * f(growth))
        if np.isfinite(s):
            scale = s
        t = 0
    return scale, t


INV_EXACT_MAX = 2.0 ** 126      # above this 1/scale is an fp32 subnormal: see test_amp_inverse_scale_above_2_126


def _inv_ref(scale):
    return np.float32(np.float32(1.0) / scale)


@pytest.mark.parametrize("interval,init", [(2000, 2.0 ** 16), (3, 2.0 ** 16), (3, 2.0 ** 120), (2000, 2.0 ** 127)])
def test_amp_update_scale_matches_apex_rules(interval, init):
    steps = 5000
    rng = np.random.default_rng(interval)
    p_bad = 0.002 if interval == 2000 else 0.3
    bad = (rng.random(steps) < p_bad).astype(np.int32)
    if init >= 2.0 ** 120:
        bad[:100] = 0                                  # grow up to 2^127, where scale * growth is inf: no growth
    if interval == 2000:
        bad[:2500] = 0                                 # long clean runs: growth at exactly 2000 clean steps
        bad[2500:2520] = 1                             # a burst of overflows: backoff down to the 1.0 clamp
    scale = torch.tensor([init], dtype=F32, device=DEV)
    tr = torch.zeros(1, dtype=torch.int32, device=DEV)
    fi = torch.zeros(1, dtype=torch.int32, device=DEV)
    hyper = hyper_t(pending=1.0)
    flags = torch.from_numpy(bad).to(DEV)
    hist = torch.zeros(steps, 4, dtype=torch.float64, device=DEV)
    pend = torch.zeros(steps, dtype=F32, device=DEV)
    for i in range(steps):
        fi.copy_(flags[i:i + 1])
        C().amp_update_scale(scale, tr, fi, 2.0, 0.5, interval, hyper)
        hist[i, 0], hist[i, 1], hist[i, 2], hist[i, 3] = scale[0], tr[0], fi[0], hyper[4]
        pend[i] = hyper[5]
    h = hist.cpu().numpy()
    s, t = np.float32(init), 0
    seen_clamp = seen_inf_cap = False
    for i in range(steps):
        s, t = _amp_model(s, t, bad[i], 2.0, 0.5, interval)
        assert (h[i, 0], h[i, 1], h[i, 2]) == (s, t, 0), (i, h[i], s, t)
        if s <= INV_EXACT_MAX:
            assert np.float32(h[i, 3]) == _inv_ref(s), (i, h[i, 3], s)
        seen_clamp |= bool(bad[i]) and s == 1.0
        with np.errstate(over="ignore"):
            seen_inf_cap |= t == 0 and not bad[i] and not np.isfinite(np.float32(s * np.float32(2.0)))
    first_clean = int(np.argmax(bad == 0))
    p = pend.cpu().numpy()
    assert (p[:first_clean] == 1).all() and (p[first_clean:] == 0).all()     # momentum_pending cleared by the first applied step
    if interval == 3 and init == 2.0 ** 16:
        assert seen_clamp
    if init >= 2.0 ** 120:
        assert seen_inf_cap


@pytest.mark.xfail(reason="known limitation: the extension is built with --use_fast_math, so 1/scale (an fp32 subnormal "
                          "for scale > 2^126) is flushed to 0, and the SGD kernels would flush such a multiplier too; a "
                          "dynamic fp16 loss scale cannot get there without its gradients overflowing first", strict=False)
def test_amp_inverse_scale_above_2_126():
    scale = torch.tensor([2.0 ** 127], dtype=F32, device=DEV)
    tr = torch.zeros(1, dtype=torch.int32, device=DEV)
    fi = torch.zeros(1, dtype=torch.int32, device=DEV)
    hyper = hyper_t()
    C().amp_update_scale(scale, tr, fi, 2.0, 0.5, 2000, hyper)
    assert scale.item() == 2.0 ** 127
    assert np.float32(hyper[4].item()) == _inv_ref(np.float32(2.0 ** 127))


# ================================================================================================ gradient wire, world 1
@pytest.fixture(scope="module")
def comm():
    from pytorch_distributed_b200.parallel.comm import FusedCommunicator
    return FusedCommunicator(device=torch.device(DEV, 0), arena_bytes=768 << 20)


def _wire_grads(sdt, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    ts = []
    for s in r50_shapes():
        t = torch.randn(s, device=DEV, generator=g) * 0.05
        t.view(-1)[: max(1, t.numel() // 16)] *= 1e-4          # fp16 wire subnormals (and -0 from underflow)
        ts.append(t.to(sdt))
    base = (torch.randn(8195, device=DEV, generator=g)).to(sdt)
    ts.append(base[1:8194])                                    # dense, odd element offset: not 16-byte aligned
    assert ts[-1].data_ptr() % 16 != 0
    return ts


WIRE_FORMS = [(F32, "fp16"), (F16, "fp16"), (BF16, "bf16")]


def _check_arena(name, arena, offsets, srcs, scale, wdt, after_reduce):
    for i, (off, t) in enumerate(zip(offsets, srcs)):
        exp = R.wire_round(t.reshape(-1), scale, wdt)
        R.assert_bits_equal("%s tensor %d" % (name, i), arena[off:off + t.numel()], reduced(exp) if after_reduce else exp)


@pytest.mark.parametrize("sdt,wire", WIRE_FORMS, ids=lambda d: str(d).replace("torch.", ""))
def test_wire_pack_unpack_check_inf_bitwise(comm, sdt, wire):
    from pytorch_distributed_b200.parallel.comm import KIND_TWO_SHOT
    wdt = WIRE_DT[wire]
    ts = _wire_grads(sdt)
    orig = [t.clone() for t in ts]
    plan = comm.make_plan([t.numel() for t in ts], wire)
    comm.found_inf.zero_()
    comm.run(plan, ts, KIND_TWO_SHOT, comm.misc_channel, scale=1.0, writeback=True, check_inf=True)
    torch.cuda.synchronize()
    comm.check()
    check_found_inf("clean", comm.found_inf, 0)
    arena = plan.arena_tensor()
    _check_arena("arena", arena, plan.layout.offsets, orig, 1.0, wdt, True)
    for i, (t, o) in enumerate(zip(ts, orig)):                 # writeback: the reduced wire values in the tensor's dtype
        R.assert_bits_equal("writeback %d" % i, t.reshape(-1), reduced(R.wire_round(o.reshape(-1), 1.0, wdt)).to(sdt))
    # negative control: one parameter's slice swapped with its neighbour's
    bad = arena.clone()
    offs = plan.layout.offsets
    k = 10
    n = min(orig[k].numel(), orig[k + 1].numel())
    a, b = bad[offs[k]:offs[k] + n].clone(), bad[offs[k + 1]:offs[k + 1] + n].clone()
    bad[offs[k]:offs[k] + n], bad[offs[k + 1]:offs[k + 1] + n] = b, a
    with pytest.raises(AssertionError, match="bitwise"):
        _check_arena("swapped", bad, offs, orig, 1.0, wdt, True)

    # found_inf is 1 exactly when some packed value is non-finite
    cases = {"clean": (None, 0)}
    if sdt == F32:
        cases["fp32 above 65504 on the fp16 wire"] = (70000.0, 1)
        cases["fp32 65519 rounds to 65504"] = (65519.0, 0)
    cases["inf"] = (math.inf, 1)
    cases["nan"] = (math.nan, 1)
    for nm, (v, want) in cases.items():
        src = [o.clone() for o in orig]
        if v is not None:
            src[-2].view(-1)[-1] = v
        comm.found_inf.zero_()
        comm.run(plan, src, KIND_TWO_SHOT, comm.misc_channel, scale=1.0, writeback=False, check_inf=True)
        check_found_inf(nm, comm.found_inf, want)
    comm.found_inf.zero_()


@pytest.mark.parametrize("wire", ["fp16", "bf16"])
def test_wire_prepacked_rescale(comm, wire):
    """Bucket views (prepacked): the gradients already sit in the arena; scale != 1 is applied to the reduced values with
    one rounding."""
    from pytorch_distributed_b200.parallel.comm import KIND_TWO_SHOT
    wdt = WIRE_DT[wire]
    numels = [math.prod(s) for s in r50_shapes()]
    plan = comm.make_plan(numels, wire)
    arena = plan.arena_tensor()
    g = torch.Generator(device=DEV).manual_seed(7)
    views = []
    for off, s in zip(plan.layout.offsets, r50_shapes()):
        v = arena[off:off + math.prod(s)].view(s)
        v.copy_(torch.randn(s, device=DEV, generator=g) * 3)
        views.append(v)
    pre = [v.clone() for v in views]
    comm.found_inf.zero_()
    scale = 0.37
    comm.run(plan, views, KIND_TWO_SHOT, comm.misc_channel, scale=scale, writeback=False, check_inf=True, prepacked=True)
    torch.cuda.synchronize()
    check_found_inf("clean", comm.found_inf, 0)
    _check_arena("prepacked x%.2f" % scale, arena, plan.layout.offsets, pre, scale, wdt, True)
    comm.found_inf.zero_()


# ================================================================================================ engine level, world 1
@pytest.fixture
def deterministic():
    flags = (torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark)
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    yield
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = flags


def _build(entry, argv):
    from pytorch_distributed_b200 import cli, driver
    from pytorch_distributed_b200.models import create_model
    torch.cuda.set_device(0)
    args = cli.parse_args(entry, ["-a", "resnet50", "-b", "8", "--synthetic", "--image-size", "64", "--quiet"] + argv)
    st = driver.STRATEGIES[entry]() if entry != "distributed" else driver.Strategy()
    torch.manual_seed(0)
    model = create_model(args.arch, num_classes=args.num_classes, fused_bn=args.fused_bn)
    model, opt = st.build(model, args, torch.device(DEV, 0), 0)
    model.train()
    return st, model, opt, args


def _batch(dtype, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(8, 3, 64, 64, device=DEV, generator=g).to(dtype).contiguous(memory_format=CL)
    y = torch.randint(0, 1000, (8,), device=DEV, generator=g)
    return x, y


def mem_flat(t: torch.Tensor) -> torch.Tensor:
    """A dense tensor's elements in memory order (channels_last weights are packed as they lie in memory)."""
    return t.as_strided((t.numel(),), (1,))


def check_arena_per_param(name, arena, eng, after_reduce, grads=None):
    """Each parameter's slice of the arena at param_elem_off holds the wire rounding of that parameter's own gradient,
    in the gradient's memory order."""
    wdt = WIRE_DT[eng.wire]
    for pid, p in enumerate(eng.params):
        g = p.grad if grads is None else grads[pid]
        off = eng.param_elem_off[pid]
        exp = R.wire_round(mem_flat(g), eng.scale, wdt)
        R.assert_bits_equal("%s param %d %s" % (name, pid, tuple(p.shape)), arena[off:off + p.numel()],
                            reduced(exp) if after_reduce else exp)


def _engine_step(st, model, opt, x, y):
    """One training step; returns the flat master / momentum before it and how many flat elements the overlap path
    (FusedSGD._apply_slice behind each bucket's all-reduce) had already updated when backward returned."""
    eng, fs = st.engine, opt._flat
    pre = (fs.master.clone(), fs.momentum.clone())
    if getattr(eng, "bucket_view", False):
        eng.zero_grads()
    else:
        opt.zero_grad()
    out = st.forward(model, x)
    loss = torch.nn.functional.cross_entropy(out.float(), y)
    st.backward(loss, opt)
    applied = opt._ov_applied if opt._ov_active else 0
    opt.step()
    torch.cuda.synchronize()
    return pre, applied


def _check_engine_update(name, opt, pre, first, gmul=1.0):
    fs = opt._flat
    h = opt._hyper[0][0][:5].tolist()
    h[4] = gmul
    g = fs.engine.grad_arena()
    ref = R.sgd_step_fp64(pre[0], pre[1], g, h, bool(opt.param_groups[0]["nesterov"]), first)
    _ratio("engine sgd", R.check_sgd(name, fs.master, fs.momentum, ref))
    if fs.model_copy is not None:
        R.assert_bits_equal(name + " model copy", fs.model_copy, fs.master.to(fs.model_copy.dtype))


ENGINE_MODES = {
    "bf16_model_bf16_wire": ["--no-overlap-optimizer"],
    "fp32_model_bf16_wire": ["--no-overlap-optimizer", "--precision", "fp32"],
    "overlap_backward": [],
    "bucket_view": ["--no-overlap-optimizer", "--bucket-view"],
}


@pytest.mark.parametrize("mode", list(ENGINE_MODES))
def test_ddp_every_parameter_gets_its_own_update(mode, deterministic):
    st, model, opt, args = _build("distributed", ENGINE_MODES[mode])
    eng = st.engine
    assert eng.wire == "bf16" and len(eng.params) == 161
    x, y = _batch(st.input_dtype)
    if mode == "overlap_backward":
        assert opt._overlap
    for step in range(2):
        if step == 0 and not opt.is_flat:
            # binds at its first step when the engine was created later; master/momentum start from the parameters
            opt._try_bind()
        assert opt.is_flat
        pre, applied = _engine_step(st, model, opt, x, y)
        # overlap mode: every bucket was updated behind its all-reduce during backward, step() only joined
        assert applied == (opt._flat.master.numel() if mode == "overlap_backward" else 0), (mode, applied)
        assert eng.writeback is False
        check_arena_per_param("%s step %d" % (mode, step), eng.grad_arena(), eng, False)
        _check_engine_update("%s step %d" % (mode, step), opt, pre, step == 0)
    # negative control: a neighbour's slice in place of a parameter's own
    bad = eng.grad_arena().clone()
    o1, o2 = eng.param_elem_off[20], eng.param_elem_off[21]
    n = min(eng.params[20].numel(), eng.params[21].numel())
    bad[o1:o1 + n], bad[o2:o2 + n] = eng.grad_arena()[o2:o2 + n].clone(), eng.grad_arena()[o1:o1 + n].clone()
    with pytest.raises(AssertionError, match="bitwise"):
        check_arena_per_param("swapped", bad, eng, False)


def test_apex_o2_overflow_skip_then_clean_steps_and_graph_replay(deterministic):
    """apex_distributed at O2 (fp16 model, fp32 masters, fp16 wire, dynamic loss scale with the non-finite test in the
    all-reduce): an overflow forced by a gradient hook skips the step bitwise, halves the scale and clears the flag; the
    next clean steps apply gmul = 1/scale (the first one initialises the momentum); a CUDA-graph replay does the same."""
    from pytorch_distributed_b200 import driver
    from pytorch_distributed_b200.utils.meters import AverageMeter
    st, model, opt, args = _build("apex_distributed", ["--precision", "fp16", "--opt-level", "O2"])
    eng, scaler = st.engine, opt._amp
    assert eng.check_inf and eng.wire == "fp16" and scaler.dynamic
    scaler.scale.fill_(2.0 ** 10)                       # far from a natural fp16 overflow at this size
    x, y = _batch(F16)
    # overflow on the very first step: nothing may change
    target = eng.params[100]
    h = target.register_hook(lambda g: torch.full_like(g, math.inf))
    opt._try_bind()
    assert opt.is_flat
    fs = opt._flat
    state0 = [t.clone() for t in (fs.master, fs.momentum, fs.model_copy)]
    _, applied = _engine_step(st, model, opt, x, y)
    assert applied == 0                                 # under a loss scaler the update waits for the whole step
    h.remove()
    for nm, a, b in zip(("master", "momentum", "model copy"), (fs.master, fs.momentum, fs.model_copy), state0):
        R.assert_bits_equal("skipped " + nm, a, b)
    assert scaler.scale.item() == 2.0 ** 9 and int(scaler.tracker.item()) == 0 and int(scaler.found_inf.item()) == 0
    # clean steps
    for step in range(2):
        s = scaler.scale.item()
        pre, _ = _engine_step(st, model, opt, x, y)
        assert int(scaler.found_inf.item()) == 0 and int(scaler.tracker.item()) == step + 1
        check_arena_per_param("apex step %d" % step, eng.grad_arena(), eng, True)
        _check_engine_update("apex step %d" % step, opt, pre, step == 0, gmul=1.0 / s)
    # one step replayed from a CUDA graph (captured and replayed by the first call)
    metrics = driver.MetricPipeline(st.comm, torch.device(DEV, 0), (AverageMeter("L"), AverageMeter("A1"), AverageMeter("A5")), reduce=True)
    step = driver.TrainStep(st, model, torch.nn.CrossEntropyLoss().to(DEV), opt, metrics, use_graph=True, warmup=0)
    s = scaler.scale.item()
    pre = (fs.master.clone(), fs.momentum.clone())
    step(x, y)
    torch.cuda.synchronize()
    assert step.graph is not None
    assert int(scaler.found_inf.item()) == 0
    check_arena_per_param("apex graph replay", eng.grad_arena(), eng, True)
    _check_engine_update("apex graph replay", opt, pre, False, gmul=1.0 / s)
    metrics.drain()


# ================================================================================================ suspected defects
def test_debug_poison_with_dynamic_loss_scaling_still_applies_steps(monkeypatch, deterministic):
    """PTD_DEBUG_POISON=1 fills the gradient arena with NaN after each step.  The alignment padding is never packed, so
    NaN left there would trip the all-reduce's non-finite test on every later step: every step skipped, the scale
    halving each time."""
    from pytorch_distributed_b200 import driver
    from pytorch_distributed_b200.utils.meters import AverageMeter
    monkeypatch.setattr(driver, "_POISON", True)
    st, model, opt, args = _build("apex_distributed", ["--precision", "fp16", "--opt-level", "O2"])
    scaler = opt._amp
    scaler.scale.fill_(2.0 ** 10)
    metrics = driver.MetricPipeline(st.comm, torch.device(DEV, 0), (AverageMeter("L"), AverageMeter("A1"), AverageMeter("A5")), reduce=True)
    step = driver.TrainStep(st, model, torch.nn.CrossEntropyLoss().to(DEV), opt, metrics, use_graph=False)
    x, y = _batch(F16)
    masters = []
    for _ in range(4):
        step(x, y)
        torch.cuda.synchronize()
        masters.append(opt._flat.master.clone())
    metrics.drain()
    assert scaler.scale.item() == 2.0 ** 10 and int(scaler.tracker.item()) == 4, (scaler.scale.item(), int(scaler.tracker.item()))
    assert all(not torch.equal(a, b) for a, b in zip(masters, masters[1:]))


def _torch_sgd_after_skipped_first(ps0, grads, inv_scales, lr, mom, damp, wd):
    """fp64 torch.optim.SGD semantics under a loss scaler: the overflowed first step is not applied, so the momentum is
    initialised by the first APPLIED step."""
    ps = [torch.nn.Parameter(p.double().clone()) for p in ps0]
    opt = torch.optim.SGD(ps, lr=lr, momentum=mom, dampening=damp, weight_decay=wd)
    for gs, inv in zip(grads, inv_scales):
        for p, g in zip(ps, gs):
            p.grad = g.double() * inv
        opt.step()
    return [p.detach() for p in ps], [opt.state[p]["momentum_buffer"] for p in ps]


def test_skipped_first_step_multi_tensor_dampening():
    from pytorch_distributed_b200.ops.fused_sgd import FusedSGD
    from pytorch_distributed_b200.parallel.amp import LossScaler
    g = torch.Generator(device=DEV).manual_seed(11)
    shapes = [(64, 3, 7, 7), (3 * R.MTA_CHUNK + 5,), (1000,)]
    params = [torch.nn.Parameter(torch.randn(s, device=DEV, generator=g)) for s in shapes]
    params.append(torch.nn.Parameter(torch.randn(300, device=DEV, generator=g).to(BF16)))   # the `low` (model copy) path
    ps0 = [p.detach().float().clone() for p in params]
    opt = FusedSGD(params, lr=0.1, momentum=0.9, dampening=0.1, weight_decay=1e-4)
    scaler = LossScaler(torch.device(DEV), init_scale=2.0 ** 8)
    opt._amp = scaler
    grads = [[(torch.randn(p.shape, device=DEV, generator=g) * 256).to(p.dtype) for p in params] for _ in range(3)]
    inv = []
    for k, gs in enumerate(grads):
        for p, gr in zip(params, gs):
            p.grad = gr.clone()
        inv.append(1.0 / scaler.scale.item())
        if k == 0:
            scaler.found_inf.fill_(1)                    # the first step overflows
        opt.step()
    torch.cuda.synchronize()
    ref_p, ref_m = _torch_sgd_after_skipped_first(ps0, grads[1:], inv[1:], 0.1, 0.9, 0.1, 1e-4)
    for i, p in enumerate(params):
        master = opt.state[p].get("master", p.detach())
        mom = opt.state[p]["momentum_buffer"]
        tol = 1e-6 * (1 + ref_m[i].abs())
        R.assert_within("momentum %d" % i, mom, ref_m[i], tol)
        R.assert_within("master %d" % i, master, ref_p[i], 1e-6 * (1 + ref_p[i].abs()))


@pytest.mark.parametrize("skip_first", [False, True])
@pytest.mark.parametrize("loss_scale", ["dynamic", 128.0])
def test_multi_tensor_param_groups_under_loss_scaler(loss_scale, skip_first):
    """Each param group has its own hyper tensor; the loss scaler must keep every group's momentum_pending and 1/scale
    right, not only those of the group stepped last.  Four clean steps (after an overflowed first one when
    `skip_first`), both groups against fp64 torch.optim.SGD with the same param groups."""
    from pytorch_distributed_b200.ops.fused_sgd import FusedSGD
    from pytorch_distributed_b200.parallel.amp import LossScaler
    g = torch.Generator(device=DEV).manual_seed(16)
    groups = [[(64, 3, 7, 7), (2 * R.MTA_CHUNK + 3,)], [(1000,), (257, 3)]]
    params = [[torch.nn.Parameter(torch.randn(s, device=DEV, generator=g)) for s in shp] for shp in groups]
    cfg = [dict(lr=0.1, dampening=0.0), dict(lr=0.03, dampening=0.1)]
    ps0 = [[p.detach().clone() for p in ps] for ps in params]
    opt = FusedSGD([dict(params=ps, **c) for ps, c in zip(params, cfg)], lr=0.1, momentum=0.9, weight_decay=1e-4)
    scaler = LossScaler(torch.device(DEV), loss_scale=loss_scale, init_scale=2.0 ** 8)
    opt._amp = scaler
    steps = 5 if skip_first else 4
    grads = [[[torch.randn(p.shape, device=DEV, generator=g) * 256 for p in ps] for ps in params] for _ in range(steps)]
    inv = []
    for k in range(steps):
        for ps, gs in zip(params, grads[k]):
            for p, gr in zip(ps, gs):
                p.grad = gr.clone()
        inv.append(1.0 / scaler.scale.item())
        if skip_first and k == 0:
            scaler.found_inf.fill_(1)
        opt.step()
    torch.cuda.synchronize()
    first_applied = 1 if skip_first else 0
    ref = [[torch.nn.Parameter(p.double().clone()) for p in ps] for ps in ps0]
    topt = torch.optim.SGD([dict(params=ps, **c) for ps, c in zip(ref, cfg)], lr=0.1, momentum=0.9, weight_decay=1e-4)
    for k in range(first_applied, steps):
        for ps, gs in zip(ref, grads[k]):
            for p, gr in zip(ps, gs):
                p.grad = gr.double() * inv[k]
        topt.step()
    for gi, (ps, rs) in enumerate(zip(params, ref)):
        for i, (p, r) in enumerate(zip(ps, rs)):
            rm = topt.state[r]["momentum_buffer"]
            R.assert_within("group %d momentum %d" % (gi, i), opt.state[p]["momentum_buffer"], rm, 1e-6 * (1 + rm.abs()))
            R.assert_within("group %d param %d" % (gi, i), p.detach(), r.detach(), 1e-6 * (1 + r.detach().abs()))


def test_skipped_first_step_flat_dampening(deterministic):
    from pytorch_distributed_b200.ops.fused_sgd import FusedSGD
    from pytorch_distributed_b200.parallel.amp import LossScaler
    from pytorch_distributed_b200.parallel.comm import FusedCommunicator
    from pytorch_distributed_b200.parallel.ddp import DistributedDataParallel
    torch.manual_seed(12)
    net = torch.nn.Sequential(torch.nn.Linear(64, 256), torch.nn.ReLU(), torch.nn.Linear(256, 10)).to(DEV)
    cm = FusedCommunicator(device=torch.device(DEV, 0), arena_bytes=32 << 20)
    ddp = DistributedDataParallel(net, comm=cm, wire_dtype="fp32", check_inf=True)
    opt = FusedSGD(ddp.parameters(), lr=0.1, momentum=0.9, dampening=0.1, weight_decay=1e-4)
    assert opt.is_flat
    scaler = LossScaler(torch.device(DEV), init_scale=2.0 ** 8)
    scaler.rebind_found_inf(cm.found_inf)
    opt._amp = scaler
    ps0 = [p.detach().clone() for p in net.parameters()]
    x, y = torch.randn(32, 64, device=DEV), torch.randint(0, 10, (32,), device=DEV)
    grads, inv = [], []
    for k in range(3):
        h = net[0].weight.register_hook(lambda g: torch.full_like(g, math.inf)) if k == 0 else None
        opt.zero_grad()
        s = scaler.scale.item()
        (torch.nn.functional.cross_entropy(ddp(x), y) * s).backward()
        if h is not None:
            h.remove()
        grads.append([p.grad.clone() for p in net.parameters()])
        inv.append(1.0 / s)
        opt.step()
        torch.cuda.synchronize()
        if k == 0:
            assert scaler.scale.item() == s / 2          # skipped
    ref_p, ref_m = _torch_sgd_after_skipped_first(ps0, grads[1:], inv[1:], 0.1, 0.9, 0.1, 1e-4)
    for i, p in enumerate(net.parameters()):
        R.assert_within("momentum %d" % i, opt.state[p]["momentum_buffer"], ref_m[i], 1e-6 * (1 + ref_m[i].abs()))
        R.assert_within("master %d" % i, p.detach(), ref_p[i], 1e-6 * (1 + ref_p[i].abs()))


# ================================================================================================ metrics_kernel, world 1
def _metric_counts(out, batch):
    return [int(round(out[k].item() * batch / 100.0)) for k in (1, 2)]


def _check_metrics(name, out, logits, target, loss):
    B = logits.size(0)
    want = R.topk_correct_ref(logits, target)
    got = _metric_counts(out, B)
    assert got == want, "%s: top-1/top-5 counts %s, reference %s" % (name, got, want)
    assert out[0].item() == (loss.item() if loss is not None else 0.0)


@pytest.mark.parametrize("dtype", [F32, BF16, F16], ids=lambda d: str(d).replace("torch.", ""))
def test_metrics_kernel_counts_exactly(comm, dtype):
    g = torch.Generator(device=DEV).manual_seed(13)
    out = torch.zeros(4, device=DEV)
    for B in (1, 31, 32, 33, 256, 1025):
        for Cn in (1, 4, 5, 31, 33, 1000, 1001):
            logits = torch.randn(B, Cn, device=DEV, generator=g).to(BF16).to(dtype)   # bf16 quantisation: many ties
            target = torch.randint(0, Cn, (B,), device=DEV, generator=g)
            rows = torch.arange(B, device=DEV)
            tie = torch.randint(0, Cn, (B,), device=DEV, generator=g)
            logits[rows[::3], tie[::3]] = logits[rows[::3], target[::3]]              # ties at the target value
            logits[rows[1::4], target[1::4]] += 4                                     # some correct ones
            loss = torch.rand((), device=DEV, generator=g) if B % 2 else None
            comm.metrics(logits, target, loss, out)
            _check_metrics("B=%d C=%d" % (B, Cn), out, logits, target, loss)
    comm.check()


def test_metrics_kernel_strided_rows_and_negative_control(comm):
    g = torch.Generator(device=DEV).manual_seed(14)
    full = torch.randn(256, 1024, device=DEV, generator=g).to(BF16)
    logits = full[:, :1000]
    assert not logits.is_contiguous()
    target = torch.randint(0, 1000, (256,), device=DEV, generator=g)
    logits[torch.arange(0, 256, 2, device=DEV), target[::2]] += 3
    full[:, 1000:] = 100                                    # beyond the row: must not be counted
    out = torch.zeros(4, device=DEV)
    comm.metrics(logits, target, None, out)
    _check_metrics("strided", out, logits, target, None)
    bad = out.clone()
    bad[1] += 100.0 / 256                                   # one top-1 count off by one
    with pytest.raises(AssertionError, match="counts"):
        _check_metrics("edited", bad, logits, target, None)


@pytest.mark.parametrize("classes", [4, 1000])
def test_metrics_kernel_out_of_range_target_is_incorrect(comm, classes):
    g = torch.Generator(device=DEV).manual_seed(15)
    logits = torch.randn(64, classes, device=DEV, generator=g)
    target = torch.randint(0, classes, (64,), device=DEV, generator=g)
    target[0], target[1], target[2] = classes, -1, classes + 7
    out = torch.zeros(4, device=DEV)
    comm.metrics(logits, target, None, out)
    _check_metrics("out-of-range targets", out, logits, target, None)
