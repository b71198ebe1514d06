"""fp16 and autocast on the wgmma 1x1-conv GEMM and the stem im2col + GEMM path.

Kernel cases run the extension entry points against the float64 references of tests/_fp64.py at ResNet-50 batch-256
shapes and at the geometry edges of launch_gemm, including the fp16 overflow contract (values >= 65520 are stored as
+-inf and make that channel's sums non-finite).  Model cases check which path a ResNet-50 training forward takes in each
precision mode (a model cast to bf16 / fp16, autocast over fp32 weights, the apex opt levels), and judge the fused path
against the cuDNN path of the same precision with a plain fp32 PyTorch oracle.
"""
import copy
import os
import sys

import pytest
import torch

TESTS = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, TESTS)
import _fp64 as R  # noqa: E402
from test_gpu_fp64 import EPS, GEMM_EDGES, RESNET50_1X1, _bn_params, _equal_all, _gen, _stem_forward, sms  # noqa: E402

pytestmark = pytest.mark.gpu

CL = torch.channels_last
DEV = "cuda"
F16 = torch.float16


def lib():
    from pytorch_distributed_b200 import _ext
    return _ext.lib()


# ================================================================================================ conv1x1_bnstats, fp16
def changed_limit(K: int) -> float:
    """Largest fraction of fp16 GEMM outputs allowed to differ from fp16(fp64) at all.  Only an element whose exact value
    lies within the fp32 accumulation error of a rounding boundary can differ, so the fraction is proportional to that
    error (which grows with K) over the spacing of the boundaries.  _fp64.check_conv1x1 allows bf16 1e-3 up to K = 1024
    (1.2e-3 was measured at K = 2048 on an H100); fp16 boundaries are 2^(10 - 7) = 8 times denser at the same magnitude."""
    return 8e-3 * max(1.0, K / 1024)


def check_conv1x1_fp16(y, x, w, max_changed=None) -> float:
    """_fp64.check_conv1x1 for fp16 operands: products of two fp16 values (11 + 11 significant bits) are exact in fp32,
    so the bound is the same - half an fp16 ulp of the stored value (2^-24 subnormal spacing near 0) plus
    K u sum_k |a_k b_k| for the accumulation.  Returns the fraction of elements that differ from fp16(fp64)."""
    assert y.dtype == F16
    K, N = x.size(1), w.size(0)
    if max_changed is None:
        max_changed = changed_limit(K)
    a = R.rows(x).double()
    b = w.reshape(N, K).double()
    ref = a @ b.t()
    mag = a.abs() @ b.abs().t()
    del a, b
    got = R.rows(y)
    R.assert_within("conv1x1 y", got, ref, 0.5 * R.ulp(got, F16) + K * R.U32 * mag)
    changed = (got != ref.to(F16)).double().mean().item()
    assert changed <= max_changed, "conv1x1 y: %.3g of the elements differ from fp16(fp64) (limit %.3g)" % (changed, max_changed)
    return changed


def _inputs16(B, K, N, H, W, seed=0):
    g = _gen(seed)
    x = torch.randn(B, K, H, W, device=DEV, generator=g).half().contiguous(memory_format=CL)
    w = (torch.randn(N, K, 1, 1, device=DEV, generator=g) * K ** -0.5).half()
    base = torch.randn(2 * N, device=DEV, generator=g) * 64      # gsum accumulates: start from nonzero sums
    base[N:] = base[N:].abs()
    return x, w, base


def _run(x, w, base):
    gs = base.clone()
    y = lib().conv1x1_bnstats(x, w, gs)
    return y, gs


def _check(x, w, base, y, gs, geo):
    assert y.dtype == F16 and y.is_contiguous(memory_format=CL)
    changed = check_conv1x1_fp16(y, x, w)
    R.check_sums("gemm_bnstats fp16", gs, R.rows(y), geo["depth"], base)
    return changed


@pytest.mark.parametrize("k,n,hw", RESNET50_1X1, ids=["%d-%d@%d" % s for s in RESNET50_1X1])
def test_fp16_conv1x1_bnstats_resnet50_batch256(k, n, hw):
    x, w, base = _inputs16(256, k, n, hw, hw)
    geo = R.gemm_geometry(256 * hw * hw, n, k, sms())
    assert geo["max_tiles_per_cta"] > 1
    y, gs = _run(x, w, base)
    changed = _check(x, w, base, y, gs, geo)
    print("K=%d N=%d: %.3g of the elements differ from fp16(fp64), limit %.3g" % (k, n, changed, changed_limit(k)))
    assert _equal_all((y, gs), _run(x, w, base))


@pytest.mark.parametrize("name,k,n,m_of", GEMM_EDGES, ids=[e[0] for e in GEMM_EDGES])
def test_fp16_conv1x1_bnstats_geometry_edges(name, k, n, m_of):
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
    x, w, base = _inputs16(M, k, n, 1, 1, seed=M)
    y, gs = _run(x, w, base)
    _check(x, w, base, y, gs, geo)


def test_fp16_conv1x1_checker_rejects_edited_result():
    x, w, base = _inputs16(8, 256, 512, 28, 28)
    y, gs = _run(x, w, base)
    _check(x, w, base, y, gs, R.gemm_geometry(8 * 28 * 28, 512, 256, sms()))
    bad = y.clone()
    v = bad[3, 100, 5, 7].double()
    bad[3, 100, 5, 7] = (v + 2 * R.ulp(v, F16)).half()                    # one element moved by 2 fp16 ulp
    with pytest.raises(AssertionError, match="conv1x1 y"):
        check_conv1x1_fp16(bad, x, w)


def test_conv1x1_bnstats_rejects_mixed_dtypes():
    x, w, base = _inputs16(2, 64, 64, 8, 8)
    with pytest.raises(RuntimeError, match="both bf16 or both fp16"):
        lib().conv1x1_bnstats(x, w.bfloat16(), base.clone())
    with pytest.raises(RuntimeError, match="bf16 or fp16"):
        lib().conv1x1_bnstats(x.float(), w.float(), base.clone())


def test_fp16_conv1x1_bnstats_overflow():
    """Columns scaled past fp16's range: y is fp16-RNE of the exact product (+-inf at |y| >= 65520) wherever the fp32
    accumulation error cannot change the rounding; the sums of every channel holding an inf are non-finite, the others
    stay finite and within their bound."""
    B, K, N, hw = 64, 64, 128, 14
    x, w, base = _inputs16(B, K, N, hw, hw, seed=50)
    big = torch.arange(N, device=DEV) % 8 == 0                           # 16 channels with |y| ~ N(0, 40000^2)
    w[big] = (w[big].float() * 40000).half()
    y, gs = _run(x, w, base)
    a = R.rows(x).double()
    b = w.reshape(N, K).double()
    ref = a @ b.t()
    err = K * R.U32 * (a.abs() @ b.abs().t())
    del a, b
    got = R.rows(y)
    # monotone rounding: the kernel's fp32 value v lies in [ref - err, ref + err], so fp16(v) is known where both ends agree
    lo, hi = (ref - err).half(), (ref + err).half()
    known = lo == hi                       # (the bound is a worst case: near 0 it exceeds the fp16 spacing)
    assert known.double().mean().item() > 0.5
    wrong = known & (got != lo)
    assert not wrong.any(), "%d determined elements differ from fp16(fp64), e.g. got %r for fp64 %r" % (
        int(wrong.sum()), got[wrong][0].item(), ref[wrong][0].item())
    inf_cols = torch.isinf(got).any(0)
    assert torch.equal(inf_cols, big), "inf outside the scaled channels, or a scaled channel without one"
    assert (got[:, big].abs() >= 65504).any() and torch.isfinite(got[:, big]).any()   # both sides of the limit are reached
    near = known & (ref.abs() >= 65504) & (ref.abs() < 65520)
    assert torch.equal(got[near].abs(), torch.full_like(got[near], 65504))    # rounds down to the largest finite fp16
    assert not torch.isfinite(gs[:N][big]).any() and not torch.isfinite(gs[N:][big]).any()
    fin = ~big
    ok = torch.cat([fin, fin])
    assert torch.isfinite(gs[ok]).all()
    sub = torch.cat([gs[:N][fin], gs[N:][fin]])
    R.check_sums("gemm_bnstats fp16 finite channels", sub, got[:, fin], R.gemm_geometry(B * hw * hw, N, K, sms())["depth"],
                 torch.cat([base[:N][fin], base[N:][fin]]))


# ================================================================================================ stem, fp16
@pytest.mark.parametrize("shape,aligned", [((16, 3, 224, 224), True), ((2, 3, 75, 91), True), ((3, 3, 64, 64), False)],
                         ids=["staged_224", "scalar_odd_rows", "scalar_unaligned"])
def test_fp16_stem_im2col_matches_definition(shape, aligned):
    from pytorch_distributed_b200.ops.stem_conv import im2col_reference
    n, c, h, w = shape
    src = torch.randn(n * h * w * c + 1, device=DEV, generator=_gen(60)).half()
    off = 0 if aligned else 1                                             # 2 bytes past a 16-byte boundary
    x = src[off: off + n * h * w * c].view(n, h, w, c).permute(0, 3, 1, 2)
    assert x.is_contiguous(memory_format=CL) and (x.data_ptr() % 16 == 0) == aligned
    a = lib().stem_im2col(x)
    ref = im2col_reference(x)
    assert a.dtype == F16 and a.shape == ref.shape and a.is_contiguous(memory_format=CL)
    assert torch.equal(a, ref)


def test_fp16_stem_gemm_feeding_stem_forward_pre():
    """The fp16 stem GEMM (im2col + conv1x1_bnstats) against fp64, and stem_forward_pre normalising with its sums."""
    from pytorch_distributed_b200.ops.stem_conv import K_PAD, pack_stem_weight
    img = torch.randn(32, 3, 224, 224, device=DEV, generator=_gen(30)).half().contiguous(memory_format=CL)
    wconv = (torch.randn(64, 3, 7, 7, device=DEV, generator=_gen(31)) * 0.1).half()
    a = lib().stem_im2col(img)
    gs = torch.zeros(2 * 64, device=DEV)
    wp = pack_stem_weight(wconv).view(64, K_PAD, 1, 1)
    yc = lib().conv1x1_bnstats(a, wp, gs)
    geo = R.gemm_geometry(yc.numel() // 64, 64, K_PAD, sms())
    check_conv1x1_fp16(yc, a, wp)
    R.check_sums("stem gemm fp16", gs, R.rows(yc), geo["depth"])
    w, b, rm0, rv0 = _bn_params(64, torch.float32, 32)
    y, saved, code, rm, rv, nbt = _stem_forward(yc, w, b, rm0, rv0, work=gs, pre=True)
    assert y.dtype == F16
    st = R.check_stats("stem_pre fp16", saved, R.rows(yc), geo["depth"], EPS)
    R.check_running("stem_pre fp16", rm, rv, rm0, rv0, st, 0.1)
    assert nbt.item() == 1
    yref, _, e_sel, _ = R.stem_forward_ref(yc, saved[:64], saved[64:], w, b)
    R.assert_within("stem_pre fp16 y", y, yref, 0.5 * R.ulp(y, y.dtype) + e_sel)
    assert torch.equal(R.code_nchw(code, *y.shape) == 15, y == 0)


# ================================================================================================ model routing
class _Counter:
    """Counts calls of the extension's conv1x1_bnstats and stem_im2col (the entry points are wrapped on the module)."""

    def __init__(self, monkeypatch):
        self.n = {"conv1x1_bnstats": 0, "stem_im2col": 0}
        mod = lib()
        for name in self.n:
            fn = getattr(mod, name)

            def wrapped(*a, _fn=fn, _name=name):
                self.n[_name] += 1
                return _fn(*a)
            monkeypatch.setattr(mod, name, wrapped)

    def take(self):
        out = (self.n["conv1x1_bnstats"], self.n["stem_im2col"])
        for k in self.n:
            self.n[k] = 0
        return out


FUSED = (34, 1)      # 33 stride-1 1x1 convolutions of ResNet-50 + the stem GEMM; one im2col


def _resnet50(mode):
    """(model, input, autocast dtype or None) for one precision mode; the model's forward applies the amp wrappers."""
    from pytorch_distributed_b200.apex import amp
    from pytorch_distributed_b200.models import create_model
    from pytorch_distributed_b200.parallel.amp import cast_model
    torch.manual_seed(0)
    m = create_model("resnet50", num_classes=100).to(DEV).to(memory_format=CL).train()
    x = torch.randn(16, 3, 96, 96, device=DEV, generator=_gen(70)).contiguous(memory_format=CL)
    ac = None
    if mode == "bf16_cast":
        cast_model(m, torch.bfloat16)
        x = x.bfloat16()
    elif mode in ("fp16_O2", "fp16_O3", "fp16_O1"):
        m = amp.initialize(m, opt_level=mode[-2:], half_dtype=F16, verbosity=0)   # O2 / O3 cast the model and the input
    elif mode == "bf16_autocast":
        ac = torch.bfloat16
    return m, x, ac


def _forward(m, x, ac):
    if ac is None:
        return m(x)
    with torch.autocast("cuda", dtype=ac):
        return m(x)


MODES = ["bf16_cast", "fp16_O2", "fp16_O3", "fp16_O1", "bf16_autocast"]


@pytest.mark.parametrize("mode", MODES)
def test_resnet50_training_forward_routes_to_gemm(mode, monkeypatch):
    from _oracle import model_flags
    from pytorch_distributed_b200.ops.bn_act import begin_step
    m, x, ac = _resnet50(mode)
    cnt = _Counter(monkeypatch)
    with model_flags(FUSED_CONV1X1=True, STEM_GEMM=True, SPLIT_RESGRAD=True):
        begin_step(torch.device(DEV))
        out = _forward(m, x, ac)
        assert cnt.take() == FUSED
        out.float().sum().backward()
        if mode in ("fp16_O1", "bf16_autocast"):                         # fp32 parameters receive fp32 gradients
            bad = [n for n, p in m.named_parameters() if p.grad is None or p.grad.dtype != torch.float32]
            assert bad == [], bad[:5]
            assert all(torch.isfinite(p.grad).all() for p in m.parameters())
        with torch.no_grad():
            m.eval()
            _forward(m, x, ac)
        assert cnt.take() == (0, 0)
        m.train()
    with model_flags(FUSED_CONV1X1=False, STEM_GEMM=False):
        begin_step(torch.device(DEV))
        _forward(m, x, ac)
    assert cnt.take() == (0, 0)


# ================================================================================================ whole-model numerics
def _small(mode):
    """Shallow bottleneck ResNet + batch for one precision mode (as tests/_oracle.py expects: the oracle sees the same weights)."""
    from _oracle import small_resnet
    from pytorch_distributed_b200.parallel.amp import cast_model
    base = small_resnet(64).to(DEV).to(memory_format=CL)
    torch.manual_seed(1)
    x = torch.randn(32, 3, 96, 96, device=DEV).contiguous(memory_format=CL)
    y = torch.randint(0, 64, (32,), device=DEV)
    if mode == "fp16_cast":
        cast_model(base, F16)
        for p in base.parameters():
            if hasattr(p, "_ptd_master_init"):
                del p._ptd_master_init
        x = x.half()
    return base, x, y, {"fp16_cast": None, "fp16_autocast": F16, "bf16_autocast": torch.bfloat16}[mode]


@pytest.mark.parametrize("mode", ["fp16_cast", "fp16_autocast", "bf16_autocast"])
def test_fused_path_vs_fp32_oracle(mode, monkeypatch):
    from _oracle import compare, fp32_oracle, model_flags, step
    from pytorch_distributed_b200.ops.bn_act import begin_step
    base, x, y, ac = _small(mode)
    oracle = fp32_oracle(base, x, y)
    cnt = _Counter(monkeypatch)

    def run(fused):
        m = copy.deepcopy(base).train()
        with model_flags(FUSED_CONV1X1=fused, STEM_GEMM=fused, SPLIT_RESGRAD=True):
            begin_step(torch.device(DEV))
            if ac is None:
                return step(m, x, y)
            with torch.autocast("cuda", dtype=ac):
                return step(m, x, y)
    default = run(False)
    assert cnt.take() == (0, 0)
    variant = run(True)
    assert cnt.take() == (4 * 2 + 1 + 1, 1)               # conv1 + conv3 of 4 blocks, layer1's projection, the stem
    torch.cuda.synchronize()
    assert all(torch.isfinite(g).all() for g in variant[1].values())
    bad = compare(variant, default, oracle)
    assert not bad, "error vs the fp32 oracle (name, variant, default path): %s" % (bad[:8],)


# ================================================================================================ reproducibility
def test_resnet50_fp16_full_depth_step_is_bitwise_reproducible():
    """Two identical full-depth fp16 ResNet-50 train steps (model cast as amp O2 does, deterministic cuDNN) through the
    fp16 GEMM and stem paths give the same outputs, gradients and BN buffers."""
    from _oracle import model_flags
    from pytorch_distributed_b200.models import create_model
    from pytorch_distributed_b200.ops.bn_act import begin_step
    from pytorch_distributed_b200.parallel.amp import cast_model
    torch.manual_seed(0)
    m0 = cast_model(create_model("resnet50", num_classes=100).to(DEV).to(memory_format=CL), F16, keep_batchnorm_fp32=True).train()
    x = torch.randn(16, 3, 96, 96, device=DEV).half().contiguous(memory_format=CL)
    y = torch.randint(0, 100, (16,), device=DEV)
    flags = (torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark)
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    runs = []
    try:
        with model_flags(FUSED_CONV1X1=True, STEM_GEMM=True, SPLIT_RESGRAD=True):
            for _ in range(2):
                m = copy.deepcopy(m0)
                begin_step(torch.device(DEV))
                out = m(x)
                torch.nn.functional.cross_entropy(out.float(), y).backward()
                runs.append((out.detach(), {n: p.grad for n, p in m.named_parameters()}, dict(m.named_buffers())))
    finally:
        torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = flags
    torch.cuda.synchronize()
    (o1, g1, b1), (o2, g2, b2) = runs
    assert o1.dtype == F16 and torch.isfinite(o1).all()
    assert all(g is not None and torch.isfinite(g).all() for g in g1.values())
    assert torch.equal(o1, o2)
    assert [n for n in g1 if not torch.equal(g1[n], g2[n])] == []
    assert [n for n in b1 if not torch.equal(b1[n], b2[n])] == []


# ================================================================================================ apex strategy, world 1
@pytest.mark.parametrize("opt_level", ["O1", "O2", "O3"])
def test_apex_strategy_fp16_steps(opt_level, monkeypatch):
    """The apex_distributed strategy built as bench.py builds it (fp16, one process, CUDA graph where the strategy allows
    it): finite losses, and every step that runs the Python forward issues the fused GEMM and im2col calls."""
    from _oracle import model_flags
    from pytorch_distributed_b200 import cli, driver
    from pytorch_distributed_b200.models import create_model
    from pytorch_distributed_b200.utils.data import SyntheticLoader
    from pytorch_distributed_b200.utils.meters import AverageMeter
    dev = torch.device(DEV, 0)
    torch.cuda.set_device(0)
    args = cli.parse_args("apex_distributed", ["-a", "resnet50", "-b", "16", "--synthetic", "--precision", "fp16", "--image-size", "96",
                                               "--opt-level", opt_level, "--quiet"])
    st = driver.STRATEGIES["apex_distributed"]()
    torch.manual_seed(0)
    with model_flags(FUSED_CONV1X1=True, STEM_GEMM=True, SPLIT_RESGRAD=True):
        model = create_model(args.arch, num_classes=args.num_classes, fused_bn=args.fused_bn)
        model, optimizer = st.build(model, args, dev, 0)
        criterion = torch.nn.CrossEntropyLoss().to(dev)
        losses = AverageMeter("Loss")
        metrics = driver.MetricPipeline(getattr(st, "comm", None), dev, (losses, AverageMeter("Acc@1"), AverageMeter("Acc@5")), reduce=True)
        use_graph = (st.graph_capable and getattr(getattr(st, "comm", None), "backend", "") == "fused"
                     and hasattr(optimizer, "refresh_hyper"))
        step = driver.TrainStep(st, model, criterion, optimizer, metrics, use_graph=use_graph, warmup=2)
        model.train()
        pf = st.prefetcher(SyntheticLoader(16, 2, 96, args.num_classes, pool=2), dev, args)
        batches = [(i.clone(), t.clone()) for i, t in pf]
        cnt = _Counter(monkeypatch)
        counts, vals = [], []
        for i in range(5):
            step(*batches[i % len(batches)])
            metrics.drain()
            counts.append(cnt.take())
            vals.append(losses.val)
    torch.cuda.synchronize()
    assert all(v == v and abs(v) < 1e4 for v in vals), vals
    python_steps = 5 if step.graph is None else 3          # with a graph: 2 eager steps + the capture, then replays
    assert counts[:python_steps] == [FUSED] * python_steps, counts
    assert counts[python_steps:] == [(0, 0)] * (5 - python_steps), counts
    print("%s: graph %s, losses %s" % (opt_level, step.graph is not None, vals))
