"""LARC in the fused SGD kernels (``larc_sgd_flat`` / ``larc_sgd_multi`` in csrc/optim.cu) on one GPU: the norm and update
passes against float64 at ResNet-50 parameter shapes with bounds derived from the reduction depth, the overflow skip,
bit-identity between the flat, per-bucket, multi-tensor, eager and CUDA-graph paths, and the training entrypoints."""
import math
import os
import subprocess
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _fp64 as R  # noqa: E402

pytestmark = pytest.mark.gpu

DEV = "cuda"
F32, BF16, F16 = torch.float32, torch.bfloat16, torch.float16
CL = torch.channels_last
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = R.U32
TRUST, EPS = 0.02, 1e-8


def C():
    from pytorch_distributed_b200 import _ext
    return _ext.lib()


def hyper_t(lr=0.1, mom=0.9, wd=1e-4, damp=0.0, gmul=1.0, pending=0.0):
    return torch.tensor([lr, mom, wd, damp, gmul, pending, 0, 0], dtype=F32, device=DEV)


# ------------------------------------------------------------------------------------------------ fp64 reference + bounds
def larc_depth(numel: int, chunk: int) -> int:
    """Longest chain of fp32 additions behind one tensor's sum of squares: 8-element groups added in sequence by one
    thread (chunk / 256 terms), the 8-level tree over the CTA's 256 threads, then the chunk partials in sequence."""
    return chunk // 256 + 8 + R.cdiv(numel, chunk)


def larc_fp64(p, g, m, hv, nesterov, first, clip, chunk):
    """One LARC + SGD step of one tensor in float64 from the fp32 state the kernel read, with bounds on |kernel - fp64|.

    Sums of squares: |S - S^| <= d u S (d = larc_depth, all terms >= 0), the gradient's terms carry the 2u of the rounded
    g * gmul as well.  sqrt adds u and halves the relative error; f = trust pn / (fma(pn, wd, gn) + eps) adds the errors of
    its numerator and denominator and one rounding for the division, clip one more for / lr.  The scaled gradient
    a = fma(wd, p, g gmul) * f carries |g gmul + wd p| e_f + rounding, and sgd_step_fp64's bound is widened by the
    propagation of that error through the momentum (coefficient 1 or |1 - d|, nesterov 1 + mom of it) and lr."""
    lr, mom, wd, d, gmul = (float(x) for x in hv[:5])
    p, g, m = p.double(), g.double() * gmul, m.double()
    dep = larc_depth(p.numel(), chunk)
    sp, sg = float((p * p).sum()), float((g * g).sum())
    pn, gn = math.sqrt(sp), math.sqrt(sg)
    rel_pn = dep * U / 2 + U
    rel_gn = (dep + 2) * U / 2 + U
    f, e_f = 1.0, 0.0
    adapt = pn != 0 and gn != 0
    if adapt:
        den = gn + pn * wd + EPS
        f = TRUST * pn / den
        rel_den = (wd * pn * rel_pn + gn * rel_gn + U * (gn + pn * wd) + U * den) / den
        rel_f = rel_pn + U + rel_den + U
        if clip:
            f = min(f / lr, 1.0)
            rel_f += U
        e_f = 1.01 * f * rel_f
        a = (g + wd * p) * f
        e_a = (g + wd * p).abs() * e_f + f * U * (g.abs() + (g + wd * p).abs()) + U * a.abs()
    else:
        a, e_a = g, U * g.abs()
    ref = R.sgd_step_fp64(p, m, a, [lr, mom, 0.0, d, 1.0], nesterov, first)
    c_m = 1.0 if (first or mom == 0.0) else abs(1.0 - d)
    c_b = (1.0 + mom * c_m) if (nesterov and mom != 0.0) else c_m
    ref["m_bound"] = ref["m_bound"] + (c_m * e_a if mom != 0.0 else 0.0)
    ref["p_bound"] = ref["p_bound"] + 1.01 * lr * c_b * e_a
    ref["stats"] = (pn, gn, f)
    ref["stats_bound"] = (1.01 * rel_pn * pn + 1e-30, 1.01 * rel_gn * gn + 1e-30, e_f if adapt else 0.0)
    return ref


def check_step(name, tensors, stats, refs):
    """tensors: list of (master, momentum) views per parameter."""
    worst = 0.0
    for i, ((pm, mm), ref) in enumerate(zip(tensors, refs)):
        worst = max(worst, R.check_sgd("%s param %d" % (name, i), pm, mm, ref))
        for k, what in enumerate(("pn", "gn", "f")):
            R.assert_within("%s param %d %s" % (name, i, what), stats[i, k:k + 1], torch.tensor([ref["stats"][k]], dtype=torch.float64,
                            device=stats.device), ref["stats_bound"][k])
    return worst


# ------------------------------------------------------------------------------------------------ ResNet-50 flat problem
def r50_params():
    from pytorch_distributed_b200.models import create_model
    torch.manual_seed(0)
    ps = [p.detach().to(DEV) for p in create_model("resnet50").parameters()]
    assert len(ps) == 161 and sum(p.numel() for p in ps) == 25_557_032
    return ps


class Flat:
    """ResNet-50 parameters laid out as the gradient engine lays out its arena (64-element aligned offsets) and the chunk
    table FusedSGD builds from that layout."""

    def __init__(self, gdt, cdt, gmul=1.0, seed=0):
        from pytorch_distributed_b200.parallel import plan as P
        ps = r50_params()
        self.numels = [p.numel() for p in ps]
        self.offs, self.n = P.tensor_layout(self.numels)
        chunk = C().LARC_CHUNK
        self.chunk = chunk
        gen = torch.Generator(device=DEV).manual_seed(seed)
        self.master = torch.zeros(self.n, device=DEV)
        self.grad = torch.zeros(self.n, dtype=gdt, device=DEV)
        self.mom = torch.zeros(self.n, device=DEV)
        info, ct = [], []
        for i, (p, o) in enumerate(zip(ps, self.offs)):
            k = p.numel()
            self.master[o:o + k] = p.flatten()
            scale = 10.0 ** (-(i % 4)) * 0.05                 # f / lr on both sides of 1 across the tensors
            g = torch.randn(k, device=DEV, generator=gen) * scale
            if i == len(ps) - 1:
                g.zero_()                                     # the zero-gradient branch
            self.grad[o:o + k] = (g / gmul).to(gdt)
            info.append((o, k, len(ct), i))
            ct += [i] * R.cdiv(k, chunk)
        self.zero_p = [i for i, p in enumerate(ps) if not bool(p.any())]
        assert self.zero_p, "ResNet-50 starts with BatchNorm betas at zero"
        self.chunks = len(ct)
        self.ct = torch.tensor(ct, dtype=torch.int32, device=DEV)
        self.info = torch.tensor(info, dtype=torch.int64, device=DEV)
        self.partials = torch.zeros(2 * self.chunks, device=DEV)
        self.stats = torch.zeros(len(ps), 3, device=DEV)
        self.copy = torch.zeros(self.n, dtype=cdt, device=DEV) if cdt is not None else None

    def step(self, hyper, first, clip, nesterov=False, found_inf=None, lo=0, hi=None):
        C().larc_sgd_flat(self.grad, self.master, self.mom, self.copy, hyper, found_inf, nesterov, first, self.ct, self.info, lo,
                          self.chunks if hi is None else hi, self.partials, self.stats, TRUST, EPS, clip)

    def views(self, t):
        return [t[o:o + k] for o, k in zip(self.offs, self.numels)]

    def refs(self, p0, m0, hyper, first, clip, nesterov=False):
        hv = hyper[:5].tolist()
        return [larc_fp64(p, g, m, hv, nesterov, first, clip, self.chunk)
                for p, g, m in zip(self.views(p0), self.views(self.grad), self.views(m0))]


PAIRS = [(g, c) for g in (F32, BF16, F16) for c in (None, BF16, F16)]


@pytest.mark.parametrize("clip", [True, False], ids=["clip", "scale"])
@pytest.mark.parametrize("gdt,cdt", PAIRS, ids=lambda d: str(d).replace("torch.", ""))
def test_flat_against_fp64_resnet50(gdt, cdt, clip):
    gmul = 2.0 ** -16 if gdt == F16 else 1.0
    fl = Flat(gdt, cdt, gmul)
    hyper = hyper_t(gmul=gmul)
    for step in range(2):
        p0, m0 = fl.master.clone(), fl.mom.clone()
        fl.step(hyper, step == 0, clip)
        refs = fl.refs(p0, m0, hyper, step == 0, clip)
        check_step("flat %s step %d" % (clip, step), list(zip(fl.views(fl.master), fl.views(fl.mom))), fl.stats, refs)
        if cdt is not None:
            R.assert_bits_equal("copy", fl.copy, fl.master.to(cdt))
        if step == 0:                          # zero-norm branches: BatchNorm betas (pn = 0) and the zero gradient (gn = 0)
            assert all(float(fl.stats[i, 0]) == 0.0 and float(fl.stats[i, 2]) == 1.0 for i in fl.zero_p)
            assert float(fl.stats[-1, 1]) == 0.0 and float(fl.stats[-1, 2]) == 1.0
    if clip:
        f = fl.stats[:, 2]
        assert bool((f == 1.0).any()) and bool(((f > 0) & (f < 1)).any())     # both sides of the clip were exercised


def test_negative_control_is_rejected():
    fl = Flat(BF16, BF16)
    hyper = hyper_t()
    p0, m0 = fl.master.clone(), fl.mom.clone()
    fl.step(hyper, True, True)
    refs = fl.refs(p0, m0, hyper, True, True)
    bad_stats = fl.stats.clone()
    i = max(range(len(refs)), key=lambda k: refs[k]["stats"][2] if refs[k]["stats"][2] < 1 else 0)
    bad_stats[i, 2] *= 1.001                         # f off by far more than its bound
    with pytest.raises(AssertionError):
        check_step("negative control f", list(zip(fl.views(fl.master), fl.views(fl.mom))), bad_stats, refs)
    bad = fl.master.clone()
    o, k = fl.offs[i], fl.numels[i]
    bad[o:o + k] = p0[o:o + k] - (p0[o:o + k] - fl.master[o:o + k]) * 1.001   # the update with f 0.1 % too large
    with pytest.raises(AssertionError):
        check_step("negative control master", list(zip(fl.views(bad), fl.views(fl.mom))), fl.stats, refs)


@pytest.mark.parametrize("cdt", [F16, BF16])
def test_found_inf_leaves_everything_bitwise(cdt):
    fl = Flat(F16, cdt, 2.0 ** -16)
    fl.copy.copy_(fl.master.to(cdt))
    fl.stats.fill_(7.0)
    before = [t.clone() for t in (fl.master, fl.mom, fl.copy, fl.stats)]
    fi = torch.ones(1, dtype=torch.int32, device=DEV)
    fl.step(hyper_t(gmul=2.0 ** -16, pending=1.0), True, True, found_inf=fi)
    torch.cuda.synchronize()
    for a, b in zip((fl.master, fl.mom, fl.copy, fl.stats), before):
        assert torch.equal(a, b)
    # the same call with the flag clear applies the step (and momentum_pending makes it a first step)
    fi.zero_()
    fl.step(hyper_t(gmul=2.0 ** -16, pending=1.0), False, True, found_inf=fi)
    assert not torch.equal(fl.master, before[0]) and not torch.equal(fl.stats, before[3])


def test_flat_multi_bucket_and_repeat_are_bit_identical():
    """Same inputs: one flat call, per-bucket chunk ranges, the multi-tensor front end, and a second run."""
    runs = []
    for kind in ("flat", "buckets", "multi", "flat"):
        fl = Flat(BF16, BF16, seed=3)
        hyper = hyper_t(mom=0.9, wd=5e-4)
        for step in range(2):
            if kind == "flat":
                fl.step(hyper, step == 0, True)
            elif kind == "buckets":
                # whole tensors per bucket, as plan.compute_buckets makes them, in reverse order like backward
                firsts = fl.info[:, 2].tolist() + [fl.chunks]
                cuts = list(range(0, len(fl.numels), 23)) + [len(fl.numels)]
                for a, b in reversed(list(zip(cuts[:-1], cuts[1:]))):
                    fl.step(hyper, step == 0, True, lo=firsts[a], hi=firsts[b])
            else:
                n = len(fl.numels)
                copies = [c for c in fl.views(fl.copy)]
                C().larc_sgd_multi(fl.views(fl.grad), fl.views(fl.master), fl.views(fl.mom), copies, hyper, None, False,
                                   [step == 0] * n, list(range(n)), fl.stats, TRUST, EPS, True)
        torch.cuda.synchronize()
        runs.append((kind, fl.master, fl.mom, fl.copy, fl.stats))
    ref = runs[0]
    for kind, *ts in runs[1:]:
        for name, a, b in zip(("master", "momentum", "copy", "stats"), ref[1:], ts):
            R.assert_bits_equal("%s vs flat %s" % (kind, name), a, b)


# ------------------------------------------------------------------------------------------------ through the engine
@pytest.fixture
def deterministic():
    flags = (torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark)
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    yield
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = flags


def _build(argv, entry="distributed"):
    from pytorch_distributed_b200 import cli, driver
    from pytorch_distributed_b200.models import create_model
    torch.cuda.set_device(0)
    args = cli.parse_args(entry, ["-a", "resnet50", "-b", "8", "--synthetic", "--image-size", "64", "--quiet", "--larc"] + argv)
    st = driver.STRATEGIES[entry]()
    torch.manual_seed(0)
    model = create_model(args.arch, num_classes=args.num_classes, fused_bn=args.fused_bn)
    model, opt = st.build(model, args, torch.device(DEV, 0), 0)
    model.train()
    return st, model, opt


def _batch(dtype, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(8, 3, 64, 64, device=DEV, generator=g).to(dtype).contiguous(memory_format=CL)
    y = torch.randint(0, 1000, (8,), device=DEV, generator=g)
    return x, y


def _train(argv, steps=3, graph=False, lr_at=None):
    from pytorch_distributed_b200 import driver
    st, model, opt = _build(argv)
    metrics = driver.MetricPipeline(st.comm, torch.device(DEV, 0), (driver.AverageMeter("l"), driver.AverageMeter("a"),
                                                                     driver.AverageMeter("b")))
    step = driver.TrainStep(st, model, torch.nn.CrossEntropyLoss().to(DEV), opt, metrics, use_graph=graph, warmup=1)
    fs = []
    for i in range(steps):
        if lr_at is not None and i == lr_at[0]:
            for g in opt.param_groups:
                g["lr"] = lr_at[1]
        x, y = _batch(st.input_dtype, seed=i)
        step(x, y)
        torch.cuda.synchronize()
        fs.append(opt.larc_stats()[:, 2].clone())
    metrics.drain()
    assert opt.is_flat and (graph is False or step.graph is not None)
    return opt._flat.master.clone(), opt._flat.momentum.clone(), opt.larc_stats().clone(), fs


def test_engine_overlap_eager_graph_bit_identical(deterministic):
    base = _train(["--no-overlap-optimizer"])
    for argv, graph in (([], False), ([], True), (["--no-overlap-optimizer"], True), (["--no-overlap-optimizer"], False)):
        got = _train(argv, graph=graph)
        for name, a, b in zip(("master", "momentum", "stats"), base[:3], got[:3]):
            R.assert_bits_equal("%s graph=%s %s" % (argv, graph, name), a, b)


def test_graph_replay_follows_lr_in_clip_mode(deterministic):
    """adjust_learning_rate between replays: refresh_hyper pushes lr, and the clipped factor min(f / lr, 1) changes."""
    _, _, _, fs = _train([], steps=4, graph=True, lr_at=(3, 0.01))
    f2, f3 = fs[2], fs[3]
    adapt = (f2 > 0) & (f2 < 1)
    assert bool(adapt.any())
    # f / lr grows 10x when lr drops 10x (the norms move little in one step): unclipped factors rise, some reach 1
    assert bool((f3[adapt] > 5 * f2[adapt]).any() | (f3[adapt] == 1.0).any())
    assert not torch.equal(f2, f3)


def _entry(script, args, tmp, n=1, port=29761, env=None):
    e = dict(os.environ, PYTHONPATH=ROOT, **(env or {}))
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "MASTER_ADDR", "MASTER_PORT"):
        e.pop(k, None)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(n), "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, script)] + args
    p = subprocess.run(cmd, env=e, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-3000:] + "\n" + p.stderr[-3000:]
    return p.stdout


COMMON = ["-a", "resnet50", "-b", "32", "--synthetic", "--steps-per-epoch", "4", "--val-steps", "1", "--epochs", "1",
          "--image-size", "96", "-p", "1", "--larc"]


def _finite_losses(out):
    import re
    losses = [float(x) for x in re.findall(r"Loss ([0-9.e+-]+|nan|inf) \(", out)]
    assert losses and all(math.isfinite(x) for x in losses), out[-2000:]


def test_distributed_py_larc_cuda_graph(tmp_path):
    _finite_losses(_entry("distributed.py", COMMON + ["--cuda-graph", "--checkpoint-dir", str(tmp_path)], tmp_path, port=29762))


def test_apex_o2_larc(tmp_path):
    _finite_losses(_entry("apex_distributed.py", COMMON + ["--opt-level", "O2", "--checkpoint-dir", str(tmp_path)], tmp_path,
                          port=29763))


def test_resume_keeps_momentum(tmp_path):
    out = str(tmp_path / "a")
    _entry("tests/mp_larc_checks.py", [out, "distributed"] + COMMON + ["--checkpoint-dir", str(tmp_path)], tmp_path, port=29764,
           env={"PTD_SAVE_OPTIMIZER": "1"})
    saved = torch.load(os.path.join(out, "rank0.pt"), weights_only=False)
    ck = torch.load(tmp_path / "checkpoint.pth.tar", weights_only=False)
    assert ck["optimizer"] is not None
    # resume for zero further steps (--epochs 1 with start epoch 1): the optimizer then holds exactly what was restored
    out2 = str(tmp_path / "b")
    os.makedirs(tmp_path / "r")
    _entry("tests/mp_larc_checks.py", [out2, "distributed"] + COMMON + ["--checkpoint-dir", str(tmp_path / "r"), "--resume",
                                                                        str(tmp_path / "checkpoint.pth.tar")], tmp_path, port=29765)
    resumed = torch.load(os.path.join(out2, "rank0.pt"), weights_only=False)
    assert len(resumed["momenta"]) == len(saved["momenta"]) == 161
    for a, b in zip(saved["momenta"], resumed["momenta"]):
        assert torch.equal(a, b)
    assert any(bool(a.any()) for a in saved["momenta"])
