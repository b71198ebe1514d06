"""fp32 gradient accumulation on one GPU: ``grad_accumulate`` / ``grad_fold`` (csrc/collectives.cu) bit for bit against torch
over the ResNet-50 bucket plan, the engine's K-pass steps against the single-pass path fed the oracle sum, CUDA-graph replay
of both kinds of pass, apex O2's overflow skip, and the entrypoints."""
import math
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CL = torch.channels_last
SENTINEL = -1234.5


def C():
    from pytorch_distributed_b200 import _ext
    return _ext.lib()


@pytest.fixture
def deterministic():
    flags = torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    yield
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = flags


# ------------------------------------------------------------------------------------------------ kernels
def _resnet50_buckets(esz=2):
    """The engine's bucket plan of ResNet-50 at world 1: (numels of each bucket, its layout), reverse registration order."""
    from pytorch_distributed_b200.models import create_model
    from pytorch_distributed_b200.parallel import plan as P
    shapes = [tuple(p.shape) for p in create_model("resnet50", num_classes=1000).parameters()]
    assert len(shapes) == 161
    order = list(range(len(shapes)))[::-1]
    numels = [math.prod(shapes[i]) for i in order]
    groups = P.compute_buckets(numels, esz, 8 << 20, 1 << 20, 256, 1 << 20)
    out = []
    for g in groups:
        ns = [numels[j] for j in g]
        offs, total = P.tensor_layout(ns)
        lay = P.build_layout(ns, 1, P.choose_grid(total, esz, 32), offs, total)
        out.append((ns, lay))
    return out


def _dev_plan(lay):
    seg_begin = torch.from_numpy(lay.seg_begin.copy()).to(DEV)
    raw = np.frombuffer(lay.segs.tobytes(), dtype=np.uint8).copy()
    return seg_begin, torch.from_numpy(raw).to(DEV)


def _launch(fold, grads, lay, plan, acc, off, split=2):
    fn = C().grad_fold if fold else C().grad_accumulate
    fn(grads, plan[0], plan[1], lay.grid, split, acc, off, lay.region_elems)


def _grads(ns, dtype, seed, misalign):
    g = torch.Generator(device=DEV).manual_seed(seed)
    out = []
    for n in ns:
        buf = torch.randn(n + misalign, device=DEV, generator=g).mul_(0.5).to(dtype)
        out.append(buf[misalign:])
    return out


def _check_plan(dtype, K, misalign, seed=0):
    buckets = _resnet50_buckets()
    total = sum(lay.region_elems for _, lay in buckets)
    acc = torch.full((total,), SENTINEL, dtype=torch.float32, device=DEV)
    ranges, cur = [], 0
    for ns, lay in buckets:
        for n, o in zip(ns, lay.offsets):
            acc[cur + o:cur + o + n].zero_()          # zero where a tensor lives, sentinel in the padding
            ranges.append((cur + o, n))
        cur += lay.region_elems
    pad = torch.ones(total, dtype=torch.bool, device=DEV)
    for o, n in ranges:
        pad[o:o + n] = False
    passes = [[_grads(ns, dtype, seed + 1000 * k + b, misalign) for b, (ns, _) in enumerate(buckets)] for k in range(K)]
    ref = [[torch.zeros(n, dtype=torch.float32, device=DEV) for n in ns] for ns, _ in buckets]
    for k in range(K):
        cur = 0
        for b, (ns, lay) in enumerate(buckets):
            grads = passes[k][b]
            expect = None
            if k < K - 1:
                for r, g in zip(ref[b], grads):
                    r.add_(g.float())
            else:
                expect = [(r + g.float()).to(dtype) for r, g in zip(ref[b], grads)]
            _launch(k == K - 1, grads, lay, _dev_plan(lay), acc, cur)
            torch.cuda.synchronize()
            for t, (n, o) in enumerate(zip(ns, lay.offsets)):
                a = acc[cur + o:cur + o + n]
                if expect is None:
                    assert torch.equal(a.view(torch.int32), ref[b][t].view(torch.int32)), (dtype, K, k, b, t)
                else:
                    assert torch.equal(grads[t].view(torch.int16 if dtype != torch.float32 else torch.int32),
                                       expect[t].view(torch.int16 if dtype != torch.float32 else torch.int32)), (dtype, K, b, t)
                    assert not a.any(), "accumulator not cleared by the fold"
            cur += lay.region_elems
    assert bool((acc[pad] == SENTINEL).all()), "padding between tensors was written"
    assert int(pad.sum()) > 0


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32])
@pytest.mark.parametrize("K", [1, 2, 3, 4])
def test_kernels_bit_exact_resnet50_plan(dtype, K):
    _check_plan(dtype, K, misalign=0, seed=K)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32])
def test_kernels_misaligned_sources(dtype):
    _check_plan(dtype, 3, misalign=1, seed=7)


def test_fold_fp16_overflow_rounds_to_inf():
    from pytorch_distributed_b200.parallel import plan as P
    ns = [1000, 77]
    offs, total = P.tensor_layout(ns)
    lay = P.build_layout(ns, 1, 2, offs, total)
    plan = _dev_plan(lay)
    acc = torch.zeros(lay.region_elems, dtype=torch.float32, device=DEV)
    sign = [torch.where(torch.arange(n, device=DEV) % 2 == 0, 1.0, -1.0) for n in ns]
    g1 = [(s * 40000.0).half() for s in sign]
    g2 = [(s * 40000.0).half() for s in sign]
    _launch(False, g1, lay, plan, acc, 0)
    _launch(True, g2, lay, plan, acc, 0)
    torch.cuda.synchronize()
    for s, g in zip(sign, g2):
        want = (s * 40000.0 + s * 40000.0).half()
        assert torch.equal(g, want) and bool(torch.isinf(g).all())
    assert not acc.any()


# ------------------------------------------------------------------------------------------------ engine (world 1, bf16 ResNet-50)
def _build(argv, entry="distributed", seed=0):
    from pytorch_distributed_b200 import cli, driver
    from pytorch_distributed_b200.models import create_model
    torch.cuda.set_device(0)
    args = cli.parse_args(entry, ["-a", "resnet50", "-b", "8", "--synthetic", "--image-size", "64", "--quiet"] + argv)
    st = driver.STRATEGIES[entry]()
    torch.manual_seed(seed)
    model = create_model(args.arch, num_classes=args.num_classes, fused_bn=args.fused_bn)
    model, opt = st.build(model, args, torch.device(DEV, 0), 0)
    model.train()
    return st, model, opt


def _batch(dtype, seed, bad=False):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(8, 3, 64, 64, device=DEV, generator=g)
    if bad:
        x.fill_(6e4)
    y = torch.randint(0, 1000, (8,), device=DEV, generator=g)
    return x.to(dtype).contiguous(memory_format=CL), y


def _metrics(st):
    from pytorch_distributed_b200 import driver
    return driver.MetricPipeline(st.comm, torch.device(DEV, 0), (driver.AverageMeter("l"), driver.AverageMeter("a"),
                                                                  driver.AverageMeter("b")))


def _state(opt, model):
    inner = getattr(opt, "optim", opt)
    fs = inner._flat
    bufs = [b.detach().clone() for b in model.buffers()]
    stats = opt.larc_stats().clone() if getattr(inner, "_larc", None) is not None else None
    return fs.master.clone(), fs.momentum.clone(), stats, bufs


def _accumulated(argv, K, steps, graph=False, warmup=1):
    from pytorch_distributed_b200 import driver
    st, model, opt = _build(argv + ["--accum-steps", str(K)])
    metrics = _metrics(st)
    step = driver.TrainStep(st, model, torch.nn.CrossEntropyLoss().to(DEV), opt, metrics, use_graph=graph, warmup=warmup)
    vals = []
    for i in range(K * steps):
        step(*_batch(st.input_dtype, seed=i))
        torch.cuda.synchronize()
        metrics.drain()
        vals.append(metrics.last)
    assert st.engine.fp32_accum and not st.engine.accum_pending and not st.engine._acc.any()
    return st, step, _state(opt, model), vals


def _oracle(argv, K, steps):
    """The single-pass path fed p.grad = round(fp32 sum of the K micro-batch gradients of loss / K)."""
    st, model, opt = _build(argv)
    eng = st.engine
    assert not eng.fp32_accum
    crit = torch.nn.CrossEntropyLoss().to(DEV)
    for s in range(steps):
        total = None
        for k in range(K):
            if eng.bucket_view:
                eng.zero_grads()
            else:
                opt.zero_grad()
            x, y = _batch(st.input_dtype, seed=s * K + k)
            with model.no_sync():
                (crit(st.forward(model, x).float(), y) / K).backward()
            if total is None:
                total = [torch.zeros_like(p, dtype=torch.float32) for p in eng.params]
            for t, p in zip(total, eng.params):
                t.add_(p.grad.float())
        if eng.bucket_view:
            eng.zero_grads()
            for p, t in zip(eng.params, total):
                p.grad.copy_(t.to(p.dtype))
        else:
            for p, t in zip(eng.params, total):
                g = torch.empty_like(p)             # p's strides: the arena holds gradients in the parameter's memory order
                g.copy_(t.to(p.dtype))
                p.grad = g
        eng.reduce_now()
        opt.step()
        torch.cuda.synchronize()
    return _state(opt, model)


ENGINE_MODES = {"overlap": [], "no_overlap": ["--no-overlap-optimizer"], "bucket_view": ["--bucket-view"], "larc": ["--larc"]}


def _assert_bits(name, a, b):
    assert a.dtype == b.dtype and a.shape == b.shape, name
    ia = a.view(torch.int32) if a.dtype == torch.float32 else a.view(torch.int16) if a.element_size() == 2 else a
    ib = b.view(torch.int32) if b.dtype == torch.float32 else b.view(torch.int16) if b.element_size() == 2 else b
    diff = int((ia != ib).sum())
    assert diff == 0, "%s: %d elements differ" % (name, diff)


@pytest.mark.parametrize("mode", list(ENGINE_MODES))
def test_engine_matches_single_pass_on_oracle_sum(mode, deterministic):
    argv = ENGINE_MODES[mode]
    _, _, got, _ = _accumulated(argv, 3, 2)
    want = _oracle(argv, 3, 2)
    _assert_bits(mode + " master", got[0], want[0])
    _assert_bits(mode + " momentum", got[1], want[1])
    if mode == "larc":
        _assert_bits("larc_stats", got[2], want[2])
    for i, (a, b) in enumerate(zip(got[3], want[3])):
        _assert_bits("%s buffer %d" % (mode, i), a, b)


def test_no_new_kernel_without_accumulation(deterministic):
    """fp32_grad_accumulation on with single-pass steps: the same launches and bits as with it off."""
    from pytorch_distributed_b200 import _ext, driver
    out = []
    for accum in (False, True):
        st, model, opt = _build(["--accum-steps", "2"] if accum else [])
        assert st.engine.fp32_accum == accum
        st.accum_steps = 1
        step = driver.TrainStep(st, model, torch.nn.CrossEntropyLoss().to(DEV), opt, _metrics(st))
        step(*_batch(st.input_dtype, seed=0))
        n0 = _ext.launches
        step(*_batch(st.input_dtype, seed=1))
        torch.cuda.synchronize()
        out.append((_ext.launches - n0, _state(opt, model)))
    assert out[0][0] == out[1][0]
    _assert_bits("master", out[0][1][0], out[1][1][0])
    _assert_bits("momentum", out[0][1][1], out[1][1][1])


@pytest.mark.parametrize("K", [2, 3])
def test_graph_matches_eager(K, deterministic):
    _, _, eager, ve = _accumulated([], K, 3, graph=False)
    _, step, graph, vg = _accumulated([], K, 3, graph=True)
    assert step.graph is not None and step.graph_accum is not None          # exactly two graphs: one per kind of pass
    assert step.graph_launches > step.graph_accum_launches > 0
    _assert_bits("master", eager[0], graph[0])
    _assert_bits("momentum", eager[1], graph[1])
    for i, (a, b) in enumerate(zip(eager[3], graph[3])):
        _assert_bits("buffer %d" % i, a, b)
    assert ve == vg


def test_step_before_synchronising_backward_raises():
    st, model, opt = _build(["--accum-steps", "2"])
    x, y = _batch(st.input_dtype, seed=0)
    with model.no_sync():
        torch.nn.functional.cross_entropy(model(x).float(), y).backward()
    with pytest.raises(RuntimeError, match="no_sync"):
        opt.step()


# ------------------------------------------------------------------------------------------------ apex O2, fp16, dynamic scale
def _apex_run(batches, init_scale=None):
    from pytorch_distributed_b200 import driver
    from pytorch_distributed_b200.parallel import amp as _amp
    st, model, opt = _build(["--opt-level", "O2", "--precision", "fp16", "--accum-steps", "3"], entry="apex_distributed")
    scaler = _amp._amp_state.scaler
    assert scaler.dynamic and st.engine.check_inf and st.engine.fp32_accum
    if init_scale is not None:
        scaler.scale.fill_(init_scale)
    step = driver.TrainStep(st, model, torch.nn.CrossEntropyLoss().to(DEV), opt, _metrics(st))
    snaps = []
    for i, (seed, bad) in enumerate(batches):
        step(*_batch(st.input_dtype, seed=seed, bad=bad))
        if i % 3 == 2:
            torch.cuda.synchronize()
            snaps.append((opt._flat.master.clone(), opt._flat.momentum.clone(), float(scaler.scale.item()),
                          bool(st.engine._acc.any())))
    return snaps


def test_apex_o2_overflow_in_one_micro_batch_skips_the_step(deterministic):
    from pytorch_distributed_b200.parallel import amp as _amp
    st, model, opt = _build(["--opt-level", "O2", "--precision", "fp16", "--accum-steps", "3"], entry="apex_distributed")
    opt._try_bind()                 # amp before DDP: the optimizer binds to the arena at its first step; bind now to read it
    master0, mom0, s0 = opt._flat.master.clone(), opt._flat.momentum.clone(), float(_amp._amp_state.scaler.scale.item())
    del st, model, opt
    got = _apex_run([(0, False), (1, True), (2, False), (3, False), (4, False), (5, False)])
    m1, v1, s1, acc1 = got[0]
    _assert_bits("master after the skipped step", m1, master0)
    _assert_bits("momentum after the skipped step", v1, mom0)
    assert s1 == s0 / 2 and not acc1
    ref = _apex_run([(3, False), (4, False), (5, False)], init_scale=s0 / 2)
    _assert_bits("master", got[1][0], ref[0][0])
    _assert_bits("momentum", got[1][1], ref[0][1])
    assert got[1][2] == ref[0][2] and not got[1][3]


# ------------------------------------------------------------------------------------------------ entrypoints
COMMON = ["-a", "resnet50", "-b", "32", "--synthetic", "--steps-per-epoch", "6", "--val-steps", "1", "--epochs", "1",
          "--image-size", "96", "-p", "1", "--accum-steps", "2", "--cuda-graph"]


@pytest.mark.parametrize("script,extra,port", [("distributed.py", [], 29801),
                                               ("apex_distributed.py", ["--opt-level", "O2"], 29802),
                                               ("horovod_distributed.py", [], 29803)])
def test_entrypoint_accum_cuda_graph(script, extra, port, tmp_path):
    e = dict(os.environ, PYTHONPATH=ROOT)
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "MASTER_ADDR", "MASTER_PORT"):
        e.pop(k, None)
    log = tmp_path / "log.jsonl"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "1", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, script)] + COMMON + extra + ["--checkpoint-dir", str(tmp_path),
                                                                                      "--log-jsonl", str(log)]
    p = subprocess.run(cmd, env=e, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-3000:] + "\n" + p.stderr[-3000:]
    assert "--cuda-graph ignored" not in p.stdout
    losses = [float(x) for x in re.findall(r"Loss ([0-9.e+-]+|nan|inf) \(", p.stdout)]
    assert losses and all(math.isfinite(x) for x in losses), p.stdout[-2000:]
    import json
    rec = [json.loads(l) for l in open(log) if '"train"' in l][0]
    assert rec["accum_steps"] == 2 and rec["optimizer_steps"] == 3
