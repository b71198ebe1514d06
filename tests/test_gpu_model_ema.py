"""ModelEma in the fused SGD kernels (csrc/optim.cu) on one GPU: every EMA variant against float64 at ResNet-50 parameter
shapes, bit-identity of the masters / momentum / model copy with and without the EMA epilogue, the overflow skip,
bit-identity of the average across the flat, per-bucket, eager and CUDA-graph paths (with a decay changed between
replays), an EMA validation between replays, and the training entrypoints."""
import gc
import json
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
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = R.U32
D = 0.999


@pytest.fixture(autouse=True)
def _release_memory():
    """The kernel tests allocate ResNet-50-sized flat buffers: hand them back to the device after each test, so that the
    training subprocesses of this and later test files find the memory free."""
    yield
    gc.collect()
    if torch.cuda.is_available():
        torch.cuda.synchronize()
        torch.cuda.empty_cache()


def C():
    from pytorch_distributed_b200 import _ext
    return _ext.lib()


def hyper_t(decay=D, lr=0.1, mom=0.9, wd=1e-4, gmul=1.0):
    from pytorch_distributed_b200.utils.ema import decay_pair
    return torch.tensor([lr, mom, wd, 0.0, gmul, 0.0, *decay_pair(decay)], dtype=F32, device=DEV)


def check_ema(name, e1, e0, p, hyper):
    """e1 = fmaf(d, e0, w p) in fp32 against d e0 + (1 - d) p in float64, d and w as the kernel read them (w may differ
    from 1 - d by the rounding of fp32(1 - d)): the product w p is rounded once (u |w p|), the fmaf once (u |e1|)."""
    d, w = float(hyper[6]), float(hyper[7])
    e0, p = e0.double(), p.double()
    ref = d * e0 + (1 - d) * p
    tol = U * (abs(w) * p.abs() + e1.double().abs()) + abs(w - (1 - d)) * p.abs()
    R.assert_within(name, e1, ref, tol)
    assert bool((e1 != e0).any()), name + ": the average did not move"


def r50_params():
    from pytorch_distributed_b200.models import create_model
    torch.manual_seed(0)
    return [p.detach().to(DEV) for p in create_model("resnet50").parameters()]


class Flat:
    """ResNet-50 parameters in the gradient engine's arena layout, with random gradients, momentum and average."""

    def __init__(self, gdt, cdt, seed=0):
        from pytorch_distributed_b200.parallel import plan as P
        ps = r50_params()
        self.numels = [p.numel() for p in ps]
        self.offs, self.n = P.tensor_layout(self.numels)
        gen = torch.Generator(device=DEV).manual_seed(seed)
        self.master = torch.zeros(self.n, device=DEV)
        for p, o in zip(ps, self.offs):
            self.master[o:o + p.numel()] = p.flatten()
        self.grad = (torch.randn(self.n, device=DEV, generator=gen) * 0.01).to(gdt)
        self.mom = torch.randn(self.n, device=DEV, generator=gen) * 0.01
        self.ema = self.master + torch.randn(self.n, device=DEV, generator=gen) * 0.01
        self.copy = torch.zeros(self.n, dtype=cdt, device=DEV) if cdt is not None else None
        chunk = C().LARC_CHUNK
        info, ct = [], []
        for i, (k, o) in enumerate(zip(self.numels, self.offs)):
            info.append((o, k, len(ct), i))
            ct += [i] * R.cdiv(k, chunk)
        self.chunks = len(ct)
        self.ct = torch.tensor(ct, dtype=torch.int32, device=DEV)
        self.info = torch.tensor(info, dtype=torch.int64, device=DEV)

    def clone(self):
        return [t.clone() if t is not None else None for t in (self.master, self.mom, self.copy, self.ema)]

    def sgd(self, bufs, hyper, nesterov, found_inf=None, ema=True, first=False):
        p, m, c, e = bufs
        C().fused_sgd_flat(self.grad, p, m, c, hyper, found_inf, nesterov, first, ema=e if ema else None)

    def larc(self, bufs, hyper, nesterov, found_inf=None, ema=True):
        p, m, c, e = bufs
        stats = torch.zeros(len(self.numels), 3, device=DEV)
        C().larc_sgd_flat(self.grad, p, m, c, hyper, found_inf, nesterov, False, self.ct, self.info, 0, self.chunks,
                          torch.zeros(2 * self.chunks, device=DEV), stats, 0.02, 1e-8, True, ema=e if ema else None)

    def live(self, t):
        """the parameters' elements (the padding between tensors is not part of the average's contract)"""
        return torch.cat([t[o:o + k] for o, k in zip(self.offs, self.numels)])


def _assert_same_step(name, a, b):
    for what, x, y in zip(("master", "momentum", "copy"), a[:3], b[:3]):
        if x is not None:
            R.assert_bits_equal("%s %s with / without EMA" % (name, what), x, y)


FLAT_CASES = [(BF16, BF16), (BF16, None), (F16, F16), (F16, None), (F32, BF16), (F32, None)]


@pytest.mark.parametrize("nesterov", [False, True], ids=["plain", "nesterov"])
@pytest.mark.parametrize("gdt,cdt", FLAT_CASES, ids=lambda d: str(d).replace("torch.", ""))
def test_flat_against_fp64(gdt, cdt, nesterov):
    f = Flat(gdt, cdt)
    h = hyper_t()
    plain, with_ema = f.clone(), f.clone()
    f.sgd(plain, h, nesterov, ema=False)
    f.sgd(with_ema, h, nesterov)
    torch.cuda.synchronize()
    _assert_same_step("fused_sgd_flat", plain, with_ema)
    R.assert_bits_equal("untouched EMA of the plain step", plain[3], f.ema)
    check_ema("fused_sgd_flat EMA", f.live(with_ema[3]), f.live(f.ema), f.live(with_ema[0]), h)


@pytest.mark.parametrize("gdt,cdt", [(BF16, BF16), (F32, None)], ids=lambda d: str(d).replace("torch.", ""))
def test_larc_flat_against_fp64(gdt, cdt):
    f = Flat(gdt, cdt)
    h = hyper_t()
    plain, with_ema = f.clone(), f.clone()
    f.larc(plain, h, False, ema=False)
    f.larc(with_ema, h, False)
    torch.cuda.synchronize()
    _assert_same_step("larc_sgd_flat", plain, with_ema)
    check_ema("larc_sgd_flat EMA", f.live(with_ema[3]), f.live(f.ema), f.live(with_ema[0]), h)


def _lists(seed=0, low=BF16):
    ps = r50_params()
    gen = torch.Generator(device=DEV).manual_seed(seed)
    grads = [(torch.randn(p.shape, device=DEV, generator=gen) * 0.01).to(low) for p in ps]
    mom = [torch.randn(p.shape, device=DEV, generator=gen) * 0.01 for p in ps]
    ema = [p + torch.randn(p.shape, device=DEV, generator=gen) * 0.01 for p in ps]
    copies = [p.to(low) for p in ps]
    return grads, ps, mom, copies, ema


def _cl(ts):
    return [t.clone() for t in ts]


@pytest.mark.parametrize("kind", ["sgd", "larc"])
def test_multi_against_fp64(kind):
    g, p, m, c, e = _lists()
    h = hyper_t()
    runs = []
    for ema in (False, True):
        pp, mm, cc, ee = _cl(p), _cl(m), _cl(c), _cl(e)
        if kind == "sgd":
            C().fused_sgd_multi(g, pp, mm, cc, h, None, False, False, ema=ee if ema else [])
        else:
            C().larc_sgd_multi(g, pp, mm, cc, h, None, False, [False] * len(p), list(range(len(p))),
                               torch.zeros(len(p), 3, device=DEV), 0.02, 1e-8, True, ema=ee if ema else [])
        runs.append((torch.cat([x.flatten() for x in pp]), torch.cat([x.flatten() for x in mm]),
                     torch.cat([x.flatten() for x in cc]), torch.cat([x.flatten() for x in ee])))
    torch.cuda.synchronize()
    _assert_same_step(kind + "_multi", runs[0], runs[1])
    e0 = torch.cat([x.flatten() for x in e])
    R.assert_bits_equal("untouched EMA without the list", runs[0][3], e0)
    check_ema(kind + "_multi EMA", runs[1][3], e0, runs[1][0], h)


@pytest.mark.parametrize("sdt", [F32, BF16, F16])
def test_ema_multi_against_fp64(sdt):
    _, p, _, _, e = _lists()
    src = [x.to(sdt) for x in p]
    h = hyper_t()
    ee = _cl(e)
    C().ema_multi(src, ee, h[6:8], None)
    torch.cuda.synchronize()
    check_ema("ema_multi", torch.cat([x.flatten() for x in ee]), torch.cat([x.flatten() for x in e]),
              torch.cat([x.float().flatten() for x in src]), h)


def test_endpoints_are_exact():
    f = Flat(BF16, BF16)
    for decay in (0.0, 1.0):
        b = f.clone()
        f.sgd(b, hyper_t(decay), False)
        torch.cuda.synchronize()
        R.assert_bits_equal("d = %g" % decay, f.live(b[3]), f.live(b[0] if decay == 0.0 else f.ema))


def test_found_inf_leaves_the_average_bitwise():
    f = Flat(F16, F16)
    h = hyper_t()
    flag = torch.ones(1, dtype=torch.int32, device=DEV)
    b = f.clone()
    f.sgd(b, h, False, found_inf=flag)
    f.larc(b, h, False, found_inf=flag)
    g, p, m, c, e = _lists(low=F16)
    ee = _cl(e)
    C().fused_sgd_multi(g, _cl(p), _cl(m), _cl(c), h, flag, False, False, ema=ee)
    C().ema_multi(p, ee, h[6:8], flag)
    torch.cuda.synchronize()
    R.assert_bits_equal("flat EMA after a skipped step", b[3], f.ema)
    for x, y in zip(ee, e):
        R.assert_bits_equal("multi EMA after a skipped step", x, y)


# ------------------------------------------------------------------------------------------------ through the engine
# Each comparison trains in a child process (tests/model_ema_paths.py): the communicator arenas, graph pools and cached
# blocks of a DDP engine stay with the process that made them, and the later subprocess tests need that memory.
def _paths(tmp_path, runs):
    out = tmp_path / "paths.pt"
    e = dict(os.environ, PYTHONPATH=ROOT)
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "MASTER_ADDR", "MASTER_PORT"):
        e.pop(k, None)
    p = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "model_ema_paths.py"), str(out), json.dumps(runs)], env=e,
                       cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-3000:] + "\n" + p.stderr[-3000:]
    return torch.load(out, weights_only=False)


def _same(tag, a, b):
    R.assert_bits_equal(tag + " master", a["master"], b["master"])
    for part in ("ema", "live"):
        assert a[part].keys() == b[part].keys()
        for k in a[part]:
            R.assert_bits_equal("%s %s %s" % (tag, part, k), a[part][k], b[part][k])


def test_flat_overlap_eager_graph_bit_identical(tmp_path):
    """A decay changed before the third step reaches the eager steps and the graph replays alike."""
    cases = [(["--no-overlap-optimizer"], False), ([], False), ([], True), (["--no-overlap-optimizer"], True)]
    got = _paths(tmp_path, [{"argv": a, "graph": g, "decay_at": 2} for a, g in cases])
    for (argv, graph), r in zip(cases[1:], got[1:]):
        _same("%s graph=%s" % (argv, graph), got[0], r)


def test_ema_validation_between_replays_changes_nothing(tmp_path):
    got = _paths(tmp_path, [{"graph": True}, {"graph": True, "eval_at": 2}])
    _same("eval between replays", got[0], got[1])


def test_larc_engine_average_matches_eager(tmp_path):
    got = _paths(tmp_path, [{"argv": ["--larc"]}, {"argv": ["--larc"], "graph": True}])
    _same("larc graph", got[0], got[1])


# ------------------------------------------------------------------------------------------------ entrypoints
COMMON = ["-a", "resnet50", "-b", "32", "--synthetic", "--steps-per-epoch", "4", "--val-steps", "1", "--epochs", "1",
          "--image-size", "96", "-p", "1", "--model-ema", "--model-ema-decay", "0.9"]


@pytest.mark.parametrize("script,extra,port", [
    ("distributed.py", ["--cuda-graph"], 29811),
    ("distributed.py", ["--cuda-graph", "--accum-steps", "2"], 29812),
    ("distributed.py", ["--cuda-graph", "--larc"], 29813),
    ("distributed.py", ["--optimizer", "torch"], 29814),
    ("apex_distributed.py", ["--opt-level", "O2", "--precision", "fp16"], 29815),
    ("horovod_distributed.py", ["--cuda-graph"], 29816),
    ("dataparallel.py", [], None),
], ids=["ddp-graph", "ddp-accum2", "ddp-larc", "torch-sgd", "apex-o2", "horovod", "dataparallel"])
def test_entrypoint_model_ema(script, extra, port, tmp_path):
    e = dict(os.environ, PYTHONPATH=ROOT)
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "MASTER_ADDR", "MASTER_PORT"):
        e.pop(k, None)
    args = COMMON + extra + ["--checkpoint-dir", str(tmp_path)]
    if port is None:
        cmd = [sys.executable, os.path.join(ROOT, script), "--gpus", "0"] + args
    else:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "1", "--master-addr", "127.0.0.1",
               "--master-port", str(port), os.path.join(ROOT, script)] + args
    p = subprocess.run(cmd, env=e, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-3000:] + "\n" + p.stderr[-3000:]
    assert " * EMA Acc@1 " in p.stdout and " * Acc@1 " in p.stdout, p.stdout[-2000:]
    ck = torch.load(tmp_path / "checkpoint.pth.tar", weights_only=False)
    sde = ck["state_dict_ema"]
    assert list(sde.keys()) == list(ck["state_dict"].keys())
    assert all(torch.isfinite(v).all() for v in sde.values() if v.is_floating_point())
    assert any(not torch.equal(sde[k], ck["state_dict"][k]) for k in sde if sde[k].is_floating_point())
