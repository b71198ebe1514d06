"""LARC (apex.parallel.LARC) without a GPU: the Python wrapper around torch.optim.SGD and FusedSGD's CPU reference path
against a float64 transcription of apex's algorithm, the wrapper's delegation, the command line, and a gloo world-2 run."""
import copy
import os
import subprocess
import sys

import pytest
import torch

from pytorch_distributed_b200 import cli
from pytorch_distributed_b200.ops.fused_sgd import FusedSGD
from pytorch_distributed_b200.parallel.amp import LossScaler
from pytorch_distributed_b200.utils.meters import adjust_learning_rate

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def larc_fp64(p, g, m, lr, momentum, wd, dampening, nesterov, first, trust, clip, eps):
    """apex.parallel.LARC + torch.optim.SGD(weight_decay=0) on one tensor, in float64.  Returns (p, m, (pn, gn, f))."""
    p, g, m = p.double(), g.double(), m.double()
    pn, gn = float(p.norm()), float(g.norm())
    f = 1.0
    if pn != 0 and gn != 0:
        f = trust * pn / (gn + pn * wd + eps)
        if clip:
            f = min(f / lr, 1.0)
        g = (g + wd * p) * f
    if momentum != 0:
        m = g.clone() if first else momentum * m + (1 - dampening) * g
        g = g + momentum * m if nesterov else m
    return p - lr * g, m, (pn, gn, f)


def _params(seed, zero_p=False, zero_g=False):
    gen = torch.Generator().manual_seed(seed)
    shapes = [(64, 3, 7, 7), (64,), (256, 64, 1, 1), (1000, 2048), (1000,)]
    ps = [torch.randn(s, generator=gen) * 0.05 for s in shapes]
    # gradient scales chosen so that clip mode both saturates (f / lr > 1) and does not
    gs = [torch.randn(s, generator=gen) * k for s, k in zip(shapes, (1e-3, 0.05, 0.05, 0.5, 1e-3))]
    if zero_p:
        ps[1].zero_()          # a BatchNorm beta at initialisation
    if zero_g:
        gs[4].zero_()
    return ps, gs


CASES = [
    dict(clip=True, wd=1e-4, momentum=0.9, dampening=0.0, nesterov=False),
    dict(clip=False, wd=1e-4, momentum=0.9, dampening=0.0, nesterov=False),
    dict(clip=True, wd=0.0, momentum=0.9, dampening=0.0, nesterov=False),
    dict(clip=True, wd=5e-4, momentum=0.9, dampening=0.0, nesterov=True),
    dict(clip=False, wd=1e-4, momentum=0.9, dampening=0.3, nesterov=False),
    dict(clip=True, wd=1e-4, momentum=0.0, dampening=0.0, nesterov=False),
]


def _run(kind, case, steps=3, zero_p=True, zero_g=True, trust=0.02, lr=0.1, eps=1e-8):
    from pytorch_distributed_b200.apex.parallel import LARC
    ps, gs = _params(0, zero_p, zero_g)
    params = [torch.nn.Parameter(p.clone()) for p in ps]
    kw = dict(lr=lr, momentum=case["momentum"], dampening=case["dampening"], weight_decay=case["wd"], nesterov=case["nesterov"])
    inner = torch.optim.SGD(params, **kw) if kind == "torch" else FusedSGD(params, **kw)
    opt = LARC(inner, trust_coefficient=trust, clip=case["clip"], eps=eps)
    ref_p = [p.double() for p in ps]
    ref_m = [torch.zeros_like(p, dtype=torch.float64) for p in ps]
    for s in range(steps):
        grads = [g * (1 + s) + 1e-4 * s for g in gs]
        if zero_g:
            grads[4] = gs[4].clone()
        for p, g in zip(params, grads):
            p.grad = g.clone()
        opt.step()
        stats = []
        for i in range(len(ps)):
            ref_p[i], ref_m[i], st = larc_fp64(ref_p[i], grads[i], ref_m[i], lr, case["momentum"], case["wd"], case["dampening"],
                                               case["nesterov"], s == 0, trust, case["clip"], eps)
            stats.append(st)
        for i, p in enumerate(params):
            # fp32 norms over up to 2M terms: a relative error of a few 1e-7 in f, scaled by the largest weight
            torch.testing.assert_close(p.detach().double(), ref_p[i], rtol=2e-5, atol=1e-5 * float(ref_p[i].abs().max()))
        if kind == "fused":
            assert opt.larc_stats().shape == (len(ps), 3)
            # torch's fp32 CPU norm of the 2M-element tensor is good to ~1e-5 relative
            torch.testing.assert_close(opt.larc_stats().double(), torch.tensor(stats, dtype=torch.float64), rtol=1e-4, atol=1e-9)
    return opt, params


@pytest.mark.parametrize("kind", ["torch", "fused"])
@pytest.mark.parametrize("ci", range(len(CASES)))
def test_larc_matches_fp64(kind, ci):
    _run(kind, CASES[ci])


def test_zero_norm_branch_gets_no_weight_decay():
    """apex leaves g as is where a norm is zero: a zero beta with a gradient moves by lr * g, a tensor with a zero gradient
    does not move at all, even with weight decay."""
    from pytorch_distributed_b200.apex.parallel import LARC
    beta = torch.nn.Parameter(torch.zeros(8))
    w = torch.nn.Parameter(torch.full((8,), 0.5))
    opt = LARC(FusedSGD([beta, w], lr=0.1, momentum=0.0, weight_decay=0.1))
    beta.grad = torch.full((8,), 0.25)
    w.grad = torch.zeros(8)
    opt.step()
    torch.testing.assert_close(beta.detach(), torch.full((8,), -0.025))
    assert torch.equal(w.detach(), torch.full((8,), 0.5))
    assert opt.larc_stats()[0].tolist() == [0.0, pytest.approx(0.25 * 8 ** 0.5), 1.0]


def test_loss_scaled_gradient_and_skipped_first_step():
    """gmul = 1 / loss scale: the fused CPU path unscales before the norms; a first step with found_inf changes nothing and
    the next one still initialises the momentum."""
    from pytorch_distributed_b200.apex.parallel import LARC
    case = CASES[0]
    ps, gs = _params(1, zero_p=True)
    params = [torch.nn.Parameter(p.clone()) for p in ps]
    opt = LARC(FusedSGD(params, lr=0.1, momentum=0.9, weight_decay=case["wd"]))
    scaler = LossScaler("cpu", "dynamic", init_scale=2.0 ** 16)
    opt._amp = scaler
    assert opt.optim._amp is scaler                   # amp.initialize sets _amp on whatever it is given
    for p, g in zip(params, gs):
        p.grad = g * 2.0 ** 16
    scaler.found_inf.fill_(1)
    opt.step()
    for p, p0 in zip(params, ps):
        assert torch.equal(p.detach(), p0)
    assert opt.larc_stats() is None
    assert scaler.loss_scale() == 2.0 ** 15
    for p, g in zip(params, gs):
        p.grad = g * 2.0 ** 15
    opt.step()
    for i, p in enumerate(params):
        ref, _, _ = larc_fp64(ps[i], gs[i], torch.zeros_like(ps[i]), 0.1, 0.9, case["wd"], 0.0, False, True, 0.02, True, 1e-8)
        torch.testing.assert_close(p.detach().double(), ref, rtol=2e-5, atol=1e-5 * float(ref.abs().max()))


def test_state_dict_round_trip():
    from pytorch_distributed_b200.apex.parallel import LARC
    opt, params = _run("fused", CASES[0], steps=2)
    sd = copy.deepcopy(opt.state_dict())          # torch's load_state_dict keeps the tensors it is given
    twin = [torch.nn.Parameter(p.detach().clone()) for p in params]
    opt2 = LARC(FusedSGD(twin, lr=0.1, momentum=0.9, weight_decay=1e-4))
    opt2.load_state_dict(sd)
    gen = torch.Generator().manual_seed(5)
    for a, b in zip(params, twin):
        a.grad = torch.randn(a.shape, generator=gen) * 1e-3
        b.grad = a.grad.clone()
    opt.step()
    opt2.step()
    for a, b in zip(params, twin):
        assert torch.equal(a.detach(), b.detach())
    for a, b in zip(params, twin):
        assert torch.equal(opt.state[a]["momentum_buffer"], opt2.state[b]["momentum_buffer"])


def test_adjust_learning_rate_changes_the_clip():
    from pytorch_distributed_b200.apex.parallel import LARC
    p = torch.nn.Parameter(torch.full((16,), 1.0))
    opt = LARC(FusedSGD([p], lr=0.1, momentum=0.9, weight_decay=0.0))
    args = cli.parse_args("distributed", ["--lr", "0.1"])
    p.grad = torch.full((16,), 1.0)
    adjust_learning_rate(opt, 0, args)
    opt.step()
    f0 = float(opt.larc_stats()[0, 2])
    assert f0 == pytest.approx(0.02 / 0.1, rel=1e-6)          # trust * pn / gn = 0.02, divided by lr = 0.1
    adjust_learning_rate(opt, 60, args)                        # lr 0.001: 0.02 / 0.001 > 1 is clipped
    assert opt.param_groups[0]["lr"] == pytest.approx(0.001)
    p.grad = torch.full((16,), 1.0)
    opt.step()
    assert float(opt.larc_stats()[0, 2]) == 1.0


def test_import_paths_and_delegation():
    import pytorch_distributed_b200.apex.parallel as ap
    from pytorch_distributed_b200.apex.parallel.LARC import LARC
    assert ap.LARC is LARC
    p = torch.nn.Parameter(torch.ones(4))
    inner = FusedSGD([p], lr=0.1, momentum=0.9)
    opt = LARC(inner, trust_coefficient=0.001, clip=False)
    assert inner._larc == (0.001, False, 1e-8)
    assert opt.param_groups is inner.param_groups and opt.state is inner.state
    assert hasattr(opt, "refresh_hyper") and hasattr(opt, "is_flat") and opt.is_flat is False and opt._flat is None
    opt.add_param_group({"params": [torch.nn.Parameter(torch.ones(2))]})
    assert len(inner.param_groups) == 2
    opt.something = 3
    assert inner.something == 3
    plain = LARC(torch.optim.SGD([torch.nn.Parameter(torch.ones(2))], lr=0.1))
    assert not hasattr(plain, "refresh_hyper") and not hasattr(plain, "is_flat")
    assert "LARC(" in repr(opt)


def test_hvd_style_subclass_wrap():
    """hvd.DistributedOptimizer subclasses the optimizer's class and shares its __dict__."""
    from pytorch_distributed_b200.apex.parallel import LARC
    p = torch.nn.Parameter(torch.full((4,), 2.0))
    opt = LARC(FusedSGD([p], lr=0.1, momentum=0.0))

    class Sub(LARC):
        def __init__(self):
            pass

        def step(self, closure=None):
            return LARC.step(self)

    w = Sub.__new__(Sub)
    w.__dict__ = opt.__dict__
    w._ptd_engine_obj = "engine"
    assert getattr(w, "_ptd_engine_obj") == "engine" and w.optim is opt.optim
    p.grad = torch.full((4,), 1.0)
    w.step()
    assert w.larc_stats() is not None and not torch.equal(p.detach(), torch.full((4,), 2.0))


def test_cli_flags():
    a = cli.parse_args("distributed", [])
    assert a.larc is False and a.larc_trust_coefficient == 0.02 and a.larc_clip is True
    a = cli.parse_args("apex_distributed", ["--larc", "--larc-trust-coefficient", "0.001", "--no-larc-clip"])
    assert a.larc is True and a.larc_trust_coefficient == 0.001 and a.larc_clip is False
    assert cli.parse_args("horovod_distributed", ["--larc", "--larc-clip"]).larc_clip is True
    assert cli.parse_args("dataparallel", ["--larc"]).larc is True
    for bad in (["--larc", "--larc-trust-coefficient", "0"], ["--larc", "--larc-trust-coefficient", "-1"],
                ["--larc", "--larc-trust-coefficient", "nan"], ["--larc-trust-coefficient", "0.01"], ["--no-larc-clip"]):
        with pytest.raises(SystemExit):
            cli.parse_args("distributed", bad)


@pytest.mark.parametrize("optimizer", ["fused", "torch"])
def test_make_optimizer_wraps(optimizer):
    from pytorch_distributed_b200 import driver
    from pytorch_distributed_b200.apex.parallel import LARC
    args = cli.parse_args("distributed", ["--larc", "--optimizer", optimizer, "--no-larc-clip"])
    opt = driver.Strategy().make_optimizer(torch.nn.Linear(4, 4), args)
    assert isinstance(opt, LARC) and opt.clip is False and opt.trust_coefficient == 0.02
    plain = driver.Strategy().make_optimizer(torch.nn.Linear(4, 4), cli.parse_args("distributed", ["--optimizer", optimizer]))
    assert not isinstance(plain, LARC)


def test_distributed_gloo_world2_ranks_agree(tmp_path):
    common = ["-a", "resnet18", "-b", "8", "--synthetic", "--steps-per-epoch", "3", "--epochs", "1", "--image-size", "32",
              "--num-classes", "10", "-p", "1", "--device", "cpu", "--checkpoint-dir", str(tmp_path), "--quiet", "--larc"]
    env = dict(os.environ, OMP_NUM_THREADS="1", PYTHONPATH=ROOT)
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "MASTER_ADDR", "MASTER_PORT"):
        env.pop(k, None)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29741", os.path.join(ROOT, "tests", "mp_larc_checks.py"), str(tmp_path / "out"), "distributed"] + common
    p = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stdout[-3000:] + "\n" + p.stderr[-3000:]
    r0 = torch.load(tmp_path / "out" / "rank0.pt", weights_only=False)
    r1 = torch.load(tmp_path / "out" / "rank1.pt", weights_only=False)
    assert r0["stats"] is not None and len(r0["masters"]) == len(r1["masters"]) > 0
    for a, b in zip(r0["masters"] + r0["momenta"], r1["masters"] + r1["momenta"]):
        assert torch.equal(a, b)
    assert torch.equal(r0["stats"], r1["stats"])
    assert (r0["stats"][:, 2] > 0).all()


@pytest.fixture
def amp_state():
    """amp.initialize configures process-wide state: put it back afterwards."""
    from pytorch_distributed_b200.parallel import amp
    st = amp._amp_state
    saved = dict(vars(st))
    yield amp
    vars(st).clear()
    vars(st).update(saved)


@pytest.mark.parametrize("opt_level", ["O0", "O1"])
def test_amp_initialize_with_larc_around_torch_sgd(amp_state, opt_level):
    """amp patches the step of the object it is given; LARC's own step must stay under that patch and call the unpatched
    inner step (otherwise each step re-enters LARC)."""
    from pytorch_distributed_b200.apex.parallel import LARC
    amp = amp_state
    torch.manual_seed(0)
    model = torch.nn.Linear(16, 8)
    p0 = [p.detach().clone() for p in model.parameters()]
    opt = LARC(torch.optim.SGD(model.parameters(), lr=0.1, momentum=0.9, weight_decay=1e-4), trust_coefficient=0.02)
    model, opt = amp.initialize(model, opt, opt_level=opt_level, half_dtype=torch.bfloat16, verbosity=0)
    x = torch.randn(4, 16)
    loss = model(x).float().square().mean()
    with amp.scale_loss(loss, opt) as scaled:
        scaled.backward()
    grads = [p.grad.detach().clone() for p in model.parameters()]
    opt.step()
    for p, p_init, g in zip(model.parameters(), p0, grads):
        ref, _, _ = larc_fp64(p_init, g, torch.zeros_like(p_init), 0.1, 0.9, 1e-4, 0.0, False, True, 0.02, True, 1e-8)
        torch.testing.assert_close(p.detach().double(), ref, rtol=2e-5, atol=1e-7)
    assert all(g["weight_decay"] == 1e-4 for g in opt.param_groups)


def test_larc_settings_reach_the_fused_optimizer():
    from pytorch_distributed_b200.apex.parallel import LARC
    inner = FusedSGD([torch.nn.Parameter(torch.ones(4))], lr=0.1, momentum=0.9)
    opt = LARC(inner)
    opt.clip = False
    opt.trust_coefficient = 0.001
    opt.eps = 1e-6
    assert inner._larc == (0.001, False, 1e-6) and (opt.clip, opt.trust_coefficient, opt.eps) == (False, 0.001, 1e-6)
    with pytest.raises(ValueError):
        opt.trust_coefficient = 0.0
    assert opt.trust_coefficient == 0.001 and inner._larc == (0.001, False, 1e-6)


def test_stats_grow_with_add_param_group():
    from pytorch_distributed_b200.apex.parallel import LARC
    a = torch.nn.Parameter(torch.full((4,), 1.0))
    opt = LARC(FusedSGD([a], lr=0.1, momentum=0.9))
    a.grad = torch.full((4,), 0.5)
    opt.step()
    first = opt.larc_stats()[0].clone()
    b = torch.nn.Parameter(torch.full((3,), 2.0))
    opt.add_param_group({"params": [b]})
    b.grad = torch.full((3,), 1.0)
    a.grad = None
    opt.step()
    st = opt.larc_stats()
    assert st.shape == (2, 3) and torch.equal(st[0], first)
    assert st[1].tolist() == [pytest.approx(2.0 * 3 ** 0.5), pytest.approx(3 ** 0.5), pytest.approx(0.4)]   # 0.02 * 2 / 0.1


def test_apex_distributed_torch_sgd_gloo_world2(tmp_path):
    """`apex_distributed.py --optimizer torch --larc`: amp's patched step around apex's Python LARC loop, two ranks."""
    common = ["-a", "resnet18", "-b", "8", "--synthetic", "--steps-per-epoch", "3", "--epochs", "1", "--image-size", "32",
              "--num-classes", "10", "-p", "1", "--device", "cpu", "--checkpoint-dir", str(tmp_path), "--quiet", "--larc",
              "--optimizer", "torch", "--opt-level", "O1"]
    env = dict(os.environ, OMP_NUM_THREADS="1", PYTHONPATH=ROOT)
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "MASTER_ADDR", "MASTER_PORT"):
        env.pop(k, None)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29742", os.path.join(ROOT, "tests", "mp_larc_checks.py"), str(tmp_path / "out"), "apex_distributed"] + common
    p = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stdout[-3000:] + "\n" + p.stderr[-3000:]
    r0 = torch.load(tmp_path / "out" / "rank0.pt", weights_only=False)
    r1 = torch.load(tmp_path / "out" / "rank1.pt", weights_only=False)
    assert r0["stats"] is None and len(r0["masters"]) > 0 and len(r0["momenta"]) == len(r0["masters"])
    for a, b in zip(r0["masters"] + r0["momenta"], r1["masters"] + r1["momenta"]):
        assert torch.isfinite(a).all() and torch.equal(a, b)
