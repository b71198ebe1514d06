"""Global-norm gradient clipping in the fused SGD step (csrc/optim.cu) on one GPU: the norm pass and finalize against float64
at ResNet-50 parameter shapes for bf16, fp16 and fp32 arenas, the multi-tensor path with mixed dtypes and two groups, the
overflow skip, bit-identity with and without clipping when nothing is clipped, eager against CUDA-graph runs, a max_norm
changed between replays, and the training entrypoints."""
import gc
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _fp64 as R  # noqa: E402

pytestmark = pytest.mark.gpu

DEV = "cuda"
F32, BF16, F16 = torch.float32, torch.bfloat16, torch.float16
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = R.U32
THREADS = 256


@pytest.fixture(autouse=True)
def _release_memory():
    yield
    gc.collect()
    if torch.cuda.is_available():
        torch.cuda.synchronize()
        torch.cuda.empty_cache()


def C():
    from pytorch_distributed_b200 import _ext
    return _ext.lib()


def _resnet50_numels():
    from pytorch_distributed_b200.models import create_model
    return [p.numel() for p in create_model("resnet50", num_classes=1000).parameters()]


def _flat_layout(numels, align=64):
    """Arena offsets with padding between tensors, and the chunk table FusedSGD._larc_table() builds for them."""
    chunk = C().LARC_CHUNK
    offs, off, info, chunk_tensor = [], 0, [], []
    for t, n in enumerate(numels):
        offs.append(off)
        info.append((off, n, len(chunk_tensor), t))
        chunk_tensor += [t] * R.cdiv(n, chunk)
        off = R.cdiv(off + n + 1, align) * align
    return offs, off, torch.tensor(chunk_tensor, dtype=torch.int32, device=DEV), torch.tensor(info, dtype=torch.int64, device=DEV)


def _depth(numels, nparts):
    """Longest chain of fp32 roundings in one partial sum of squares: the per-thread loop over a chunk, the CTA tree, the
    finalize's per-thread loop over the partials and its tree."""
    chunk = C().LARC_CHUNK
    return chunk // THREADS + 5 + 3 + R.cdiv(nparts, THREADS) + 5 + 3


def _norm_bound(total64, depth):
    """|total - ||g gmul||| for sums of non-negative squares: each square carries 2u, each addition u of the running sum,
    the square root halves the relative error and adds u."""
    return 1.01 * total64 * ((depth + 2) / 2 * U + U) + 1e-30


def _clip_ref(total, max_norm, gmul):
    """coef and the clipped slot 4, in the kernel's fp32 arithmetic (numpy float32 rounds to nearest like __fdiv_rn)."""
    t = np.float32(total)
    coef = np.float32(max_norm) / (t + np.float32(1e-6))
    coef = np.float32(1.0) if coef > 1 else coef
    return coef, np.float32(gmul) * coef


@pytest.mark.parametrize("gdt", [BF16, F16, F32])
def test_flat_norm_and_update_against_float64(gdt):
    numels = _resnet50_numels()
    offs, n, ct, info = _flat_layout(numels)
    gen = torch.Generator(device=DEV).manual_seed(0)
    grad = (torch.randn(n, device=DEV, generator=gen) * 64).to(gdt)
    pad = torch.ones(n, dtype=torch.bool, device=DEV)
    for o, k in zip(offs, numels):
        pad[o:o + k] = False
    grad[pad] = 1e3                                              # the alignment padding must stay out of the norm
    master = torch.randn(n, device=DEV, generator=gen)
    mom = torch.randn(n, device=DEV, generator=gen)
    gmul, max_norm = 1.0 / 1024, 1.0
    hyper = torch.tensor([0.1, 0.9, 1e-4, 0.0, gmul, 0.0, 0.0, 0.0, max_norm], device=DEV)
    clipped = torch.zeros_like(hyper)
    partials = torch.zeros(2 * ct.numel(), device=DEV)
    total, count = torch.zeros((), device=DEV), torch.zeros(1, dtype=torch.int32, device=DEV)
    C().grad_sumsq_flat(grad, ct, info, partials, hyper, None)
    C().clip_finalize(partials, ct.numel(), [hyper], [clipped], None, total, count)
    torch.cuda.synchronize()
    g64 = grad.double() * gmul
    t64 = g64[~pad].square().sum().sqrt().item()
    bound = _norm_bound(t64, _depth(numels, ct.numel()))
    assert abs(total.item() - t64) <= bound, (total.item(), t64, bound)
    with_pad = g64.square().sum().sqrt().item()
    assert abs(total.item() - with_pad) > bound, "negative control: a norm over the padding must break the bound"
    coef, slot4 = _clip_ref(total.item(), max_norm, np.float32(gmul))
    assert coef < 1 and int(count) == 1
    assert clipped[4].item() == float(slot4)
    assert torch.equal(clipped[:4], hyper[:4]) and torch.equal(clipped[5:], hyper[5:])
    m0, mo0 = master.clone(), mom.clone()
    C().fused_sgd_flat(grad, master, mom, None, clipped, None, False, False)
    ref = R.sgd_step_fp64(m0, mo0, grad, clipped.cpu().tolist(), nesterov=False, first=False)
    R.check_sgd("flat %s clipped" % gdt, master, mom, ref)
    # run to run: the same bits
    again = torch.zeros((), device=DEV)
    C().grad_sumsq_flat(grad, ct, info, partials, hyper, None)
    C().clip_finalize(partials, ct.numel(), [hyper], [clipped], None, again, count)
    R.assert_bits_equal("total, second run", again, total)


def test_multi_tensor_mixed_dtypes_two_groups_against_float64():
    from pytorch_distributed_b200.ops.fused_sgd import FusedSGD
    numels = _resnet50_numels()[:40]
    gen = torch.Generator(device=DEV).manual_seed(1)
    params = []
    for i, k in enumerate(numels):
        dt = (F32, BF16, F16)[i % 3]
        p = torch.nn.Parameter(torch.randn(k, device=DEV, generator=gen).to(dt))
        p.grad = (torch.randn(k, device=DEV, generator=gen) * 8).to(dt)
        params.append(p)
    groups = [{"params": params[:20]}, {"params": params[20:], "lr": 0.05, "weight_decay": 1e-3}]
    opt = FusedSGD(groups, lr=0.1, momentum=0.9, weight_decay=1e-4, clip_grad_norm=2.0)
    m0 = [p.detach().float().clone() for p in params]
    opt.step()
    torch.cuda.synchronize()
    t64 = torch.stack([p.grad.double().square().sum() for p in params]).sum().sqrt().item()
    nparts = sum(R.cdiv(k, C().LARC_CHUNK) for k in numels)
    total = opt.grad_norm().item()
    assert abs(total - t64) <= _norm_bound(t64, _depth(numels, nparts)), (total, t64)
    coef, slot4 = _clip_ref(total, 2.0, 1.0)
    assert coef < 1 and int(opt.clipped_steps()) == 1
    for gi, g in enumerate(groups):
        hyp = opt._clip_state.hyper[gi]
        assert hyp[4].item() == float(slot4)
        for p in g["params"]:
            i = next(j for j, q in enumerate(params) if q is p)
            master = p.detach() if p.dtype == F32 else opt.state[p]["master"]
            ref = R.sgd_step_fp64(m0[i], torch.zeros_like(m0[i]), p.grad, hyp.cpu().tolist(), nesterov=False, first=True)
            R.check_sgd("multi group %d %s" % (gi, p.dtype), master, opt.state[p]["momentum_buffer"], ref)


def test_overflow_changes_nothing():
    numels = _resnet50_numels()[:30]
    offs, n, ct, info = _flat_layout(numels)
    gen = torch.Generator(device=DEV).manual_seed(2)
    grad = torch.randn(n, device=DEV, generator=gen).to(BF16)
    master, mom, ema = (torch.randn(n, device=DEV, generator=gen) for _ in range(3))
    copy = master.to(BF16)
    hyper = torch.tensor([0.1, 0.9, 1e-4, 0.0, 1.0, 0.0, 0.5, 0.5, 0.01], device=DEV)
    clipped = torch.full_like(hyper, 7.0)
    partials = torch.zeros(2 * ct.numel(), device=DEV)
    total, count = torch.full((), 3.0, device=DEV), torch.full((1,), 5, dtype=torch.int32, device=DEV)
    found_inf = torch.ones(1, dtype=torch.int32, device=DEV)
    before = [t.clone() for t in (master, mom, ema, copy, clipped, total, count, partials)]
    C().grad_sumsq_flat(grad, ct, info, partials, hyper, found_inf)
    C().clip_finalize(partials, ct.numel(), [hyper], [clipped], found_inf, total, count)
    C().fused_sgd_flat(grad, master, mom, copy, clipped, found_inf, False, False, ema=ema)
    torch.cuda.synchronize()
    for name, a, b in zip(("master", "momentum", "ema", "copy", "clipped hyper", "total", "count", "partials"), before,
                          (master, mom, ema, copy, clipped, total, count, partials)):
        R.assert_bits_equal("after a skipped step: " + name, b, a)


# ------------------------------------------------------------------------------------------------ through the engine
def _paths(tmp_path, runs):
    out = tmp_path / "paths.pt"
    e = dict(os.environ, PYTHONPATH=ROOT)
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "MASTER_ADDR", "MASTER_PORT"):
        e.pop(k, None)
    p = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "clip_paths.py"), str(out), json.dumps(runs)], env=e,
                       cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-3000:] + "\n" + p.stderr[-3000:]
    return torch.load(out, weights_only=False)


def _same(tag, a, b):
    R.assert_bits_equal(tag + " master", a["master"], b["master"])
    R.assert_bits_equal(tag + " momentum", a["momentum"], b["momentum"])
    for k in a["live"]:
        R.assert_bits_equal("%s live %s" % (tag, k), a["live"][k], b["live"][k])


def test_coef_one_is_bit_identical_to_no_clipping(tmp_path):
    """max_norm = 1e30 never clips: eager and graph, overlap on and off, the same bits as the run without clipping."""
    big = ["--clip-grad-norm", "1e30"]
    cases = [([], False), (big, False), (big + ["--no-overlap-optimizer"], False), ([], True), (big, True),
             (big + ["--no-overlap-optimizer"], True)]
    got = _paths(tmp_path, [{"argv": a, "graph": g} for a, g in cases])
    for (argv, graph), r in zip(cases[1:], got[1:]):
        _same("%s graph=%s" % (argv, graph), got[0], r)
    assert got[1]["clipped"] == 0 and torch.isfinite(got[1]["grad_norm"])


def test_active_clipping_eager_graph_repeat_and_change(tmp_path):
    clip = ["--clip-grad-norm", "0.5"]
    runs = [{"argv": clip}, {"argv": clip}, {"argv": clip, "graph": True},
            {"argv": clip, "set_at": 2, "set_to": 0.05}, {"argv": clip, "graph": True, "set_at": 2, "set_to": 0.05}, {}]
    got = _paths(tmp_path, runs)
    _same("repeat", got[0], got[1])
    _same("graph", got[0], got[2])
    _same("max_norm changed between replays", got[3], got[4])
    R.assert_bits_equal("grad_norm graph", got[2]["grad_norm"], got[0]["grad_norm"])
    assert got[0]["clipped"] == 4 and got[2]["clipped"] == 4
    assert not torch.equal(got[0]["master"], got[5]["master"]) and not torch.equal(got[0]["master"], got[3]["master"])


# ------------------------------------------------------------------------------------------------ entrypoints
COMMON = ["-a", "resnet50", "-b", "32", "--synthetic", "--steps-per-epoch", "4", "--val-steps", "1", "--epochs", "1",
          "--image-size", "96", "-p", "1", "--clip-grad-norm", "1.0"]


@pytest.mark.parametrize("script,extra,port", [
    ("distributed.py", ["--cuda-graph"], 29831),
    ("distributed.py", ["--cuda-graph", "--larc", "--accum-steps", "2", "--model-ema"], 29832),
    ("distributed.py", ["--optimizer", "torch"], 29833),
    # a static loss scale: with the dynamic one the first steps of a short fp16 run overflow and are skipped, norm and all
    ("apex_distributed.py", ["--opt-level", "O2", "--precision", "fp16", "--loss-scale", "128"], 29834),
    ("horovod_distributed.py", ["--cuda-graph"], 29835),
    ("horovod_distributed.py", ["--optimizer", "torch"], 29836),
    ("dataparallel.py", [], None),
], ids=["ddp-graph", "ddp-larc-accum2-ema", "torch-sgd", "apex-o2-fp16", "horovod", "horovod-torch-sgd", "dataparallel"])
def test_entrypoint_clip_grad_norm(script, extra, port, tmp_path):
    e = dict(os.environ, PYTHONPATH=ROOT)
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "MASTER_ADDR", "MASTER_PORT"):
        e.pop(k, None)
    log = tmp_path / "log.jsonl"
    args = COMMON + extra + ["--checkpoint-dir", str(tmp_path), "--log-jsonl", str(log)]
    if port is None:
        cmd = [sys.executable, os.path.join(ROOT, script), "--gpus", "0"] + args
    else:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "1", "--master-addr", "127.0.0.1",
               "--master-port", str(port), os.path.join(ROOT, script)] + args
    p = subprocess.run(cmd, env=e, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-3000:] + "\n" + p.stderr[-3000:]
    rec = [json.loads(line) for line in open(log) if '"train"' in line][-1]
    assert rec["grad_norm"] is not None and np.isfinite(rec["grad_norm"]) and rec["grad_norm"] > 0, rec
    assert 0 <= rec["clipped_steps"] <= 4, rec
    ck = torch.load(tmp_path / "checkpoint.pth.tar", weights_only=False)
    assert all(torch.isfinite(v).all() for v in ck["state_dict"].values() if v.is_floating_point())
