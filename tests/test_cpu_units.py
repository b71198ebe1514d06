"""CPU unit tier (SURVEY section 4): CLI, meters, accuracy, LR schedule, checkpoint layout, plans/buckets, loss scaler,
fusion queue, FusedSGD reference path."""
import io
import math
import os
from contextlib import redirect_stdout

import numpy as np
import pytest
import torch

from pytorch_distributed_b200 import cli
from pytorch_distributed_b200.parallel import plan as P
from pytorch_distributed_b200.utils.meters import AverageMeter, ProgressMeter, accuracy, adjust_learning_rate, step_lr


# ------------------------------------------------------------------ CLI
def test_cli_defaults_match_reference():
    a = cli.parse_args("distributed", [])
    assert (a.arch, a.workers, a.epochs, a.start_epoch, a.batch_size) == ("resnet18", 4, 90, 0, 3200)
    assert (a.lr, a.momentum, a.weight_decay, a.print_freq) == (0.1, 0.9, 1e-4, 10)
    assert a.evaluate is False and a.pretrained is False and a.seed is None and a.local_rank == -1


@pytest.mark.parametrize("flag", ["--local_rank", "--local-rank"])
def test_cli_accepts_both_local_rank_spellings(flag):
    a = cli.parse_args("distributed", [flag + "=3"])
    assert a.local_rank == 3
    assert cli.resolve_local_rank(a) == 3


def test_cli_local_rank_env_fallback(monkeypatch):
    monkeypatch.setenv("LOCAL_RANK", "5")
    a = cli.parse_args("apex_distributed", [])
    assert cli.resolve_local_rank(a) == 5


def test_cli_entry_specific_flags():
    assert cli.parse_args("distributed_slurm_main", ["--dist-file", "f"]).dist_file == "f"
    assert cli.parse_args("dataparallel", ["--gpus", "0,1"]).gpus == "0,1"
    assert cli.parse_args("apex_distributed", []).opt_level == "O1"
    assert cli.parse_args("horovod_distributed", []).compression == "fp16"
    with pytest.raises(SystemExit):
        cli.parse_args("multiprocessing_distributed", ["--local_rank", "1"])   # reference: only 2 scripts take it


def test_cli_arch_choices_cover_torchvision_and_native():
    names = cli.model_names()
    for n in ("resnet18", "resnet50", "vgg16", "mobilenet_v2", "wide_resnet50_2"):
        assert n in names
    with pytest.raises(SystemExit):
        cli.parse_args("distributed", ["-a", "not_a_model"])


def test_cli_aliases():
    a = cli.parse_args("distributed", ["--learning-rate", "0.5", "--weight-decay", "0.01", "-b", "64", "-j", "7", "-p", "3", "-e"])
    assert (a.lr, a.weight_decay, a.batch_size, a.workers, a.print_freq, a.evaluate) == (0.5, 0.01, 64, 7, 3, True)


# ------------------------------------------------------------------ meters
def test_average_meter_format_and_math():
    m = AverageMeter("Loss", ":.4e")
    m.update(2.0, 4)
    m.update(4.0, 4)
    assert m.avg == 3.0 and m.val == 4.0 and m.count == 8
    assert str(m) == "Loss 4.0000e+00 (3.0000e+00)"
    t = AverageMeter("Time", ":6.3f")
    t.update(0.25)
    assert str(t) == "Time  0.250 ( 0.250)"


def test_progress_meter_line_format():
    a, b = AverageMeter("Time", ":6.3f"), AverageMeter("Acc@1", ":6.2f")
    a.update(1.5)
    b.update(12.5)
    p = ProgressMeter(5005, [a, b], prefix="Epoch: [3]")
    assert p.line(7) == "Epoch: [3][   7/5005]\tTime  1.500 ( 1.500)\tAcc@1  12.50 ( 12.50)"
    buf = io.StringIO()
    with redirect_stdout(buf):
        ProgressMeter(10, [a], prefix="Test: ").display(3)
    assert buf.getvalue() == "Test: [ 3/10]\tTime  1.500 ( 1.500)\n"


def test_accuracy_matches_numpy_oracle():
    rng = np.random.default_rng(0)
    out = rng.standard_normal((64, 50)).astype(np.float32)
    tgt = rng.integers(0, 50, 64)
    order = np.argsort(-out, axis=1)
    exp1 = 100.0 * np.mean(order[:, 0] == tgt)
    exp5 = 100.0 * np.mean([(t in o[:5]) for o, t in zip(order, tgt)])
    a1, a5 = accuracy(torch.from_numpy(out), torch.from_numpy(tgt), topk=(1, 5))
    assert a1.shape == (1,) and abs(a1.item() - exp1) < 1e-4 and abs(a5.item() - exp5) < 1e-4


def test_accuracy_k5_does_not_crash_like_reference_q1():
    out = torch.randn(8, 10)
    a1, a5 = accuracy(out, torch.randint(0, 10, (8,)), topk=(1, 5))
    assert 0 <= a1.item() <= a5.item() <= 100


def test_lr_schedule():
    class A:
        lr = 0.1
    opt = torch.optim.SGD([torch.nn.Parameter(torch.zeros(1))], lr=0.1)
    for epoch, want in ((0, 0.1), (29, 0.1), (30, 0.01), (59, 0.01), (60, 0.001), (89, 0.001)):
        assert math.isclose(adjust_learning_rate(opt, epoch, A), want, rel_tol=1e-9)
        assert math.isclose(opt.param_groups[0]["lr"], want, rel_tol=1e-9)
    assert math.isclose(step_lr(1.0, 95), 1e-3)


# ------------------------------------------------------------------ checkpoint
def test_checkpoint_layout_and_best_copy(tmp_path):
    from pytorch_distributed_b200.models import create_model
    from pytorch_distributed_b200.utils.checkpoint import export_state_dict, load_checkpoint, save_checkpoint
    m = create_model("resnet18", num_classes=7)
    sd = export_state_dict(m)
    state = {"epoch": 3, "arch": "resnet18", "state_dict": sd, "best_acc1": 12.5}
    save_checkpoint(state, False, directory=str(tmp_path))
    assert os.path.exists(tmp_path / "checkpoint.pth.tar") and not os.path.exists(tmp_path / "model_best.pth.tar")
    save_checkpoint(state, True, directory=str(tmp_path))
    assert os.path.exists(tmp_path / "model_best.pth.tar")
    ck = torch.load(tmp_path / "checkpoint.pth.tar", weights_only=False)
    assert set(ck) >= {"epoch", "arch", "state_dict", "best_acc1"}
    # torchvision-compatible keys
    import torchvision
    tv = torchvision.models.resnet18(num_classes=7)
    assert list(ck["state_dict"].keys()) == list(tv.state_dict().keys())
    tv.load_state_dict(ck["state_dict"])
    m2 = create_model("resnet18", num_classes=7)
    load_checkpoint(str(tmp_path / "checkpoint.pth.tar"), m2)
    for a, b in zip(m.state_dict().values(), m2.state_dict().values()):
        assert torch.equal(a, b)


def test_native_resnet50_matches_torchvision_forward():
    import torchvision
    from pytorch_distributed_b200.models import create_model
    torch.manual_seed(0)
    ours = create_model("resnet50", num_classes=11, fused_bn=False).eval()
    tv = torchvision.models.resnet50(num_classes=11).eval()
    tv.load_state_dict(ours.state_dict())
    x = torch.randn(2, 3, 64, 64)
    with torch.no_grad():
        torch.testing.assert_close(ours(x), tv(x), rtol=1e-4, atol=1e-4)
    assert sum(p.numel() for p in create_model("resnet50").parameters()) == 25557032


# ------------------------------------------------------------------ plans / buckets
def test_tensor_layout_alignment():
    offs, total = P.tensor_layout([5, 64, 65, 1])
    assert offs == [0, 64, 128, 256] and total == 320
    assert all(o % P.ALIGN_ELEMS == 0 for o in offs)


@pytest.mark.parametrize("world", [1, 2, 8])
@pytest.mark.parametrize("grid", [1, 3, 32])
def test_build_layout_segments_cover_every_element_once(world, grid):
    rng = np.random.default_rng(1)
    numels = [int(n) for n in rng.integers(1, 5000, 37)] + [1, 64, 100000]
    lay = P.build_layout(numels, world, grid)
    assert lay.block_elems % (world * 8) == 0 and lay.region_elems >= lay.total
    seen = [np.zeros(n, dtype=np.int32) for n in numels]
    for b in range(grid):
        lo, hi = b * lay.block_elems, (b + 1) * lay.block_elems
        for s in lay.segs[lay.seg_begin[b]:lay.seg_begin[b + 1]]:
            t, ln, so, ao = int(s["tensor"]), int(s["len"]), int(s["src_off"]), int(s["arena_off"])
            assert lo <= ao and ao + ln <= hi                       # stays inside its CTA range
            assert ao == lay.offsets[t] + so                        # consistent mapping
            assert so % 8 == 0 or so == 0                           # 16-byte aligned starts inside tensors
            seen[t][so:so + ln] += 1
    assert all((s == 1).all() for s in seen)


def test_compute_buckets_caps_and_order():
    numels = [10, 10, 300000, 300000, 300000, 5]
    b = P.compute_buckets(numels, 4, cap_bytes=2 * 300000 * 4, first_cap_bytes=100)
    assert b[0] == [0, 1] and sum(len(x) for x in b) == 6 and [i for x in b for i in x] == list(range(6))
    many = P.compute_buckets([1] * 1000, 4, 1 << 30, None, max_tensors=256)
    assert max(len(x) for x in many) == 256


def test_resnet50_bucket_count_is_reasonable():
    from pytorch_distributed_b200.models import create_model
    ns = [p.numel() for p in create_model("resnet50").parameters()][::-1]
    b = P.compute_buckets(ns, 2, 25 << 20, 1 << 20)
    assert 2 <= len(b) <= 6 and sum(len(x) for x in b) == 161


# ------------------------------------------------------------------ loss scaler (host path)
def test_loss_scaler_state_machine_cpu():
    from pytorch_distributed_b200.parallel.amp import LossScaler
    s = LossScaler("cpu", "dynamic", init_scale=1024.0, growth_interval=3)
    for _ in range(3):
        s.update()
    assert s.loss_scale() == 2048.0
    s.found_inf.fill_(1)
    s.update()
    assert s.loss_scale() == 1024.0 and not s.host_found_inf()
    st = s.state_dict()
    s2 = LossScaler("cpu", "dynamic")
    s2.load_state_dict(st)
    assert s2.loss_scale() == 1024.0
    fixed = LossScaler("cpu", 128.0)
    fixed.found_inf.fill_(1)
    fixed.update()
    assert fixed.loss_scale() == 128.0


def test_amp_scale_loss_skips_step_on_overflow_cpu():
    from pytorch_distributed_b200.ops.fused_sgd import FusedSGD
    from pytorch_distributed_b200.parallel import amp
    m = torch.nn.Linear(4, 2)
    opt = FusedSGD(m.parameters(), lr=0.1)
    m, opt = amp.initialize(m, opt, opt_level="O1", half_dtype=torch.float16, loss_scale="dynamic", verbosity=0)
    amp._amp_state.scaler.scale.fill_(4.0)
    w0 = m.weight.detach().clone()
    loss = m(torch.ones(1, 4)).sum() * float("inf")
    with amp.scale_loss(loss, opt) as sl:
        sl.backward()
    opt.step()
    assert torch.equal(m.weight, w0)                               # skipped
    assert amp._amp_state.scaler.loss_scale() == 2.0               # halved
    opt.zero_grad()
    loss = m(torch.ones(1, 4)).sum()
    with amp.scale_loss(loss, opt) as sl:
        sl.backward()
    opt.step()
    torch.testing.assert_close(m.weight, w0 - 0.1 * torch.ones_like(w0))   # unscaled correctly (grad == 1)
    amp._amp_state.enabled = False
    amp._amp_state.scaler = None


# ------------------------------------------------------------------ FusedSGD reference path == torch SGD
@pytest.mark.parametrize("nesterov", [False, True])
def test_fused_sgd_cpu_matches_torch(nesterov):
    from pytorch_distributed_b200.ops.fused_sgd import FusedSGD
    torch.manual_seed(0)
    a = [torch.nn.Parameter(torch.randn(5, 3)), torch.nn.Parameter(torch.randn(7))]
    b = [torch.nn.Parameter(p.detach().clone()) for p in a]
    oa = FusedSGD(a, lr=0.1, momentum=0.9, weight_decay=1e-2, nesterov=nesterov)
    ob = torch.optim.SGD(b, lr=0.1, momentum=0.9, weight_decay=1e-2, nesterov=nesterov)
    for _ in range(4):
        for p, q in zip(a, b):
            g = torch.randn_like(p)
            p.grad, q.grad = g.clone(), g.clone()
        oa.step()
        ob.step()
    for p, q in zip(a, b):
        torch.testing.assert_close(p.data, q.data)


# ------------------------------------------------------------------ horovod-style fusion queue (C++)
def test_fusion_queue_grouping_and_order():
    from pytorch_distributed_b200 import _ext
    if not _ext.available():
        pytest.skip("native extension not built")
    q = _ext.lib().FusionQueue(1000, 1.0)
    hs = [q.enqueue("t%d" % i, 400, i) for i in range(5)]      # 400+400 -> 3rd would overflow 1000 => closes [0,1]
    g1 = q.next_group(50.0)
    g2 = q.next_group(50.0)
    assert g1 == hs[:2] and g2 == hs[2:4]
    assert q.next_group(5.0) == []                               # t4 still open
    q.flush()
    assert q.next_group(50.0) == hs[4:]
    assert q.pending() == 5
    q.mark_done(hs)
    assert q.pending() == 0 and all(q.wait(h, 10.0) for h in hs)
    big = q.enqueue("big", 5000, 9)                              # a single tensor above the threshold is its own group
    assert q.next_group(50.0) == [big]
    st = q.stats()
    assert st["groups"] == 4 and st["tensors"] == 6
    q.shutdown()


def test_launch_helpers(monkeypatch):
    from pytorch_distributed_b200 import launch
    p = launch.pick_port(23456)
    assert launch.port_is_free(p)
    monkeypatch.setenv("SLURM_PROCID", "1")
    monkeypatch.setenv("SLURM_NPROCS", "2")
    monkeypatch.setenv("SLURM_JOBID", "42")
    a = cli.parse_args("distributed_slurm_main", ["--dist-file", "/tmp/df"])
    node, nodes, world, url = launch.slurm_topology(a, 4)
    assert (node, nodes, world) == (1, 2, 8) and url == "file:///tmp/df.42"
    monkeypatch.setenv("RANK", "3")
    monkeypatch.setenv("WORLD_SIZE", "4")
    monkeypatch.setenv("LOCAL_RANK", "3")
    assert launch.torchrun_env() == (3, 3, 4)


def test_compute_buckets_tail_bucket_is_split_off():
    """The last bucket is the only exposed one: the trailing tensors (up to the tail cap) get their own small bucket."""
    from pytorch_distributed_b200.parallel import plan as P
    numels = [1000, 2_000_000, 3_000_000, 4_000_000, 100_000, 50_000, 30_000, 9_000]
    plain = P.compute_buckets(numels, 2, 8 << 20, 1 << 20, 256)
    tail = P.compute_buckets(numels, 2, 8 << 20, 1 << 20, 256, tail_cap_bytes=256 << 10)
    flat = lambda bs: [i for b in bs for i in b]          # noqa: E731
    assert flat(plain) == flat(tail) == list(range(len(numels)))              # order preserved, nothing lost
    assert tail[-1] == [5, 6, 7]                                              # 100 + 60 + 18 KB fit in 256 KiB, the next 200 KB do not
    assert sum(numels[i] for i in tail[-1]) * 2 <= (256 << 10) and len(tail) >= len(plain)
    assert P.compute_buckets([10, 20], 4, 1 << 20, None, 256, tail_cap_bytes=4) == [[0, 1]]      # nothing fits the cap: unchanged
    # every bucket respects the tensor limit
    many = P.compute_buckets([8] * 1000, 2, 1 << 30, None, 256, tail_cap_bytes=1 << 10)
    assert all(len(b) <= 256 for b in many) and flat(many) == list(range(1000))


def test_choose_grid_granularity():
    from pytorch_distributed_b200.parallel import plan as P
    assert P.choose_grid(1 << 20, 2, 32) == 8                       # 2 MiB at 256 KiB per CTA
    assert P.choose_grid(1 << 20, 2, 32, 32 << 10) == 32            # tail bucket: 32 KiB per CTA, capped by max_ctas
    assert P.choose_grid(100, 2, 32, 16 << 10) == 1
    lay = P.build_layout([1000, 3000, 77], world=8, grid=P.choose_grid(4096 + 64, 2, 32, 1 << 10))
    assert lay.block_elems % (8 * 8) == 0 and lay.region_elems >= 1000 + 3000 + 77


def test_reference_install_manifest(tmp_path, monkeypatch):
    """oracle/install_reference.py: the copy is verified against the sha256 manifest; a tampered file is reported."""
    import hashlib
    import shutil
    from oracle import install_reference as inst
    src = tmp_path / "reference"                      # a stand-in reference tree with its own manifest
    src.mkdir()
    manifest = {}
    for fn in ("distributed.py", "start.sh"):
        data = ("# %s\n" % fn).encode()
        (src / fn).write_bytes(data)
        manifest[fn] = hashlib.sha256(data).hexdigest()
    monkeypatch.setattr(inst, "MANIFEST", manifest)
    monkeypatch.setattr(inst, "REF_DIR", str(tmp_path / "_ref"))
    monkeypatch.setattr(inst, "DEFAULT_DIRS", [str(tmp_path / "absent")])
    monkeypatch.delenv(inst.ENV, raising=False)
    assert inst.install(force=True).startswith("NOT INSTALLED")
    monkeypatch.setattr(inst, "DEFAULT_DIRS", [str(src)])             # found at the default location ...
    assert inst.install(force=True).startswith("installed") and inst.verify() == []
    monkeypatch.setattr(inst, "DEFAULT_DIRS", [str(tmp_path / "absent")])
    monkeypatch.setenv(inst.ENV, str(src))
    msg = inst.install(force=True)
    assert "installed" in msg and inst.verify(str(tmp_path / "_ref")) == []
    with open(tmp_path / "_ref" / "distributed.py", "a") as f:
        f.write("# tampered\n")
    assert inst.verify(str(tmp_path / "_ref")) == ["distributed.py"]
    shutil.rmtree(tmp_path / "_ref")
    assert len(inst.verify(str(tmp_path / "_ref"))) == len(inst.MANIFEST)


def test_timeline_summary_tool_on_a_synthetic_trace(tmp_path):
    """tools/timeline_summary.py: step delimiting by the metric kernel, exposed-tail computation, kernel table."""
    import json
    import subprocess
    import sys
    evs = []
    t = 0.0
    for step in range(3):
        evs.append({"ph": "X", "cat": "kernel", "name": "void ptd::metrics_kernel<bf16>(x)", "ts": t, "dur": 20.0, "args": {"stream": 9, "grid": [1, 1, 1]}})
        for k in range(5):
            evs.append({"ph": "X", "cat": "kernel", "name": "cudnn_wgrad_kernel_%d" % k, "ts": t + 30 + k * 100, "dur": 90.0, "args": {"stream": 7, "grid": [100, 1, 1]}})
        evs.append({"ph": "X", "cat": "kernel", "name": "void ptd::fused_allreduce_kernel<bf16, true>(x)", "ts": t + 300, "dur": 50.0, "args": {"stream": 9, "grid": [32, 1, 1]}})
        # the tail bucket starts after the last backward kernel ended (t + 520): 25 us of exposed communication + optimizer
        evs.append({"ph": "X", "cat": "kernel", "name": "void ptd::fused_allreduce_kernel<bf16, true>(x)", "ts": t + 522, "dur": 18.0, "args": {"stream": 9, "grid": [29, 1, 1]}})
        evs.append({"ph": "X", "cat": "kernel", "name": "void ptd::fused_sgd_flat_kernel<bf16>(x)", "ts": t + 540, "dur": 5.0, "args": {"stream": 9, "grid": [200, 1, 1]}})
        evs.append({"ph": "X", "cat": "kernel", "name": "forward_kernel", "ts": t + 550, "dur": 400.0, "args": {"stream": 7, "grid": [100, 1, 1]}})
        t += 1000.0
    path = tmp_path / "tl.json"
    path.write_text(json.dumps({"traceEvents": evs}))
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, os.path.join(root, "tools", "timeline_summary.py"), str(path), "--top", "5"], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    assert "last complete step (metric kernel to metric kernel): 1.000 ms" in out.stdout
    assert "exposed tail): 25.0 us" in out.stdout
    assert "fused_allreduce_kernel" in out.stdout and "(nothing: exposed)" in out.stdout
