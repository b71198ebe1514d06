"""Multi-GPU checks of synchronised BatchNorm, launched by tests/test_gpu_multi_sync_bn.py (or by hand) under torchrun;
every rank must print PASS.

    python -m torch.distributed.run --nproc-per-node 8 --master-addr 127.0.0.1 tests/mp_sync_bn_checks.py

1. ResNet-50 (fp32, channels_last, per-rank batches that differ) converted with ``convert_sync_batchnorm`` under this
   package's DDP on the fused communicator, against torchvision's ResNet-50 converted with
   ``torch.nn.SyncBatchNorm.convert_sync_batchnorm`` under torch DDP, from the same weights and data, one training
   forward + backward: the loss, the running statistics and the DDP-averaged gradients within the tolerances stated below
   (TF32 off).
2. The synchronised running statistics are bitwise equal on every rank.
3. Five bf16 training steps of ``driver.TrainStep`` with the step captured in a CUDA graph after two eager ones (as
   ``--cuda-graph`` runs it) leave the same parameters and running statistics, bit for bit, as five eager steps: the
   exchange kernels replay with their device call counters.
"""
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# Stated tolerances.  The fused fp32 BatchNorm kernels already differ from torch's BatchNorm on ONE rank (random-init
# ResNet-50, 128 x 128, this batch; same numbers before synchronised BatchNorm existed): weight gradients by up to ~14 %
# of their largest magnitude in layer3 / layer4 (one-pass E[x^2] - E[x]^2 in fp32 against torch's Welford, amplified
# through ~50 BatchNorm backwards), while the loss agrees to 1e-5.  Synchronisation must not add to that.
TOL = 2e-3          # loss
STAT_TOL = 2e-3     # running statistics (1.5e-5 on one rank)
GRAD_TOL = 0.25     # DDP-averaged weight gradients, of the largest magnitude per tensor
GRAD_COS = 0.995    # ... and their direction (0.9998 on one rank)


def rel(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-12)).item()


def same_on_all_ranks(t):
    got = [torch.empty_like(t) for _ in range(dist.get_world_size())]
    dist.all_gather(got, t.contiguous())
    return all(torch.equal(g, got[0]) for g in got)


def main():
    rank, local, world = int(os.environ["RANK"]), int(os.environ["LOCAL_RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    import torchvision
    from pytorch_distributed_b200.models import create_model
    from pytorch_distributed_b200.models.resnet import SyncBNAct, convert_sync_batchnorm
    from pytorch_distributed_b200.parallel.ddp import DistributedDataParallel
    cl = torch.channels_last

    # ---- 1 / 2: parity with torch DDP + nn.SyncBatchNorm
    torch.manual_seed(0)
    ours = convert_sync_batchnorm(create_model("resnet50", num_classes=10)).to(dev).to(memory_format=cl)
    ref = torchvision.models.resnet50(num_classes=10)
    ref.load_state_dict(ours.state_dict())
    ref = torch.nn.SyncBatchNorm.convert_sync_batchnorm(ref).to(dev).to(memory_format=cl)
    ddp = DistributedDataParallel(ours, device_ids=[local], comm="fused", wire_dtype="fp32")
    tddp = torch.nn.parallel.DistributedDataParallel(ref, device_ids=[local])
    g = torch.Generator(device=dev).manual_seed(100 + rank)
    batch = 16 + (rank % 3)                                 # per-rank batches differ
    x = torch.randn(batch, 3, 128, 128, device=dev, generator=g).contiguous(memory_format=cl)
    t = torch.randint(0, 10, (batch,), device=dev, generator=g)
    losses = []
    for m in (ddp, tddp):
        loss = torch.nn.functional.cross_entropy(m(x).float(), t)
        loss.backward()
        losses.append(loss.detach())
    torch.cuda.synchronize()
    ref_p, ref_sd = dict(ref.named_parameters()), ref.state_dict()
    worst = {"loss": rel(losses[0], losses[1]), "grad_rel": 0.0, "grad_cos": 1.0, "stat_rel": 0.0}
    for k, p in ours.named_parameters():                   # the DDP-averaged gradients
        a, b = p.grad.double().flatten(), ref_p[k].grad.double().flatten()
        worst["grad_rel"] = max(worst["grad_rel"], rel(a, b))
        worst["grad_cos"] = min(worst["grad_cos"], (a @ b / (a.norm() * b.norm()).clamp_min(1e-300)).item())
    for k, v in ours.state_dict().items():
        if v.is_floating_point() and ("running" in k):
            worst["stat_rel"] = max(worst["stat_rel"], rel(v, ref_sd[k]))
    print("[rank %d] vs torch DDP + SyncBatchNorm: %s" % (rank, worst), flush=True)
    assert worst["loss"] < TOL and worst["stat_rel"] < STAT_TOL, worst
    assert worst["grad_rel"] < GRAD_TOL and worst["grad_cos"] > GRAD_COS, worst
    for name, m in ours.named_modules():
        if isinstance(m, SyncBNAct):
            if world > 1:
                assert m._sync is not None and m._sync.native is not None, name + " did not bind to the fused communicator"
            stats = torch.cat([m.running_mean, m.running_var, m.num_batches_tracked.view(1).double().float()])
            assert same_on_all_ranks(stats), name + ": running statistics differ across ranks"

    # ---- 3: the training step captured in a CUDA graph (driver.TrainStep, as --cuda-graph runs it) equals the eager step
    from pytorch_distributed_b200 import cli, driver
    from pytorch_distributed_b200.utils.meters import AverageMeter
    finals = []
    for use_graph in (False, True):
        args = cli.parse_args("distributed", ["-a", "resnet50", "-b", str(8 * world), "--synthetic", "--quiet", "--sync-bn",
                                              "--num-classes", "10"] + (["--cuda-graph"] if use_graph else []))
        st = driver.Strategy()
        torch.manual_seed(1)
        model = driver.apply_sync_bn(create_model("resnet50", num_classes=10), args, st, dev)
        model, opt = st.build(model, args, dev, local)
        metrics = driver.MetricPipeline(st.comm, dev, (AverageMeter("Loss"), AverageMeter("Acc@1"), AverageMeter("Acc@5")))
        step = driver.TrainStep(st, model, torch.nn.CrossEntropyLoss().to(dev), opt, metrics, use_graph=use_graph, warmup=2)
        gs = torch.Generator(device=dev).manual_seed(7 + rank)
        for _ in range(5):
            x = torch.randn(8, 3, 128, 128, device=dev, generator=gs).to(st.input_dtype).contiguous(memory_format=cl)
            step(x, torch.randint(0, 10, (8,), device=dev, generator=gs))
        metrics.drain()
        torch.cuda.synchronize()
        assert (step.graph is not None) == use_graph
        finals.append([t.detach().clone() for t in list(st.unwrapped(model).parameters()) + list(st.unwrapped(model).buffers())])
    assert all(torch.equal(a, b) for a, b in zip(*finals)), "the graph-replayed steps differ from the eager steps"
    dist.barrier()
    print("PASS rank %d (world %d)" % (rank, world), flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
