"""Short ResNet-50 training runs on one GPU through DistributedDataParallel (world 1) and FusedSGD with gradient clipping, in a
process of their own so that the communicator arenas and CUDA-graph pools they hold go away with it.  Writes, per run, the
flat fp32 masters and momentum, the live model's state dict (on the CPU), grad_norm() and clipped_steps() to OUT.

    python tests/clip_paths.py OUT '[{"argv": ["--clip-grad-norm", "0.5"], "graph": true, "set_at": 2, "set_to": 0.1}, ...]'
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

DEV = "cuda"


def _batch(dtype, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(8, 3, 64, 64, device=DEV, generator=g).to(dtype).contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 1000, (8,), device=DEV, generator=g)
    return x, y


def train(argv, steps=4, graph=False, set_at=None, set_to=None):
    """``steps`` steps; ``set_at``: call set_clip_grad_norm(set_to) before that step."""
    from pytorch_distributed_b200 import cli, driver
    from pytorch_distributed_b200.models import create_model
    torch.cuda.set_device(0)
    args = cli.parse_args("distributed", ["-a", "resnet50", "-b", "8", "--synthetic", "--image-size", "64", "--quiet"] + argv)
    st = driver.STRATEGIES["distributed"]()
    torch.manual_seed(0)
    model = create_model(args.arch, num_classes=args.num_classes, fused_bn=args.fused_bn)
    model, opt = st.build(model, args, torch.device(DEV, 0), 0)
    model.train()
    metrics = driver.MetricPipeline(st.comm, torch.device(DEV, 0), (driver.AverageMeter("l"), driver.AverageMeter("a"),
                                                                     driver.AverageMeter("b")))
    step = driver.TrainStep(st, model, torch.nn.CrossEntropyLoss().to(DEV), opt, metrics, use_graph=graph, warmup=1)
    for i in range(steps):
        if set_at is not None and i == set_at:
            opt.set_clip_grad_norm(set_to)
        x, y = _batch(st.input_dtype, seed=i)
        step(x, y)
        torch.cuda.synchronize()
    metrics.drain()
    assert opt.is_flat and (graph is False or step.graph is not None)
    gn, cnt = opt.grad_norm(), opt.clipped_steps()
    return {"master": opt._flat.master.cpu(), "momentum": opt._flat.momentum.cpu(),
            "live": {k: v.detach().float().cpu() for k, v in model.module.state_dict().items()},
            "grad_norm": None if gn is None else gn.cpu(), "clipped": None if cnt is None else int(cnt)}


def main():
    out, runs = sys.argv[1], json.loads(sys.argv[2])
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    torch.save([train(r.get("argv", []), graph=r.get("graph", False), set_at=r.get("set_at"), set_to=r.get("set_to"))
                for r in runs], out)


if __name__ == "__main__":
    main()
