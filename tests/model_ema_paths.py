"""Short ResNet-50 training runs on one GPU through DistributedDataParallel (world 1), FusedSGD and a ModelEma, in a process
of their own so that the communicator arenas, CUDA-graph pools and cached blocks they hold go away with it.  Writes, per
run, the flat fp32 masters, ``ModelEma.state_dict()`` and the live model's state dict (fp32, on the CPU) to OUT.

    python tests/model_ema_paths.py OUT '[{"argv": ["--larc"], "graph": true, "decay_at": 2, "eval_at": null}, ...]'
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


def train(argv, steps=4, graph=False, decay_at=None, eval_at=None):
    """``steps`` steps; ``decay_at``: set the decay to 0.5 before that step; ``eval_at``: evaluate the EMA copy before it."""
    from pytorch_distributed_b200 import cli, driver
    from pytorch_distributed_b200.models import create_model
    from pytorch_distributed_b200.utils.ema import ModelEma
    torch.cuda.set_device(0)
    args = cli.parse_args("distributed", ["-a", "resnet50", "-b", "8", "--synthetic", "--image-size", "64", "--quiet"] + argv)
    st = driver.STRATEGIES["distributed"]()
    torch.manual_seed(0)
    model = create_model(args.arch, num_classes=args.num_classes, fused_bn=args.fused_bn)
    model, opt = st.build(model, args, torch.device(DEV, 0), 0)
    model.train()
    ema = ModelEma(model, decay=0.9, optimizer=opt)
    metrics = driver.MetricPipeline(st.comm, torch.device(DEV, 0), (driver.AverageMeter("l"), driver.AverageMeter("a"),
                                                                     driver.AverageMeter("b")))
    step = driver.TrainStep(st, model, torch.nn.CrossEntropyLoss().to(DEV), opt, metrics, use_graph=graph, warmup=1, ema=ema)
    for i in range(steps):
        if decay_at is not None and i == decay_at:
            ema.decay = 0.5
        if eval_at is not None and i == eval_at:
            ema.sync_module()
            with torch.no_grad():
                ema.module(_batch(st.input_dtype, seed=100)[0])
        x, y = _batch(st.input_dtype, seed=i)
        step(x, y)
        torch.cuda.synchronize()
    metrics.drain()
    assert opt.is_flat and (graph is False or step.graph is not None)
    return {"master": opt._flat.master.cpu(),
            "ema": {k: v.detach().float().cpu() for k, v in ema.state_dict().items()},
            "live": {k: v.detach().float().cpu() for k, v in model.module.state_dict().items()}}


def main():
    out, runs = sys.argv[1], json.loads(sys.argv[2])
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    torch.save([train(r.get("argv", []), graph=r.get("graph", False), decay_at=r.get("decay_at"), eval_at=r.get("eval_at"))
                for r in runs], out)


if __name__ == "__main__":
    main()
