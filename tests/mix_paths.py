"""Short ResNet-50 training runs on one GPU with MixUp / CutMix / label smoothing through DistributedDataParallel (world 1) and
FusedSGD, eager or under a CUDA graph, in a process of their own so that the communicator arenas and graph pools go away with
it.  Writes, per run and per step, the draw, the mixed batch and the step's (loss, acc1, acc5), then the flat fp32 masters (on
the CPU) to OUT.

    python tests/mix_paths.py OUT '[{"argv": ["--mixup-alpha", "0.2"], "graph": true}, ...]'
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


def train(argv, steps=6, graph=False):
    from pytorch_distributed_b200 import cli, driver
    from pytorch_distributed_b200.models import create_model
    torch.cuda.set_device(0)
    args = cli.parse_args("distributed", ["-a", "resnet50", "-b", "8", "--synthetic", "--image-size", "64", "--quiet", "--seed", "0"] + argv)
    st = driver.STRATEGIES["distributed"]()
    torch.manual_seed(0)
    model = create_model(args.arch, num_classes=args.num_classes, fused_bn=args.fused_bn)
    model, opt = st.build(model, args, torch.device(DEV, 0), 0)
    model.train()
    bm = st.batch_mix
    metrics = driver.MetricPipeline(st.comm, torch.device(DEV, 0), (driver.AverageMeter("l"), driver.AverageMeter("a"),
                                                                     driver.AverageMeter("b")))
    step = driver.TrainStep(st, model, torch.nn.CrossEntropyLoss().to(DEV), opt, metrics, use_graph=graph, warmup=1)
    rec = []
    for i in range(steps):
        x, y = _batch(st.input_dtype, seed=i)
        step(x, y)
        metrics.drain()
        torch.cuda.synchronize()
        rec.append({"draw": dict(bm.last), "mixed": bm._static[1].float().cpu(), "metrics": metrics.last,
                    "graph": step.graph is not None})
    assert opt.is_flat and (graph is False or step.graph is not None)
    return {"steps": rec, "master": opt._flat.master.cpu(), "graph": step.graph is not None}


def main():
    out, runs = sys.argv[1], json.loads(sys.argv[2])
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    torch.save([train(r.get("argv", []), graph=r.get("graph", False)) for r in runs], out)


if __name__ == "__main__":
    main()
