"""Shared command line for every entrypoint.

Flag surface = /root/reference/distributed.py:25-102 (the same block is copied
into all six reference scripts; ``--local_rank`` exists only in distributed.py:73
and apex_distributed.py:76, ``--dist-file`` only in distributed_slurm_main.py:102).
Reference-compatible defaults are kept; everything else is additive.

Deviations (SURVEY Q2/Q3): both ``--local_rank`` and ``--local-rank`` are accepted
and fall back to $LOCAL_RANK; ``-j/--workers`` is honoured.
"""
from __future__ import annotations

import argparse
import math
import os


def model_names():
    from .models import available_models
    return available_models()


def build_parser(entry: str = "distributed") -> argparse.ArgumentParser:
    p = argparse.ArgumentParser(description="H100-native ImageNet training (%s)" % entry)
    p.add_argument("--data", metavar="DIR", default=os.environ.get("IMAGENET_DIR", ""),
                   help="path to dataset (DIR/train, DIR/val ImageFolder trees); "
                        "empty or --synthetic => synthetic ImageNet-shaped data")
    p.add_argument("-a", "--arch", metavar="ARCH", default="resnet18", choices=model_names(),
                   help="model architecture (default: resnet18)")
    p.add_argument("-j", "--workers", default=4, type=int, metavar="N",
                   help="number of data loading workers (default: 4)")
    p.add_argument("--epochs", default=90, type=int, metavar="N", help="number of total epochs to run")
    p.add_argument("--start-epoch", default=0, type=int, metavar="N",
                   help="manual epoch number (useful on restarts)")
    p.add_argument("-b", "--batch-size", default=3200, type=int, metavar="N",
                   help="mini-batch size (default: 3200): total batch of all GPUs on the node")
    p.add_argument("--lr", "--learning-rate", default=0.1, type=float, metavar="LR",
                   help="initial learning rate", dest="lr")
    p.add_argument("--momentum", default=0.9, type=float, metavar="M", help="momentum")
    p.add_argument("--wd", "--weight-decay", default=1e-4, type=float, metavar="W",
                   help="weight decay (default: 1e-4)", dest="weight_decay")
    p.add_argument("-p", "--print-freq", default=10, type=int, metavar="N",
                   help="print frequency (default: 10)")
    p.add_argument("-e", "--evaluate", dest="evaluate", action="store_true",
                   help="evaluate model on validation set")
    p.add_argument("--pretrained", dest="pretrained", action="store_true", help="use pre-trained model")
    p.add_argument("--seed", default=None, type=int, help="seed for initializing training.")

    if entry in ("distributed", "apex_distributed"):
        p.add_argument("--local_rank", "--local-rank", default=-1, type=int, dest="local_rank",
                       help="local rank injected by the launcher (falls back to $LOCAL_RANK)")
    if entry == "distributed_slurm_main":
        p.add_argument("--dist-file", default=None, type=str, help="shared file for file:// rendezvous")
    if entry == "dataparallel":
        p.add_argument("--gpus", default=None, type=str,
                       help="comma separated device ids (default: all visible; the reference hard-codes 0,1,2,3)")
    if entry == "apex_distributed":
        p.add_argument("--opt-level", default="O1", choices=["O0", "O1", "O2", "O3"],
                       help="amp optimisation level (reference passes none => O1)")
        p.add_argument("--loss-scale", default="dynamic", help="'dynamic' or a float")
    if entry == "horovod_distributed":
        p.add_argument("--compression", default="fp16", choices=["none", "fp16", "bf16"],
                       help="wire compression for the DistributedOptimizer (reference: fp16)")

    # ---- additive, H100-native knobs (all have reference-compatible defaults) ----
    x = p.add_argument_group("b200")
    x.add_argument("--synthetic", action="store_true", help="force synthetic ImageNet-shaped data")
    x.add_argument("--synthetic-size", default=None, type=int, metavar="N",
                   help="images per synthetic epoch (default: 1,281,167 train / 50,000 val; "
                        "--steps-per-epoch overrides)")
    x.add_argument("--steps-per-epoch", default=None, type=int, help="cap iterations per epoch (tests/bench)")
    x.add_argument("--val-steps", default=None, type=int, help="cap validation iterations")
    x.add_argument("--image-size", default=224, type=int)
    x.add_argument("--num-classes", default=1000, type=int)
    x.add_argument("--comm", default="auto", choices=["auto", "fused", "nccl", "gloo"],
                   help="gradient data plane: fused = sm_90a peer-memory kernels, nccl/gloo = library all-reduce")
    x.add_argument("--wire-dtype", default="bf16", choices=["bf16", "fp16", "fp32"],
                   help="gradient wire format of the fused all-reduce")
    x.add_argument("--bucket-cap-mb", default=8.0, type=float,
                   help="gradient bucket size cap in MiB of wire data (torch's default is 25; NVSwitch has no per-link cost, "
                        "so smaller buckets only buy earlier overlap; first bucket 1 MiB, tail bucket 1 MiB)")
    x.add_argument("--precision", default=None, choices=["fp32", "bf16", "fp16"],
                   help="compute precision (default: bf16 on CUDA, fp32 on CPU)")
    x.add_argument("--channels-last", dest="channels_last", action="store_true", default=None)
    x.add_argument("--no-channels-last", dest="channels_last", action="store_false")
    x.add_argument("--fused-bn", dest="fused_bn", action="store_true", default=None,
                   help="use the hand-written NHWC BN(+add)+ReLU kernels in the ResNet family")
    x.add_argument("--no-fused-bn", dest="fused_bn", action="store_false")
    x.add_argument("--optimizer", default="fused", choices=["fused", "torch"],
                   help="fused = hand-written multi-tensor SGD kernel; torch = torch.optim.SGD")
    x.add_argument("--larc", action="store_true",
                   help="layer-wise adaptive rates (apex.parallel.LARC) around the optimizer; fused into the SGD kernels with "
                        "--optimizer fused")
    x.add_argument("--larc-trust-coefficient", default=None, type=_positive_float, metavar="T",
                   help="LARC trust coefficient (default: 0.02, apex's)")
    x.add_argument("--larc-clip", dest="larc_clip", action="store_true", default=None,
                   help="LARC clip mode: the adaptive factor is min(f / lr, 1) (default)")
    x.add_argument("--no-larc-clip", dest="larc_clip", action="store_false",
                   help="LARC scale mode: the gradient is multiplied by f itself")
    x.add_argument("--clip-grad-norm", default=None, type=_positive_float, metavar="MAX",
                   help="clip the unscaled, reduced gradient of every optimizer step to the global L2 norm MAX, as "
                        "torch.nn.utils.clip_grad_norm_ (torchvision's flag); fused into the SGD step with --optimizer fused "
                        "(default: off)")
    x.add_argument("--accum-steps", default=1, type=_positive_int, metavar="N",
                   help="gradient accumulation: one optimizer step per N consecutive batches (effective batch -b x N); the fused "
                        "engine sums the earlier passes in fp32 on each GPU and reduces once, in the last pass (default: 1)")
    x.add_argument("--model-ema", action="store_true",
                   help="keep an exponential moving average of the weights (fp32, updated inside the fused optimizer step), "
                        "validate it after each epoch and save it as state_dict_ema")
    x.add_argument("--model-ema-decay", default=None, type=float, metavar="D",
                   help="decay of --model-ema: e = D e + (1 - D) p after every optimizer step, 0 <= D < 1 (default: 0.9999)")
    x.add_argument("--label-smoothing", default=0.0, type=_unit_float, metavar="EPS",
                   help="cross-entropy against (1 - EPS) target + EPS / classes, 0 <= EPS <= 1 (torch's label_smoothing; "
                        "default: 0.0)")
    x.add_argument("--mixup-alpha", default=0.0, type=_alpha, metavar="A",
                   help="MixUp with lambda ~ Beta(A, A) on every training batch, as torchvision's transforms.v2.MixUp; one pass "
                        "of a fused kernel on the GPU (default: 0.0 = off)")
    x.add_argument("--cutmix-alpha", default=0.0, type=_alpha, metavar="A",
                   help="CutMix with lambda ~ Beta(A, A), as torchvision's transforms.v2.CutMix; with --mixup-alpha too, each "
                        "batch takes one of the two at random (default: 0.0 = off)")
    x.add_argument("--auto-augment", default=None, choices=["ta_wide", "imagenet", "cifar10", "svhn"],
                   help="per-sample augmentation of the training crops: ta_wide is torchvision's transforms.v2.TrivialAugmentWide, "
                        "imagenet, cifar10 and svhn are transforms.v2.AutoAugment with that policy (all bilinear); fused into "
                        "the normalising kernel on the GPU (default: none)")
    x.add_argument("--random-erase", default=0.0, type=_unit_float, metavar="P",
                   help="erase a random box of each training image with probability P, as torchvision's RandomErasing(P) after "
                        "the normalisation (default: 0.0)")
    x.add_argument("--cuda-graph", action="store_true", help="capture the train step in a CUDA graph")
    x.add_argument("--sync-bn", action="store_true",
                   help="synchronise BatchNorm statistics across the data-parallel ranks (torch.nn.SyncBatchNorm semantics; "
                        "fused into the BN kernels with --comm fused)")
    x.add_argument("--overlap-optimizer", dest="overlap_optimizer", action="store_true", default=True,
                   help="fused optimizer: update each gradient bucket right behind its all-reduce, inside backward (default)")
    x.add_argument("--no-overlap-optimizer", dest="overlap_optimizer", action="store_false")
    x.add_argument("--bucket-view", action="store_true",
                   help="DDP gradient_as_bucket_view: p.grad are views of the symmetric arena (no write-back / pack pass)")
    x.add_argument("--device", default=None, help="cuda|cpu (default: cuda if available)")
    x.add_argument("--dist-backend", default=None, help="control-plane backend (default nccl on CUDA, gloo on CPU)")
    x.add_argument("--dist-url", default=None, help="override rendezvous URL")
    x.add_argument("--world-size", default=None, type=int, help="processes to spawn (mp/hvd self-launch)")
    x.add_argument("--resume", default="", type=str, help="checkpoint to resume from (extension; SURVEY Q10)")
    x.add_argument("--checkpoint-dir", default=".", type=str)
    x.add_argument("--log-jsonl", default="", type=str, help="append machine-readable step records here")
    x.add_argument("--quiet", action="store_true")
    return p


def resolve_local_rank(args) -> int:
    lr = getattr(args, "local_rank", -1)
    if lr is None or lr < 0:
        lr = int(os.environ.get("LOCAL_RANK", "0"))
    args.local_rank = lr
    return lr


def _positive_int(s: str) -> int:
    v = int(s)
    if v < 1:
        raise argparse.ArgumentTypeError("must be an integer >= 1, got %r" % (s,))
    return v


def _positive_float(s: str) -> float:
    v = float(s)
    if not (v > 0 and math.isfinite(v)):
        raise argparse.ArgumentTypeError("must be a positive finite number, got %r" % (s,))
    return v


def _unit_float(s: str) -> float:
    v = float(s)
    if not 0.0 <= v <= 1.0:
        raise argparse.ArgumentTypeError("must lie in [0, 1], got %r" % (s,))
    return v


def _alpha(s: str) -> float:
    v = float(s)
    if not (v >= 0 and math.isfinite(v)):
        raise argparse.ArgumentTypeError("must be a finite number >= 0, got %r" % (s,))
    return v


def parse_args(entry: str, argv=None):
    parser = build_parser(entry)
    args = parser.parse_args(argv)
    if not args.larc and (args.larc_trust_coefficient is not None or args.larc_clip is not None):
        parser.error("--larc-trust-coefficient / --larc-clip / --no-larc-clip need --larc")
    if not args.model_ema and args.model_ema_decay is not None:
        parser.error("--model-ema-decay needs --model-ema")
    if args.model_ema_decay is not None and not (0.0 <= args.model_ema_decay < 1.0):
        parser.error("--model-ema-decay must lie in [0, 1), got %r" % (args.model_ema_decay,))
    if args.accum_steps > 1 and entry == "dataparallel":
        parser.error("--accum-steps needs one process per GPU; the single-process DataParallel entrypoint does not support it")
    if args.steps_per_epoch is not None and args.steps_per_epoch < args.accum_steps:
        parser.error("--steps-per-epoch %d is less than --accum-steps %d: an epoch would hold no optimizer step" %
                     (args.steps_per_epoch, args.accum_steps))
    if args.larc_trust_coefficient is None:
        args.larc_trust_coefficient = 0.02
    if args.larc_clip is None:
        args.larc_clip = True
    if args.model_ema_decay is None:
        args.model_ema_decay = 0.9999
    args.entry = entry
    return args
