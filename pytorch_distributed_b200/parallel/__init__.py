"""Parallel engines: DDP (multi-process), DataParallel (single process), apex-style amp, horovod-style optimizer."""
from .ddp import DistributedDataParallel, GradientEngine  # noqa: F401
from .comm import make_communicator, FusedCommunicator, TorchCommunicator  # noqa: F401
from ..models.resnet import SyncBNAct as SyncBatchNorm  # noqa: F401  (torch.nn.SyncBatchNorm, convert_sync_batchnorm classmethod)
