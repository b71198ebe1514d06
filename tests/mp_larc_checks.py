"""One rank of an entrypoint's training loop (as distributed.py / apex_distributed.py / horovod_distributed.py run it, launched
by torch.distributed.run) that, at the end, writes what this rank's optimizer holds to OUT/rank<r>.pt: the fp32 masters,
the momentum buffers and ``larc_stats()``.  Tests compare the files of all ranks bit for bit.

    python -m torch.distributed.run --nproc-per-node 2 tests/mp_larc_checks.py OUT ENTRY <driver flags>
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from pytorch_distributed_b200 import cli, driver, launch  # noqa: E402
from pytorch_distributed_b200.parallel import amp as _amp  # noqa: E402


def main():
    out, entry, argv = sys.argv[1], sys.argv[2], sys.argv[3:]
    args = cli.parse_args(entry, argv)
    env = launch.torchrun_env()
    assert env is not None, "launch with torch.distributed.run"
    args.nprocs = env[2]
    local_rank = env[1] if entry == "horovod_distributed" else cli.resolve_local_rank(args)
    driver.seed_everything(args)
    seen = {}

    class Recording(driver.STRATEGIES[entry]):
        def build(self, model, args, device, local_rank):
            model, opt = super().build(model, args, device, local_rank)
            seen["opt"], seen["st"] = opt, self
            return model, opt

    st = Recording()
    driver.main_worker(local_rank, args.nprocs, args, strategy=st)
    opt = seen["opt"]
    if torch.cuda.is_available():
        torch.cuda.synchronize()
    params = [p for g in opt.param_groups for p in g["params"]]
    masters = [m.detach().float().cpu().clone() for m in _amp.master_params(opt)]
    momenta = [opt.state[p]["momentum_buffer"].detach().float().cpu().clone() for p in params if "momentum_buffer" in opt.state.get(p, {})]
    stats = opt.larc_stats() if hasattr(opt, "larc_stats") else None
    os.makedirs(out, exist_ok=True)
    torch.save({"masters": masters, "momenta": momenta, "stats": None if stats is None else stats.cpu().clone(),
                "flat": bool(getattr(opt, "is_flat", False))},
               os.path.join(out, "rank%d.pt" % int(os.environ.get("RANK", local_rank))))


if __name__ == "__main__":
    main()
