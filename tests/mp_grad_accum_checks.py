"""One rank of an entrypoint's training loop with ``--accum-steps`` (launched by torch.distributed.run) that, at the end, writes
what this rank's optimizer holds to OUT/rank<r>.pt: the fp32 masters and momentum buffers, and whether the engine's fp32
accumulator is back at zero with nothing pending.  Tests compare the files of all ranks bit for bit.

    python -m torch.distributed.run --nproc-per-node 2 tests/mp_grad_accum_checks.py OUT ENTRY <driver flags>
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
    opt, eng = seen["opt"], getattr(seen["st"], "engine", None)
    if torch.cuda.is_available():
        torch.cuda.synchronize()
    params = [p for g in opt.param_groups for p in g["params"]]
    masters = [m.detach().float().cpu().clone() for m in _amp.master_params(opt)]
    momenta = [opt.state[p]["momentum_buffer"].detach().float().cpu().clone() for p in params if "momentum_buffer" in opt.state.get(p, {})]
    acc = getattr(eng, "_acc", None)
    os.makedirs(out, exist_ok=True)
    torch.save({"masters": masters, "momenta": momenta, "fp32_accum": bool(getattr(eng, "fp32_accum", False)),
                "acc_clear": acc is None or not bool(acc.any()), "pending": bool(getattr(eng, "accum_pending", False))},
               os.path.join(out, "rank%d.pt" % int(os.environ.get("RANK", local_rank))))


if __name__ == "__main__":
    main()
