"""One rank of an entrypoint's training loop with ``--model-ema`` (launched by torch.distributed.run) that, at the end, writes
this rank's weight averages (``ModelEma.state_dict()``, fp32) to OUT/rank<r>.pt.  Tests compare the files of all ranks
bit for bit.

    python -m torch.distributed.run --nproc-per-node 2 tests/mp_model_ema_checks.py OUT ENTRY <driver flags>
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from pytorch_distributed_b200 import cli, driver, launch  # noqa: E402


def main():
    out, entry, argv = sys.argv[1], sys.argv[2], sys.argv[3:]
    args = cli.parse_args(entry, argv)
    env = launch.torchrun_env()
    assert env is not None, "launch with torch.distributed.run"
    args.nprocs = env[2]
    local_rank = env[1] if entry == "horovod_distributed" else cli.resolve_local_rank(args)
    driver.seed_everything(args)
    st = driver.STRATEGIES[entry]()
    driver.main_worker(local_rank, args.nprocs, args, strategy=st)
    if torch.cuda.is_available():
        torch.cuda.synchronize()
    ema = st.model_ema
    sd = {k: v.detach().cpu().clone() for k, v in ema.state_dict().items()}
    os.makedirs(out, exist_ok=True)
    torch.save({"ema": sd, "flat": ema._fused is not None and bool(getattr(ema._fused, "is_flat", False))},
               os.path.join(out, "rank%d.pt" % int(os.environ.get("RANK", local_rank))))


if __name__ == "__main__":
    main()
