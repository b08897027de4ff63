"""Multi-GPU parity run (real kernels + NCCL all-to-all or the peer-memory link), launched by tests/ranks.py torchrun as
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P tests/dist_nccl_check.py SUITE...
Each argument names a case list of tests/ranks.py SUITES (`api --more`, `sort`, `shift`, `knn`, `pattern`).  Every rank runs
the same DataStream programs and checks the gathered result against the oracle; rank 0 prints `<case>: ok` after each case
and the marker ranks.NCCL_MARKER at the end."""
import os
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import torch
import torch.distributed as dist

import ranks


def main(suites):
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    with tempfile.TemporaryDirectory() as files:
        ranks.run_cases([n for s in suites for n in ranks.SUITES[s]], dist.get_rank(), dist.get_world_size(), files)
    dist.barrier()
    dist.destroy_process_group()
    if local == 0:
        print(ranks.NCCL_MARKER, flush=True)


if __name__ == "__main__":
    main(sys.argv[1:])
