"""The order-preserving join cases (tests/ordered_join_api_cases.py) on real kernels across ranks, launched by
tests/test_gpu_ordered_join.py through ranks.torchrun:
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N ... tests/dist_nccl_ordered_join_check.py
It is tests/dist_nccl_check.py with this feature's case list: rank 0 prints `<case>: ok` after each case and the marker
ranks.NCCL_MARKER at the end."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import dist_nccl_check

if __name__ == "__main__":
    dist_nccl_check.main(["ordered_join"])
