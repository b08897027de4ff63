"""OrderedStream.pattern_recognize on N NCCL ranks with the real kernels: launched with
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P tests/dist_nccl_pattern_check.py
Every rank runs the API cases of tests/pattern_cases.py and checks the gathered result against the brute-force oracle."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import torch
import torch.distributed as dist


def main():
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    import pattern_cases as P
    from quokka_b200.df import QuokkaContext
    for case in P.API_CASES:
        case(QuokkaContext())
        if dist.get_rank() == 0:
            print(f"{case.__name__}: ok", flush=True)
    dist.barrier()
    dist.destroy_process_group()
    if local == 0:
        print("DIST_NCCL_PATTERN_OK", flush=True)


if __name__ == "__main__":
    main()
