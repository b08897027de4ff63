"""OrderedStream.shift on N NCCL ranks with the real kernels: launched with
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P tests/dist_nccl_shift_check.py
Every rank runs the API cases of tests/shift_api_cases.py and checks the gathered result against the reference."""
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
    import shift_api_cases as A
    from quokka_b200.df import QuokkaContext
    golden = os.path.join(HERE, "golden")
    for case, args in ((A.case_shift_lag_lead, ()), (A.case_shift_in_place, ()), (A.case_shift_fills, ()),
                       (A.case_shift_nulls_from_left_join, ()), (A.case_sort_then_shift, ()), (A.case_shift_then_asof, (golden,)),
                       (A.case_shift_out_of_order, ())):
        case(QuokkaContext(), *args)
        if dist.get_rank() == 0:
            print(f"{case.__name__}: ok", flush=True)
    dist.barrier()
    dist.destroy_process_group()
    if local == 0:
        print("DIST_NCCL_SHIFT_OK", flush=True)


if __name__ == "__main__":
    main()
