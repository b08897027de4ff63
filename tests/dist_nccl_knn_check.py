"""Vector columns and DataStream.vector_nn_join on N NCCL ranks with the real kernels: launched with
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P tests/dist_nccl_knn_check.py
Vector rows cross the peer-memory exchange (the broadcast edge of the final phase, collect()) and every rank checks the gathered
result against the fp64 reference of tests/knn_cases.py."""
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
    import knn_cases as K
    from quokka_b200.df import QuokkaContext
    for name in ("case_vector_roundtrip", "case_vector_ops", "case_knn_api", "case_knn_fewer_rows"):
        qc = QuokkaContext()
        getattr(K, name)(qc)
        g = qc.last_graph
        if dist.get_rank() == 0:
            print(f"{name}: ok  (exchange calls {g.exchange.calls if g else 0}, via peer memory {g.exchange.peer_calls if g else 0})", flush=True)
    dist.barrier()
    dist.destroy_process_group()
    if local == 0:
        print("DIST_NCCL_KNN_OK", flush=True)


if __name__ == "__main__":
    main()
