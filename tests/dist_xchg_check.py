"""Multi-GPU parity of runtime.Exchange, launched with
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P tests/dist_xchg_check.py
Runs the checks of tests/xchg_cases.py over the peer-memory shuffle (csrc/exchange.cu), or over NCCL all_to_all_single with
QK_P2P=0.  On the link it also checks payloads larger than the mailbox (rounds, with QK_MAILBOX_MB set) and the exchange
driven from two lanes (threads + streams) at once."""
import os
import sys
import threading

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import torch
import torch.distributed as dist


def main():
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    import xchg_cases as XC
    from quokka_b200 import runtime as RT
    w, me = dist.get_world_size(), dist.get_rank()
    link = RT.native_link(dev)
    want_link = os.environ.get("QK_P2P", "1") != "0"
    assert (link is not None) == want_link, "the peer-memory link must be present exactly when QK_P2P is not 0"
    ex = RT.Exchange(dev)
    XC.run_all(ex, dev)

    # two lanes at once: different channels, different streams, interleaved in whatever order the threads run (the link
    # only: library collectives issued from two threads would not come in the same order on every rank)
    if link is not None:
        errors = []

        def lane(li):
            try:
                torch.cuda.set_device(dev)
                RT._lane.index = li
                with torch.cuda.stream(torch.cuda.Stream(dev)):
                    for rep in range(6):
                        XC.check_hash(ex, dev, 200_003 + li, 100 + 10 * li + rep, tag=f"lane{li}")
            except BaseException as e:
                errors.append(e)
        ts = [threading.Thread(target=lane, args=(li,)) for li in range(min(2, RT.N_LANES))]
        [t_.start() for t_ in ts]
        [t_.join() for t_ in ts]
        if errors:
            raise errors[0]
    torch.cuda.synchronize()
    peer_calls = ex.peer_calls
    assert link is not None or peer_calls == 0

    # payload larger than the mailbox: rounds
    if os.environ.get("QK_MAILBOX_MB"):
        XC.check_hash(ex, dev, 1_500_000, 40, tag="oversize")
    dist.barrier()
    dist.destroy_process_group()
    if me == 0:
        print(f"DIST_XCHG_OK world={w} exchanges_via_peer_memory={peer_calls}", flush=True)


if __name__ == "__main__":
    main()
