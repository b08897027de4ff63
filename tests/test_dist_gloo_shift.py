"""OrderedStream.shift on two gloo ranks (kernels replaced by tests/cpu_shim.py + tests/shift_shim.py): range-partitioned input
from from_arrow_sorted and from sort(), keys straddling the ranks' boundary and keys with fewer than |n| rows on each rank, lag
and lead, by=None; the gathered result equals the one-rank answer row for row, and ranks holding out-of-order ranges raise."""
import os
import sys
import traceback

import torch.multiprocessing as mp

from test_dist_gloo import _free_port, _Patch

HERE = os.path.dirname(os.path.abspath(__file__))


def _worker(rank, world, port, out_dir):
    try:
        sys.path.insert(0, HERE)
        sys.path.insert(0, os.path.dirname(HERE))
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
        import torch.distributed as dist
        dist.init_process_group("gloo", rank=rank, world_size=world)
        import shift_shim
        shift_shim.install(_Patch())
        import shift_api_cases as A
        from quokka_b200.df import QuokkaContext
        golden = os.path.join(HERE, "golden")
        A.case_shift_lag_lead(QuokkaContext())
        A.case_shift_in_place(QuokkaContext())
        A.case_shift_fills(QuokkaContext())
        A.case_shift_nulls_from_left_join(QuokkaContext())
        A.case_sort_then_shift(QuokkaContext())
        A.case_shift_then_asof(QuokkaContext(), golden)
        A.case_shift_out_of_order(QuokkaContext())
        dist.barrier()
        dist.destroy_process_group()
        open(os.path.join(out_dir, f"ok{rank}"), "w").write("ok")
    except Exception:
        open(os.path.join(out_dir, f"fail{rank}"), "w").write(traceback.format_exc())
        raise


def test_shift_two_ranks_gloo(tmp_path):
    port = _free_port()
    ctx = mp.get_context("spawn")
    procs = [ctx.Process(target=_worker, args=(r, 2, port, str(tmp_path))) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=600)
    fails = [open(os.path.join(tmp_path, f)).read() for f in os.listdir(tmp_path) if f.startswith("fail")]
    assert not fails, "\n".join(fails)
    assert all(os.path.exists(os.path.join(tmp_path, f"ok{r}")) for r in range(2)), [p.exitcode for p in procs]
