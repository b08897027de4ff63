"""DataStream.approximate_quantile on two gloo ranks (kernels replaced by tests/cpu_shim.py + tests/quantile_shim.py): each
rank sketches its share of the rows and the final phase merges the entries of both.  Both ranks must get the one-rank
answer exactly: the numpy sketch of all the rows, bit for bit."""
import os
import sys
import traceback

import numpy as np
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
        import pyarrow as pa
        import quantile_shim
        quantile_shim.install(_Patch())
        import quantile_cases as QC
        from quokka_b200.df import QuokkaContext
        cols = QC.special_columns(20_011, 17)
        names = list(cols)
        qc = QuokkaContext()
        qs = [0.0, 0.1, 0.5, 0.9, 1.0]
        t = qc.from_arrow(pa.table(cols)).approximate_quantile(names, qs).collect()
        QC.assert_matches(t, names, qs, [cols[c] for c in names], what=f"rank {rank}")
        QC.case_quantile_tpch_606(qc)
        QC.case_quantile_empty(qc)
        dist.barrier()
        dist.destroy_process_group()
        open(os.path.join(out_dir, f"ok{rank}"), "w").write("ok")
    except Exception:
        open(os.path.join(out_dir, f"fail{rank}"), "w").write(traceback.format_exc())
        raise


def test_quantile_two_ranks_gloo(tmp_path):
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
