"""DataStream.gramian / covariance on two gloo ranks (kernels replaced by tests/cpu_shim.py + tests/gram_shim.py): each rank folds its share of the
rows with its own shift, and the final phase re-centres the partials on the global mean.  Both ranks must get the one-rank
result within the summation bound of tests/gram_cases.py."""
import os
import sys
import traceback

import numpy as np
import torch.multiprocessing as mp

from test_dist_gloo import _free_port, _Patch

HERE = os.path.dirname(os.path.abspath(__file__))


def _data():
    rng = np.random.default_rng(17)
    n = 20_011
    return {"a": rng.normal(3e4, 5.0, n), "b": rng.integers(-1000, 1000, n).astype(np.int64),
            "c": rng.normal(-2.0, 1e-3, n).astype(np.float32), "d": rng.normal(0, 1e6, n)}


def _worker(rank, world, port, out_dir):
    try:
        sys.path.insert(0, HERE)
        sys.path.insert(0, os.path.dirname(HERE))
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
        import torch.distributed as dist
        dist.init_process_group("gloo", rank=rank, world_size=world)
        import pyarrow as pa
        import gram_shim
        gram_shim.install(_Patch())
        import gram_cases as GC
        from quokka_b200.df import QuokkaContext
        cols = _data()
        names = list(cols)
        x = np.stack([cols[c].astype(np.float64) for c in names], axis=1)
        qc = QuokkaContext()
        d = qc.from_arrow(pa.table(cols))
        g, b = GC.gram_ref(x)
        GC.assert_within(GC.table_matrix(d.gramian(names).collect(), names), g, b, f"gramian on rank {rank}")
        shift = x.mean(axis=0)
        g, b = GC.gram_ref(x, shift)
        GC.assert_within(GC.table_matrix(d.gramian(names, demean=shift).collect(), names), g, b, f"gramian demean on rank {rank}")
        c, b = GC.cov_ref(x)
        GC.assert_within(GC.table_matrix(d.covariance(names), names), c, b, f"covariance on rank {rank}")
        GC.case_gram_filtered_ints(qc)
        GC.case_gram_empty(qc)
        dist.barrier()
        dist.destroy_process_group()
        open(os.path.join(out_dir, f"ok{rank}"), "w").write("ok")
    except Exception:
        open(os.path.join(out_dir, f"fail{rank}"), "w").write(traceback.format_exc())
        raise


def test_gram_two_ranks_gloo(tmp_path):
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
