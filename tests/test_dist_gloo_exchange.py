"""runtime.Exchange over torch.distributed collectives on gloo ranks (kernels replaced by tests/cpu_shim.py): the parity
checks of tests/xchg_cases.py -- hash edges at several sizes with empty ranks, broadcast with per-rank dictionaries and
a validity mask, single owner, the small all-gather -- that tests/dist_xchg_check.py runs on GPUs."""
import os
import sys
import traceback

import pytest
import torch
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
        import cpu_shim
        cpu_shim.install(_Patch())
        import xchg_cases as XC
        from quokka_b200 import runtime as RT
        dev = torch.device("cpu")
        ex = RT.Exchange(dev)
        XC.run_all(ex, dev)
        assert ex.peer_calls == 0
        dist.barrier()
        dist.destroy_process_group()
        open(os.path.join(out_dir, f"ok{rank}"), "w").write("ok")
    except Exception:
        open(os.path.join(out_dir, f"fail{rank}"), "w").write(traceback.format_exc())
        raise


@pytest.mark.parametrize("world", [2, 3])
def test_exchange_parity_gloo(tmp_path, world):
    port = _free_port()
    ctx = mp.get_context("spawn")
    procs = [ctx.Process(target=_worker, args=(r, world, port, str(tmp_path))) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=600)
    fails = [open(os.path.join(tmp_path, f)).read() for f in os.listdir(tmp_path) if f.startswith("fail")]
    assert not fails, "\n".join(fails)
    assert all(os.path.exists(os.path.join(tmp_path, f"ok{r}")) for r in range(world)), [p.exitcode for p in procs]
