"""runtime.Exchange over torch.distributed collectives on gloo ranks (kernels replaced by tests/cpu_shim.py): the parity
checks of tests/xchg_cases.py -- hash edges at several sizes with empty ranks, broadcast with per-rank dictionaries and
a validity mask, single owner, the small all-gather -- that tests/dist_xchg_check.py runs on GPUs."""
import pytest

import ranks


def case_exchange_parity():
    import torch
    import xchg_cases as XC
    from quokka_b200 import runtime as RT
    dev = torch.device("cpu")
    ex = RT.Exchange(dev)
    XC.run_all(ex, dev)
    assert ex.peer_calls == 0


@pytest.mark.parametrize("world", [2, 3])
def test_exchange_parity_gloo(tmp_path, world):
    ranks.spawn(tmp_path, world, ranks.gloo_rank, ["test_dist_gloo_exchange:case_exchange_parity"])
