"""Multi-rank parity on real GPUs, driver-visible: when the box shows >= 2 GPUs, spawn 2 NCCL ranks (one per GPU) and run
(a) the exchange against numpy (tests/dist_xchg_check.py), over the peer-memory link and over NCCL all_to_all_single
(QK_P2P=0), and (b) the DataStream parity programs with every join shuffled (tests/dist_nccl_check.py).  Skipped on a
single-GPU box."""
import pytest
import torch

import ranks

pytestmark = pytest.mark.gpu


def _need_two():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")


def test_peer_memory_exchange_two_ranks():
    _need_two()
    rc, out = ranks.torchrun("dist_xchg_check.py", 2)
    assert rc == 0 and "DIST_XCHG_OK" in out, out[-4000:]


def test_peer_memory_exchange_rounds_when_the_mailbox_is_small():
    _need_two()
    rc, out = ranks.torchrun("dist_xchg_check.py", 2, env={"QK_MAILBOX_MB": "1"})
    assert rc == 0 and "DIST_XCHG_OK" in out, out[-4000:]


def test_nccl_exchange_two_ranks_without_the_link():
    _need_two()
    rc, out = ranks.torchrun("dist_xchg_check.py", 2, env={"QK_P2P": "0"})
    assert rc == 0 and "DIST_XCHG_OK" in out, out[-4000:]


def test_datastream_programs_two_ranks():
    _need_two()
    ranks.nccl_suites("api", "--more")
