"""Multi-rank parity on real GPUs, driver-visible: when the box shows >= 2 GPUs, spawn 2 NCCL ranks (one per GPU) and run
(a) the exchange against numpy (tests/dist_xchg_check.py), over the peer-memory link and over NCCL all_to_all_single
(QK_P2P=0), and (b) the DataStream parity programs with every join shuffled (tests/dist_nccl_check.py).  Skipped on a
single-GPU box."""
import os
import socket
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _torchrun(script, nproc, env=None, args=(), timeout=600):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}", "--master-addr", "127.0.0.1",
           "--master-port", str(_free_port()), os.path.join(HERE, script), *args]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=timeout, env={**os.environ, **(env or {})})
    return r.returncode, r.stdout.decode(errors="replace")


def _need_two():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")


def test_peer_memory_exchange_two_ranks():
    _need_two()
    rc, out = _torchrun("dist_xchg_check.py", 2)
    assert rc == 0 and "DIST_XCHG_OK" in out, out[-4000:]


def test_peer_memory_exchange_rounds_when_the_mailbox_is_small():
    _need_two()
    rc, out = _torchrun("dist_xchg_check.py", 2, env={"QK_MAILBOX_MB": "1"})
    assert rc == 0 and "DIST_XCHG_OK" in out, out[-4000:]


def test_nccl_exchange_two_ranks_without_the_link():
    _need_two()
    rc, out = _torchrun("dist_xchg_check.py", 2, env={"QK_P2P": "0"})
    assert rc == 0 and "DIST_XCHG_OK" in out, out[-4000:]


def test_datastream_programs_two_ranks():
    _need_two()
    rc, out = _torchrun("dist_nccl_check.py", 2, args=("--more",))
    assert rc == 0 and "DIST_NCCL_OK" in out, out[-4000:]
