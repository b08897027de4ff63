"""runtime.Exchange over the peer-memory link protocol on CPU: the in-process link of tests/inproc_link.py with the channel
calls restated in numpy (tests/xchg_shim.py), W virtual ranks in threads.  The same cases run on one H100 against the
kernels in tests/test_gpu_xchg.py."""
import numpy as np
import pytest
import torch

import inproc_link as IL
import xchg_cases as XC
import xchg_shim
from quokka_b200 import _lib as L
from quokka_b200 import runtime as RT

CPU = torch.device("cpu")


def _exchange_on_link(monkeypatch, world, mailbox_bytes, cases):
    xchg_shim.install(monkeypatch)
    IL.install(monkeypatch)
    link = IL.InprocLink(world, mailbox_bytes, CPU, xchg_shim)

    def rank_body(r):
        ex = RT.Exchange(CPU)
        cases(ex, CPU)
        return ex

    exs = IL.run_ranks(link, rank_body)
    assert link.guard_clean()
    return exs


@pytest.mark.parametrize("world", [2, 3, 5, 16])
def test_exchange_cases_on_link(monkeypatch, world):
    exs = _exchange_on_link(monkeypatch, world, (16 << 20) + (128 << 20) // world, XC.run_all)
    assert all(ex.peer_calls > 0 for ex in exs)


@pytest.mark.parametrize("world", [2, 5])
def test_exchange_rounds_on_link(monkeypatch, world):
    """A 64 KB mailbox: the payloads go in rounds; the skewed edge makes rounds split again."""
    real = RT.Exchange._native_oversize

    def counted(self, *a):          # per Exchange, i.e. per rank thread
        self.depth = getattr(self, "depth", 0) + 1
        self.rounds_entered = getattr(self, "rounds_entered", 0) + 1
        self.max_depth = max(getattr(self, "max_depth", 0), self.depth)
        try:
            return real(self, *a)
        finally:
            self.depth -= 1

    monkeypatch.setattr(RT.Exchange, "_native_oversize", counted)
    exs = _exchange_on_link(monkeypatch, world, 64 << 10, XC.run_rounds)
    assert all(ex.rounds_entered >= 5 for ex in exs), "an edge of run_rounds did not go in rounds"
    assert max(ex.max_depth for ex in exs) >= 2, "no round overflowed a receiver"


def test_shim_limits():
    """The shim refuses what the C ABI refuses (the kernel-level tests of test_gpu_xchg.py check the C ABI itself)."""
    link = IL.InprocLink(2, 1 << 16, CPU, xchg_shim)
    ch = link.channels[0]
    ch.epoch = 1
    x = torch.zeros(10, dtype=torch.int64)
    too_many = [torch.zeros(4, dtype=torch.uint8)] * (L.XCHG_MAX_BUFS + 1)
    bad = [
        lambda: ch.push(too_many, [0, 0], [4, 4], [[0] * len(too_many)] * 2),
        lambda: ch.push([x], [0, 0], [10, 10], [[0], [(1 << 16) + 8]]),                         # offset outside the mailbox
        lambda: ch.push([x], [0, 0], [10, 10], [[0], [(1 << 16) - 8]]),                         # rows that do not fit
        lambda: ch.push([x], [0, 0], [10, 10], [[0], [4]]),                                     # misaligned destination offset
        lambda: ch.push_scatter([torch.zeros(10, 3)], torch.zeros(10, dtype=torch.int32), torch.tensor([0, 10, 10]), [[0], [0]]),
        lambda: ch.push_scatter([torch.zeros(10, dtype=torch.float16)], torch.zeros(10, dtype=torch.int32), torch.tensor([0, 10, 10]), [[0], [0]]),
        lambda: ch.recv([8], [torch.zeros(4, dtype=torch.int64)]),                              # misaligned mailbox offset
        lambda: ch.recv([0], [torch.zeros(17, dtype=torch.uint8)[1:]]),                        # misaligned output
    ]
    for i, call in enumerate(bad):
        with pytest.raises(L.QkError):
            call()
    c = link.ctrl(0)
    assert not c.data_flag.any() and int(c.err[0]) == 0, "a refused call released a flag or waited"
    assert not link.buf.any(), "a refused call wrote"
    ch.epoch = 0
    with pytest.raises(L.QkError):
        ch.push([x], [0, 0], [10, 10], [[0], [0]])                                              # epoch 0
    bad_ctrl = xchg_shim.XchgChannel(2, 0, [link.ctrl_ptrs[0], link.ctrl_ptrs[1] + 8], link.mailbox_ptrs, link.mailbox_bytes, CPU)
    with pytest.raises(L.QkError):
        bad_ctrl.meta([1])
    assert np.all(link.ctrl(1).meta_flag == 0)
