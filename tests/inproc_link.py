"""An in-process peer-memory link: W virtual ranks of the K6 shuffle (csrc/exchange.cu) on ONE device.  A link never needs W
GPUs -- a peer is only a device pointer -- so W control blocks and W mailboxes that are slices of one allocation run exactly
the kernel code W GPUs would.

No wait kernel may ever spin: W spinning kernels are not guaranteed to be resident together, and streams alias onto a few
hardware queues, so two "ranks" could serialise falsely and one would wait out its deadline.  The harness therefore orders
every launch so that each flag a wait reads is already released:

  * meta round: the ranks post in turn, r = 0 .. W-1.  Before rank r's qk_xchg_meta, the rows and meta flags of the ranks
    t > r whose turn has not come are written into rank r's control block (what rank t's kernel would store there); after
    the turn they are overwritten with POISON, so that the check at the end of the round sees only what the kernels wrote;
  * payload: every rank's push completes (its stream synchronised) before any rank's recv is launched.

As a backstop every wait's flags are read before it is launched (`HarnessError` if one is missing), and channels get a
deadline of a few seconds, so a harness bug becomes a QkError, not a long spin.

`ops` is quokka_b200.ops (the kernels) or tests/xchg_shim.py (numpy, CPU).  `run_ranks` drives runtime.Exchange: one
thread and one stream per virtual rank, runtime.native_link / world_size / rank patched to thread-local values."""
from __future__ import annotations

import threading
import types

import numpy as np
import torch

from quokka_b200 import _lib as L

MP, MW, CTRL = L.MAX_PEERS, L.XCHG_META_WORDS, L.XCHG_CTRL_BYTES

# byte layout of `struct XchgCtrl` (csrc/exchange.cu): meta_flag[MP] u64, data_flag[MP] u64, err u64, push_done u32, pad u32,
# meta[2][MP][MW] i64 -- the one place the tests restate it
META_FLAG_OFF = 0
DATA_FLAG_OFF = META_FLAG_OFF + 8 * MP
ERR_OFF = DATA_FLAG_OFF + 8 * MP
PUSH_DONE_OFF = ERR_OFF + 8
META_OFF = PUSH_DONE_OFF + 8
CTRL_USED = META_OFF + 2 * MP * MW * 8
assert CTRL_USED <= CTRL

POISON = -0x5A5A5A5A5A5A5A5B


class HarnessError(AssertionError):
    """The harness was about to launch a wait whose flag is not released: a bug in the harness, never in the kernels."""


def ctrl_view(raw: np.ndarray):
    """Named numpy views of one control block (`raw`: its uint8 bytes); writes go through to `raw`."""
    return types.SimpleNamespace(
        meta_flag=raw[META_FLAG_OFF:DATA_FLAG_OFF].view(np.uint64),
        data_flag=raw[DATA_FLAG_OFF:ERR_OFF].view(np.uint64),
        err=raw[ERR_OFF:PUSH_DONE_OFF].view(np.uint64),
        push_done=raw[PUSH_DONE_OFF:PUSH_DONE_OFF + 4].view(np.uint32),
        meta=raw[META_OFF:CTRL_USED].view(np.int64).reshape(2, MP, MW))


def meta_row(world: int, words, part_offsets=None) -> np.ndarray:
    """The row qk_xchg_meta posts: the host words, words[0 .. world) replaced by the plan's counts when it has one."""
    row = np.zeros(MW, dtype=np.int64)
    row[:len(words)] = [int(x) for x in words]
    if part_offsets is not None:
        offs = part_offsets.cpu().numpy().astype(np.int64)
        row[:world] = offs[1:world + 1] - offs[:world]
    return row


class InprocLink:
    """W channels over one allocation: W control blocks, then W mailboxes, then a mailbox-sized guard zone that no kernel
    may write (`guard_clean`)."""

    def __init__(self, world: int, mailbox_bytes: int, device, ops, timeout_ms: int = 5000):
        self.world, self.device, self.ops = int(world), torch.device(device), ops
        self.mailbox_bytes = (int(mailbox_bytes) + 4095) // 4096 * 4096
        self.head = (self.world * CTRL + 65535) // 65536 * 65536
        self.buf = torch.zeros(self.head + (self.world + 1) * self.mailbox_bytes, dtype=torch.uint8, device=self.device)
        base = self.buf.data_ptr()
        self.ctrl_ptrs = [base + r * CTRL for r in range(self.world)]
        self.mailbox_ptrs = [base + self.head + r * self.mailbox_bytes for r in range(self.world)]
        self.channels = [ops.XchgChannel(self.world, r, self.ctrl_ptrs, self.mailbox_ptrs, self.mailbox_bytes, self.device, timeout_ms)
                         for r in range(self.world)]
        self._sync()

    # ------------------------------------------------------------------ raw access
    def _sync(self):
        if self.device.type == "cuda":
            torch.cuda.current_stream(self.device).synchronize()

    def ctrl(self, r: int):
        """A host copy of rank r's control block (named views)."""
        self._sync()
        return ctrl_view(self.buf[r * CTRL:r * CTRL + CTRL_USED].cpu().numpy().copy())

    def mailbox(self, r: int) -> torch.Tensor:
        o = self.head + r * self.mailbox_bytes
        return self.buf[o:o + self.mailbox_bytes]

    def guard_clean(self) -> bool:
        o = self.head + self.world * self.mailbox_bytes
        return not bool(self.buf[o:o + self.mailbox_bytes].any())

    def _write(self, byte_off: int, words: np.ndarray):
        src = torch.from_numpy(np.ascontiguousarray(words).view(np.uint8).copy())
        self.buf[byte_off:byte_off + src.numel()].copy_(src)

    def _put_row(self, r: int, t: int, epoch: int, row: np.ndarray):
        self._write(r * CTRL + META_OFF + ((epoch & 1) * MP + t) * MW * 8, row.astype(np.int64))

    def prewrite(self, r: int, t: int, epoch: int, row: np.ndarray):
        """What rank t's meta kernel of `epoch` stores into rank r's control block: its row, then its flag."""
        self._put_row(r, t, epoch, row)
        self._write(r * CTRL + META_FLAG_OFF + 8 * t, np.array([epoch], dtype=np.uint64))

    def require_flags(self, r: int, kind: str, epoch: int):
        """Backstop: every flag the wait of rank r (`kind` = "meta" or "data") will read is already released."""
        c = self.ctrl(r)
        flags = c.meta_flag if kind == "meta" else c.data_flag
        skip = r if kind == "meta" else -1          # a meta kernel releases its own flag before it waits on it
        missing = [t for t in range(self.world) if t != skip and int(flags[t]) < epoch]
        if missing:
            raise HarnessError(f"rank {r}: {kind} flags of ranks {missing} not released for epoch {epoch} before the wait")

    # ------------------------------------------------------------------ the meta round
    def meta_turn(self, r: int, words, part_offsets=None, ahead=()):
        """Rank r posts its row of the channel's next epoch.  `ahead`: (t, row) of the ranks whose turn for this epoch has
        not come; their rows and flags are pre-written into rank r's block, and poisoned again once the turn is over."""
        ch = self.channels[r]
        epoch = ch.epoch + 1
        for t, row in ahead:
            self.prewrite(r, t, epoch, row)
        self.require_flags(r, "meta", epoch)
        out = ch.meta(words, part_offsets)
        for t, _ in ahead:
            self._put_row(r, t, epoch, np.full(MW, POISON, dtype=np.int64))
        self._sync()
        return out

    def check_round(self, r: int, epoch: int, rows):
        """After every rank's turn of `epoch`: rank r's block holds the row every rank's kernel wrote."""
        got = self.ctrl(r).meta[epoch & 1, :self.world]
        for t in range(self.world):
            assert np.array_equal(got[t], rows[t]), (r, t, epoch, got[t][:8], rows[t][:8])

    def meta_round(self, words, part_offsets=None):
        """One meta round of every rank, in turn (words[r] / part_offsets[r]: rank r's).  Returns every rank's matrix,
        after checking them and every control block against the expected rows."""
        W = self.world
        part_offsets = part_offsets if part_offsets is not None else [None] * W
        epoch = self.channels[0].epoch + 1
        assert all(ch.epoch + 1 == epoch for ch in self.channels), "meta_round: the channels are at different epochs"
        rows = [meta_row(W, words[r], part_offsets[r]) for r in range(W)]
        outs = [self.meta_turn(r, words[r], part_offsets[r], [(t, rows[t]) for t in range(r + 1, W)]) for r in range(W)]
        for r in range(W):
            self.check_round(r, epoch, rows)
            assert np.array_equal(outs[r], np.stack(rows)), r
        return outs

    def recv(self, r: int, src_byte_off, outs):
        """Rank r's receive, after the pushes of every rank (the backstop checks that they released their flags)."""
        self._sync()
        self.require_flags(r, "data", self.channels[r].epoch)
        self.channels[r].recv(src_byte_off, outs)


# ------------------------------------------------------------------ runtime.Exchange on the in-process link
class _Rank:
    """The `.channels[0]` runtime.Exchange sees on one virtual rank: the real channel, with the calls ordered across the
    rank threads (meta in turns, every push before any recv)."""

    def __init__(self, link: InprocLink, r: int, barrier: threading.Barrier, rows: list):
        self.link, self.ch, self.barrier, self.rows = link, link.channels[r], barrier, rows
        self.world, self.rank, self.mailbox_bytes = link.world, r, link.mailbox_bytes

    def meta(self, words, part_offsets=None):
        W, r = self.world, self.rank
        epoch = self.ch.epoch + 1
        self.rows[r] = (epoch, meta_row(W, words, part_offsets))
        self.barrier.wait()
        assert all(e == epoch for e, _ in self.rows), ("ranks disagree on the epoch", [e for e, _ in self.rows])
        rows = [row for _, row in self.rows]
        out = None
        for turn in range(W):
            if turn == r:
                out = self.link.meta_turn(r, words, part_offsets, [(t, rows[t]) for t in range(r + 1, W)])
            self.barrier.wait()
        self.link.check_round(r, epoch, rows)
        assert np.array_equal(out, np.stack(rows)), (r, epoch)
        self.barrier.wait()          # nobody posts the next epoch's row before every rank has checked this one
        return out

    def _pushed(self):
        self.link._sync()
        self.barrier.wait()

    def push(self, *a):
        self.ch.push(*a)
        self._pushed()

    def push_scatter(self, *a):
        self.ch.push_scatter(*a)
        self._pushed()

    def recv(self, src_byte_off, outs):
        self.link.recv(self.rank, src_byte_off, outs)


_tls = threading.local()


def install(patch):
    """runtime.world_size / rank / native_link answer for the calling rank thread (1 / 0 / None elsewhere)."""
    from quokka_b200 import runtime as RT
    patch.setattr(RT, "world_size", lambda: getattr(_tls, "world", 1))
    patch.setattr(RT, "rank", lambda: getattr(_tls, "rank", 0))
    patch.setattr(RT, "native_link", lambda device: getattr(_tls, "link", None))


def run_ranks(link: InprocLink, fn, timeout_s: float = 600.0):
    """fn(rank) on every virtual rank, each in its own thread (and CUDA stream), with runtime's view of the world patched
    by `install`.  Returns the per-rank results; re-raises the first failure."""
    W = link.world
    barrier = threading.Barrier(W, timeout=timeout_s)
    rows = [(0, None)] * W
    results, errors = [None] * W, [None] * W

    def body(r):
        _tls.world, _tls.rank = W, r
        _tls.link = types.SimpleNamespace(channels=[_Rank(link, r, barrier, rows)], mailbox_bytes=link.mailbox_bytes)
        try:
            if link.device.type == "cuda":
                with torch.cuda.stream(torch.cuda.Stream(link.device)):
                    results[r] = fn(r)
                    link._sync()
            else:
                results[r] = fn(r)
        except BaseException as e:      # noqa: B902 -- reported below; the other ranks must not wait for this one
            errors[r] = e
            barrier.abort()
        finally:
            del _tls.world, _tls.rank, _tls.link

    threads = [threading.Thread(target=body, args=(r,), name=f"inproc-rank{r}") for r in range(W)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    real = [e for e in errors if e is not None and not isinstance(e, threading.BrokenBarrierError)]
    if real or any(e is not None for e in errors):
        raise (real or [e for e in errors if e is not None])[0]
    return results
