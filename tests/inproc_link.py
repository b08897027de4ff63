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

As a backstop every wait's flags are read before it is launched (`HarnessError` if one is missing), channels get a
deadline of a few seconds, and the rank barrier of a channel times out after a minute, so a harness bug becomes an error,
not a long spin or a stall.

`ops` is quokka_b200.ops (the kernels) or tests/xchg_shim.py (numpy, CPU).  `run_ranks` runs a function on every virtual
rank: one thread and one stream per rank, with the world, the rank, the link and the lane streams answered per rank
(`install`).  A rank sees its link as runtime.NativeLink lays it out: channel 0 for the driver thread, channel 1 + i for
pipeline lane i, each channel an InprocLink of its own.  `run_program_ranks` runs DataStream programs (tests/ranks.py
run_cases) that way and checks every channel afterwards."""
from __future__ import annotations

import collections
import sys
import tempfile
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

    def __init__(self, world: int, mailbox_bytes: int, device, ops, timeout_ms: int = 5000, barrier_timeout_s: float = 60.0):
        self.world, self.device, self.ops = int(world), torch.device(device), ops
        self.barrier = threading.Barrier(self.world, timeout=barrier_timeout_s)      # the rank threads of this channel
        self.rows = [(0, None)] * self.world
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

    def check_clean_end(self, what=""):
        """After a run: the guard zone is untouched, no wait of any rank timed out, and every rank's channel has seen the
        same number of epochs."""
        self._sync()
        assert self.guard_clean(), f"{what}: a kernel wrote past the last mailbox"
        errs = [int(self.ctrl(r).err[0]) for r in range(self.world)]
        assert not any(errs), f"{what}: error words {[hex(e) for e in errs]}"
        epochs = [ch.epoch for ch in self.channels]
        assert len(set(epochs)) == 1, f"{what}: the ranks end at different epochs {epochs}"

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
    """One channel runtime.Exchange sees on one virtual rank: the real channel, with the calls ordered across the rank
    threads of that channel (meta in turns, every push before any recv)."""

    def __init__(self, link: InprocLink, r: int):
        self.link, self.ch, self.barrier, self.rows = link, link.channels[r], link.barrier, link.rows
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


_tls = threading.local()              # .ctx: the virtual rank of the calling thread
_running = [0]                        # rank runs in progress
_real = {}                            # the functions `install` replaces, saved before anything is patched


def _ctx():
    ctx = getattr(_tls, "ctx", None)
    if ctx is None and _running[0]:
        raise HarnessError(f"thread {threading.current_thread().name!r} belongs to no virtual rank, and ranks are running")
    return ctx


def _world_size():
    ctx = _ctx()
    return ctx.world if ctx is not None else 1


def _rank():
    ctx = _ctx()
    return ctx.rank if ctx is not None else 0


def _native_link(device):
    ctx = _ctx()
    return ctx.link if ctx is not None else None


def _lane_streams(device):
    """Every virtual rank owns its lane streams, as a real rank (a process) does."""
    ctx = _ctx()
    if ctx is None:
        return _real["lane_streams"](device)
    if ctx.lane_streams is None:
        from quokka_b200 import runtime as RT
        ctx.lane_streams = [torch.cuda.Stream(device) for _ in range(RT.N_LANES)]
    return ctx.lane_streams


class _RankThread(threading.Thread):
    """A thread that runtime starts from a rank's thread (a pipeline lane) belongs to that rank."""

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self._rank_ctx = getattr(_tls, "ctx", None)

    def run(self):
        _tls.ctx = self._rank_ctx
        try:
            super().run()
        finally:
            _tls.ctx = None


class _Threading(types.ModuleType):
    """runtime's `threading`, with Thread replaced by _RankThread."""
    Thread = _RankThread

    def __getattr__(self, name):
        return getattr(threading, name)


def install(patch):
    """columns.world_size / columns.rank / runtime.native_link answer for the virtual rank of the calling thread (1 / 0 / None
    outside a run), wherever a quokka_b200 module bound them by name; runtime's lane threads join the rank that starts them,
    and runtime.lane_streams gives each rank streams of its own."""
    from quokka_b200 import columns as C
    from quokka_b200 import runtime as RT
    if not _real:
        _real.update(world_size=C.world_size, rank=C.rank, native_link=RT.native_link, lane_streams=RT.lane_streams)
    fakes = [(_real["world_size"], _world_size), (_real["rank"], _rank), (_real["native_link"], _native_link),
             (_real["lane_streams"], _lane_streams)]
    for name, mod in list(sys.modules.items()):
        if mod is None or not (name == "quokka_b200" or name.startswith("quokka_b200.")):
            continue
        for attr, value in list(vars(mod).items()):
            for real, fake in fakes:
                if value is real:
                    patch.setattr(mod, attr, fake)
    patch.setattr(RT, "threading", _Threading("threading"))


def make_links(world: int, mailbox_bytes: int, device, ops) -> list:
    """The channels of runtime.NativeLink: 1 + runtime.N_LANES in-process links of `mailbox_bytes` each."""
    from quokka_b200 import runtime as RT
    return [InprocLink(world, mailbox_bytes, device, ops) for _ in range(1 + RT.N_LANES)]


def run_ranks(links, fn):
    """fn(rank) on every virtual rank, each in its own thread (and CUDA stream), with runtime's view of the world answered
    per rank by `install`.  `links`: one InprocLink, or the channels of make_links.  Returns the per-rank results;
    re-raises the first failure (after aborting every channel's barrier, so no rank waits for a failed one)."""
    links = [links] if isinstance(links, InprocLink) else list(links)
    W, device = links[0].world, links[0].device
    results, errors = [None] * W, [None] * W

    def body(r):
        _tls.ctx = types.SimpleNamespace(world=W, rank=r, lane_streams=None, link=types.SimpleNamespace(
            channels=[_Rank(link, r) for link in links], mailbox_bytes=links[0].mailbox_bytes))
        try:
            if device.type == "cuda":
                with torch.cuda.stream(torch.cuda.Stream(device)):
                    results[r] = fn(r)
                    links[0]._sync()
            else:
                results[r] = fn(r)
        except BaseException as e:      # noqa: B902 -- reported below; the other ranks must not wait for this one
            errors[r] = e
            for link in links:
                link.barrier.abort()
        finally:
            _tls.ctx = None

    threads = [threading.Thread(target=body, args=(r,), name=f"inproc-rank{r}") for r in range(W)]
    _running[0] += 1
    try:
        for t in threads:
            t.start()
        for t in threads:
            t.join()
    finally:
        _running[0] -= 1
    real = [e for e in errors if e is not None and not isinstance(e, threading.BrokenBarrierError)]
    if real or any(e is not None for e in errors):
        raise (real or [e for e in errors if e is not None])[0]
    return results


# ------------------------------------------------------------------ DataStream programs on in-process ranks
def _count_calls(patch, ops, counts, lock):
    """Counts, in `counts`, the calls that only multi-rank execution makes: an ordered join's placement of the owners'
    matches, an as-of merge over the ranks' time ranges with the carried rows of earlier / later ranks (the streaming path
    passes a carry of its own on one rank too, so only SortedAsofExecutor._join_carried's calls count), a shift with
    boundary rows, the merge of top-k lists and of quantile sketch entries, an exchange that goes in rounds, a left join's
    NULL columns on a rank without build rows; and the most lanes a TaskGraph ran on."""
    from quokka_b200 import executors as X
    from quokka_b200 import runtime as RT
    carried = threading.local()         # .on: inside _join_carried on this thread

    def bump(key, n=1):
        with lock:
            counts[key] += n

    def wrap(owner, name, key_of, static=False):
        real = getattr(owner, name)

        def counted(*a, **kw):
            for key in key_of(*a, **kw):
                bump(key)
            return real(*a, **kw)
        patch.setattr(owner, name, staticmethod(counted) if static else counted)

    def asof_keys(*a, **kw):
        if not getattr(carried, "on", False):
            return []
        back = a[5] if len(a) > 5 else kw.get("carry_in")
        return (["asof_carry"] if back is not None else []) + (["asof_carry_fwd"] if kw.get("carry_fwd") is not None else [])

    wrap(ops.JoinTable, "place", lambda *a, **kw: ["join_place"], static=True)
    wrap(ops, "asof_merge", asof_keys)
    wrap(ops, "shift_gather", lambda a, b, *r, **kw: ["shift_boundary"] if b is not None else [])
    wrap(ops, "knn_merge", lambda *a, **kw: ["knn_merge"])
    wrap(ops.QuantileSketch, "merge", lambda *a, **kw: ["qsketch_merge"])
    wrap(RT.Exchange, "_native_oversize", lambda *a, **kw: ["exchange_rounds"])
    wrap(X.BuildProbeJoinExecutor, "_unmatched", lambda *a, **kw: ["left_template"])
    real_carried = X.SortedAsofExecutor._join_carried

    def join_carried(self, *a, **kw):
        carried.on = True
        try:
            return real_carried(self, *a, **kw)
        finally:
            carried.on = False
    patch.setattr(X.SortedAsofExecutor, "_join_carried", join_carried)
    real_run = RT.TaskGraph.run

    def run(self):
        out = real_run(self)
        with lock:
            counts["lanes_used"] = max(counts["lanes_used"], self.lanes_used)
        return out
    patch.setattr(RT.TaskGraph, "run", run)


def run_program_ranks(world: int, names, device, mailbox_bytes: int) -> collections.Counter:
    """tests/ranks.py run_cases(names) on `world` virtual ranks in threads of this process: on the kernels (quokka_b200.ops)
    over the in-process link when `device` is CUDA, on tests/cpu_shim.py with the channels of tests/xchg_shim.py on CPU.
    Every case checks what each rank gathers.  Afterwards every channel must end clean (InprocLink.check_clean_end).
    Returns the counters of _count_calls, summed over the ranks."""
    import pytest
    import ranks
    device = torch.device(device)
    counts, lock = collections.Counter(), threading.Lock()
    with pytest.MonkeyPatch.context() as mp, tempfile.TemporaryDirectory() as files:
        if device.type == "cuda":
            from quokka_b200 import ops
        else:
            import cpu_shim as ops
            ops.install(mp)
        _count_calls(mp, ops, counts, lock)
        install(mp)
        links = make_links(world, mailbox_bytes, device, ops)
        run_ranks(links, lambda r: ranks.run_cases(names, r, world, files))
        for i, link in enumerate(links):
            link.check_clean_end(f"channel {i}")
    return counts


# the counters of _count_calls that a suite of tests/ranks.py SUITES must reach at world > 1, on any mailbox
REACHES = {
    "api": ["asof_carry"],
    "sort": ["asof_carry"],
    "shift": ["shift_boundary"],
    "knn": ["knn_merge"],
    "ordered_join": ["join_place"],
    "asof_strategy": ["asof_carry", "asof_carry_fwd"],
    "quantile": ["qsketch_merge"],
}
IN_ROUNDS_AT_1MB = ("ordered_join", "asof_strategy")         # suites whose larger exchanges go in rounds with 1 MB mailboxes
