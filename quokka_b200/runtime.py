"""In-process, push-based driver: the part of the reference runtime that sits between operators --
TaskGraph construction (pyquokka/quokka_runtime.py:118-394), the two worker loops
(IOTaskManager.execute / ExecTaskManager.execute, pyquokka/core.py:484-965) and the shuffle
(TaskManager.push + the Flight mailbox, core.py:276-376, flight.py:44-264) -- re-thought for one process per
GPU (SPMD over torch.distributed):

  * every rank builds the same graph; an actor has one channel per rank (or a single channel on rank 0);
  * a produced batch is pushed through each outgoing edge (partition_fn), exchanged with an all-to-all of
    the partitioned column buffers (NCCL over NVLink; gloo on CPU for tests) and handed to the consumer's
    `execute` immediately -- partitions are consumed as they arrive, there is no global barrier between
    operators, only the stage rule "every build input before the first probe batch" (df.py:1558-1568);
  * empty partitions still take part in the exchange (the reference's `__empty__` sentinel,
    core.py:333-335) so all ranks issue the same sequence of collectives.

Fault tolerance (lineage, HBQ spill, Redis tables, the coordinator) is out of scope: SURVEY.md section 8.
"""
from __future__ import annotations

import copy
import os
import pickle
import threading
import zlib

import torch
import torch.distributed as dist

from . import _lib as L
from . import ops
from .columns import DeviceColumn, DeviceTable, as_device_table, concat_tables, rank, unify_dictionaries, world_size
from .edge import Parts, partition_fn
from .placement_strategy import CustomChannelsStrategy, SingleChannelStrategy
from .target_info import BroadcastPartitioner, PassThroughPartitioner, TargetInfo


def _default_device():
    from . import columns
    return columns.default_device()


# ------------------------------------------------------------------ the shuffle
_DT = {"torch.uint8": torch.uint8, "torch.int32": torch.int32, "torch.int64": torch.int64,
       "torch.float32": torch.float32, "torch.float64": torch.float64, "torch.float16": torch.float16}
_VALID_FLAG, _WIDTH_MASK = 1 << 32, (1 << 32) - 1     # meta word of a column: row bytes | _VALID_FLAG when it has a mask


def _col_dt(t: torch.Tensor) -> str:
    """Schema string of a column buffer: the dtype, and the row width of a vector column ("torch.float32[768]")."""
    return str(t.dtype) if t.dim() == 1 else f"{t.dtype}[{t.shape[1]}]"


def _parse_dt(dt: str):
    """(torch dtype, lanes) of a schema string; lanes = 0 for a scalar column."""
    base, _, lanes = dt.partition("[")
    return _DT[base], (int(lanes[:-1]) if lanes else 0)


def _row_bytes(dt: str) -> int:
    t, lanes = _parse_dt(dt)
    return t.itemsize * max(1, lanes)


def _empty(n: int, dt: str, device) -> torch.Tensor:
    t, lanes = _parse_dt(dt)
    return torch.empty((n, lanes) if lanes else n, dtype=t, device=device)


def _flat(t: torch.Tensor) -> torch.Tensor:
    """A dense buffer: 1-D for a scalar column, (n, d) row-major for a vector column (a one-row slice of a 2-D state keeps its
    row stride and reports is_contiguous())."""
    if t.dim() == 1 and (t.numel() == 0 or t.stride(0) == 1):
        return t
    if t.dim() == 2:
        return t.contiguous()
    out = torch.empty(t.numel(), dtype=t.dtype, device=t.device)      # fresh storage: unit stride guaranteed
    out.copy_(t.reshape(-1))
    return out


def _checksum(schema) -> int:
    return (zlib.crc32(repr(schema).encode()) | 1) if schema is not None else 0


class NativeLink:
    """The process-wide symmetric allocation behind the peer-memory shuffle (csrc/exchange.cu): `nchannels` channels,
    each a control block + a mailbox.  Every rank's allocation is mapped into every other rank's address space (CUDA IPC
    / fabric handles through torch symmetric memory), so a producer's kernels store rows straight into the consumers' HBM.
    Channel 0 belongs to the driver thread, channel 1 + i to pipeline lane i, so that chunks in flight on different CUDA
    streams never share flags or mailbox space and every channel sees the same sequence of exchanges on every rank."""

    CTRL = L.XCHG_CTRL_BYTES

    def __init__(self, device, nchannels: int, mailbox_bytes: int):
        import torch.distributed._symmetric_memory as symm
        mailbox_bytes = (int(mailbox_bytes) + 4095) // 4096 * 4096
        head = (nchannels * self.CTRL + 65535) // 65536 * 65536
        self.buf = symm.empty(head + nchannels * mailbox_bytes, dtype=torch.uint8, device=device)
        self.hdl = symm.rendezvous(self.buf, dist.group.WORLD)
        ptrs = [int(p) for p in self.hdl.buffer_ptrs]
        self.buf[:head].zero_()
        torch.cuda.synchronize(device)
        self.hdl.barrier(channel=0)                          # every control block is zero before anybody posts
        torch.cuda.synchronize(device)
        w, me = world_size(), rank()
        tmo = int(float(os.environ.get("QK_XCHG_TIMEOUT_S", "120")) * 1000)     # a rank may lag by a first-touch allocation of tens of GB
        self.channels = [ops.XchgChannel(w, me, [p + i * self.CTRL for p in ptrs],
                                         [p + head + i * mailbox_bytes for p in ptrs], mailbox_bytes, device, tmo)
                         for i in range(nchannels)]
        self.mailbox_bytes = mailbox_bytes


_lane_streams = {}                   # device index -> the lanes' CUDA streams (process-wide: their allocator pools stay warm)


def lane_streams(device):
    key = device.index if device.index is not None else torch.cuda.current_device()
    if key not in _lane_streams:
        _lane_streams[key] = [torch.cuda.Stream(device) for _ in range(N_LANES)]
    return _lane_streams[key]


_link = {"obj": None, "failed": False}
_lane = threading.local()            # .index: pipeline lane of the calling thread (absent = the driver thread)
N_LANES = max(1, int(os.environ.get("QK_LANES", "2")))


def lane_channel() -> int:
    return 1 + getattr(_lane, "index", -1)


def native_link(device):
    """The peer-memory link, or None (no CUDA / single rank / gloo / QK_P2P=0 / symmetric memory unavailable).  Creating
    it is a collective; all ranks agree on the outcome (a rank-local failure makes every rank fall back to NCCL)."""
    if _link["failed"] or device.type != "cuda" or world_size() == 1 or os.environ.get("QK_P2P", "1") == "0":
        return None
    if dist.get_backend() != "nccl":
        return None
    if _link["obj"] is None:
        ok, err = 1, None
        try:
            obj = NativeLink(device, 1 + N_LANES, int(float(os.environ.get("QK_MAILBOX_MB", "2048")) * (1 << 20)))
        except Exception as e:                                   # no P2P / fabric support on this box, or out of memory
            ok, err, obj = 0, e, None
        flag = torch.tensor([ok], device=device, dtype=torch.int32)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN)
        if int(flag.item()) == 0:
            _link["failed"] = True
            if rank() == 0:
                print(f"[quokka_b200] peer-memory shuffle unavailable ({type(err).__name__ if err else 'a peer failed'}: {err}); using NCCL all-to-all", flush=True)
            return None
        _link["obj"] = obj
    return _link["obj"]


# ------------------------------------------------------------------ the exchange protocol, shared by both transports
class _SendPlan:
    """Which rows this rank sends where: rows [lo[d], hi[d]) of `table` go to rank d (a broadcast names the same rows for
    every rank), or -- `dest` set -- `table` is a hash partition not yet materialised: row i has position dest[i] in the
    partition order, and `doffs` (device int64[world + 1]) holds where each destination's rows start."""

    def __init__(self, parts, single_owner, w: int):
        self.table = self.dest = self.doffs = None
        self.lo, self.hi = [0] * w, [0] * w
        if isinstance(parts, Parts):
            if single_owner is None and parts.pending is not None and parts.doffs.numel() == w + 1:
                if len(parts.pending[0]) > 0:
                    self.table, self.dest, self.doffs = parts.pending
            else:
                t = parts.table
                if t is not None and len(t) > 0:
                    self.table = t
                    if single_owner is not None:
                        self.hi[single_owner] = len(t)
                    else:
                        offs = parts.offsets
                        for d in range(min(w, len(offs) - 1)):
                            self.lo[d], self.hi[d] = offs[d], offs[d + 1]
        else:
            owner = (lambda c_: single_owner) if single_owner is not None else (lambda c_: c_)
            by_rank = {}
            for c_, p_ in sorted(parts.items()):
                if p_ is not None and len(p_) > 0:
                    by_rank.setdefault(owner(c_), []).append(p_)
            flat = [p_ for r in sorted(by_rank) for p_ in by_rank[r]]
            if flat and all(p_ is flat[0] for p_ in flat) and all(len(v) == 1 for v in by_rank.values()):
                self.table = flat[0]                              # broadcast / single owner: the same rows to every destination
                for r in by_rank:
                    self.hi[r] = len(self.table)
            elif flat:
                self.table = concat_tables(flat)
                pos = 0
                for r in sorted(by_rank):
                    self.lo[r] = pos
                    pos = self.hi[r] = pos + sum(len(p_) for p_ in by_rank[r])
        self.schema = Exchange._schema_of(self.table) if self.table is not None else None

    @property
    def counts(self) -> list:
        """Rows for each destination (zeros for an unmaterialised hash partition: its counts are on the device)."""
        return [h - l for l, h in zip(self.lo, self.hi)]


class _Meta:
    """Every rank's meta row, in one layout for both transports: rows for each destination rank in words [0, w), then
    from word `head` the header: the checksum of the sender's schema (0: no table), the checksum of the schema it has
    cached for the edge, the column count and every column's row bytes | _VALID_FLAG when it has a validity mask.  On the
    link `head` is 16 (qk_xchg_meta may overwrite words [0, w) with the device counts, and the link takes at most
    QK_MAX_PEERS = 16 ranks); the collective path puts the header after max(16, w) counts."""

    HASH, CACHED, NCOLS, WIDTHS = 0, 1, 2, 4
    MAXC = L.XCHG_MAX_BUFS // 2      # columns of an edge: with a validity mask each, one push of QK_XCHG_MAX_BUFS buffers

    @classmethod
    def row(cls, counts: list, mine, cached, head: int) -> list:
        if mine is not None and len(mine) > cls.MAXC:
            raise L.QkError(f"exchange: more than {cls.MAXC} columns on one edge")
        words = [0] * (head + cls.WIDTHS + cls.MAXC)
        words[:len(counts)] = counts
        words[head + cls.HASH], words[head + cls.CACHED] = _checksum(mine), _checksum(cached)
        for i, (_, dt, _, _, hv) in enumerate(mine or []):
            words[head + cls.WIDTHS + i] = _row_bytes(dt) | (_VALID_FLAG if hv else 0)
        words[head + cls.NCOLS] = len(mine or [])
        return words

    def __init__(self, m, w: int, head: int):
        """m: everybody's row, an integer array [world][words]."""
        self.counts = m[:, :w]                                    # counts[s][d]: rows rank s sends to rank d
        self.total = int(self.counts.sum())
        self.n_recv = [int(self.counts[:, d].sum()) for d in range(w)]
        self.hash = [int(x) for x in m[:, head + self.HASH]]
        self.cached = [int(x) for x in m[:, head + self.CACHED]]
        src = next((r for r in range(w) if int(m[r, head + self.NCOLS]) > 0), None)      # a rank that has a table
        ncols = int(m[src, head + self.NCOLS]) if src is not None else 0
        flags = m[:, head + self.WIDTHS: head + self.WIDTHS + ncols]
        self.col_valid = [bool((flags[:, i] & _VALID_FLAG).any()) for i in range(ncols)]
        # validity masks travel as extra uint8 columns after the data columns
        self.widths = [int(flags[src, i]) & _WIDTH_MASK for i in range(ncols)] + [1 for v in self.col_valid if v]

    def sent_bytes(self, me: int) -> int:
        """Bytes rank `me` sends to other ranks."""
        return (int(self.counts[me].sum()) - int(self.counts[me, me])) * sum(self.widths)


def _recode(c: DeviceColumn, union) -> DeviceColumn:
    """`c` with its codes re-mapped onto the agreed union dictionary."""
    if union is None or c.dictionary == union:
        return c
    return unify_dictionaries([DeviceColumn(torch.zeros(0, dtype=c.data.dtype, device=c.data.device), union, c.arrow_type), c])[1][1]


def _send_columns(table: DeviceTable, schema, col_valid) -> list:
    """The buffers that cross ranks, one per width of the meta: the columns of `table` in schema order, re-coded onto the
    agreed dictionaries, then the validity mask of every column that has one on any rank (all ones where this rank's
    column has none)."""
    cols, masks = [], []
    for (name, _, union, _, _), v in zip(schema, col_valid):
        c = _recode(table[name], union)
        cols.append(_flat(c.data))
        if v:
            masks.append(c.valid if c.valid is not None else torch.ones(len(c), dtype=torch.uint8, device=c.data.device))
    return cols + masks


def _recv_buffers(n: int, schema, col_valid, device) -> list:
    return [_empty(n, dt, device) for _, dt, _, _, _ in schema] + [torch.empty(n, dtype=torch.uint8, device=device) for v in col_valid if v]


def _split(outs: list, schema, col_valid, rows_from) -> list:
    """The received buffers (in _send_columns order; the rows of rank s after those of ranks < s, rows_from[s] of them)
    as one DeviceTable per source rank that sent rows."""
    masks = iter(outs[len(schema):])
    valid = [next(masks) if v else None for v in col_valid]
    tables, r0 = [], 0
    for s_, n in enumerate(rows_from):
        r1 = r0 + int(n)
        if r1 > r0:
            t = DeviceTable({name: DeviceColumn(o[r0:r1], union, atype, None if v is None else v[r0:r1])
                             for (name, _, union, atype, _), o, v in zip(schema, outs, valid)})
            t.src_rank = s_              # ordered consumers put the ranks' time ranges back in order with this
            tables.append(t)
        r0 = r1
    return tables


class Exchange:
    """All-to-all of partitioned column buffers (the reference's push -> Flight do_put / do_get,
    core.py:276-376, flight.py:44-264), over one of two transports:

      * the peer-memory link (csrc/exchange.cu, `native_link`): one meta round, then every rank stores its rows straight
        into the receivers' mailboxes -- one host round trip per exchange, no library collective;
      * torch.distributed (gloo on CPU; NCCL when there is no link): an all-gather of the meta rows, then one
        variable-split all_to_all_single per column.

    Both speak one protocol: every rank posts a meta row (`_Meta`: rows per destination, schema checksums, column widths);
    column names / dtypes / dictionaries travel (pickled) only when an edge is first used or a dictionary changes
    (`_agree`); dictionary columns are re-coded onto the union dictionary and validity masks travel as extra uint8
    columns (`_send_columns`); a receiver gets one table per source rank that sent rows (`_split`)."""

    def __init__(self, device):
        self.device = device
        self.bytes_sent = 0        # payload bytes this rank sent to other ranks, validity masks included
        self.calls = 0
        self.peer_calls = 0        # exchanges (and rounds of one) that moved their rows over the link
        self.schemas = {}          # edge key -> [(name, dtype str, dictionary, arrow type, has_valid)]
        self.recv_totals = {}      # edge key -> rows every rank has RECEIVED on that edge so far (known to all ranks from the counts)

    @staticmethod
    def _schema_of(t: DeviceTable):
        return [(n, _col_dt(c.data), c.dictionary, c.arrow_type, c.valid is not None) for n, c in t.columns.items()]

    def allgather_words(self, words: list) -> list:
        """[[words of rank 0], [words of rank 1], ...]: a handful of integers from every rank.  On the peer-memory link
        this is one meta round (one tiny kernel + one host wait); otherwise an all-gather."""
        w = world_size()
        if w == 1:
            return [list(words)]
        link = native_link(self.device)
        if link is not None:
            m = link.channels[lane_channel()].meta([0] * L.MAX_PEERS + [int(x) for x in words])
            return [[int(x) for x in m[r, L.MAX_PEERS:L.MAX_PEERS + len(words)]] for r in range(w)]
        t = torch.tensor([int(x) for x in words], dtype=torch.int64, device=self.device)
        out = torch.empty(w * len(words), dtype=torch.int64, device=self.device)
        dist.all_gather_into_tensor(out, t)
        return out.cpu().view(w, len(words)).tolist()

    def max_over_ranks(self, words: list) -> list:
        """The element-wise maximum of `words` over all ranks (one allgather_words)."""
        return [max(col) for col in zip(*self.allgather_words(words))]

    def __call__(self, parts, n_target: int, single_owner: int | None = None, edge_key=None) -> list:
        """parts: {target_channel: DeviceTable} or edge.Parts.  Target channel c lives on rank c (or on
        `single_owner` when the consumer has a single channel).  Returns the tables received by this rank,
        one per source rank that sent rows, in source-rank order (`src_rank` on each, at more than one rank) on both
        transports -- a payload that goes in rounds too, a source's rounds one after the other.  Callers rely on that order
        and do not sort."""
        if world_size() == 1:
            if isinstance(parts, Parts):
                return parts.tables()
            return [p for _, p in sorted(parts.items()) if p is not None and len(p) > 0]
        link = native_link(self.device)
        if link is not None:
            return self._native_call(link, parts, single_owner, edge_key)
        return self._collective_call(parts, single_owner, edge_key)

    def to_ranks(self, table, edge_key, ranks=None) -> list:
        """`table` (None or empty: nothing) to every rank in `ranks` (default: all of them, this one included).  Returns the
        tables this rank received in source-rank order, each with its `src_rank`, at one rank too."""
        w = world_size()
        send = table is not None and len(table) > 0
        got = self({r: table for r in (range(w) if ranks is None else ranks)} if send else {}, w, edge_key=edge_key)
        if w == 1:                           # the table itself came back: the caller gets a view that names its source
            got = [DeviceTable(g.columns) for g in got]
            for g in got:
                g.src_rank = 0
        return got

    def hand_off(self, table, bounds, edge_key) -> list:
        """Rows [bounds[r], bounds[r + 1]) of `table` (None or empty: nothing) to rank r.  This rank's own slice stays where
        it is, without a trip through the mailbox.  Returns the own and received slices in source-rank order, each with its
        `src_rank`."""
        w, me = world_size(), rank()
        parts, own = {}, None
        if table is not None and len(table) > 0:
            parts = {r: table.slice(bounds[r], bounds[r + 1]) for r in range(w) if r != me and bounds[r + 1] > bounds[r]}
            own = table.slice(bounds[me], bounds[me + 1])
        got = self(parts, w, edge_key=edge_key)
        if own is None or len(own) == 0:
            return got
        own.src_rank = me
        return [g for g in got if g.src_rank < me] + [own] + [g for g in got if g.src_rank > me]

    # ------------------------------------------------------------------ what both transports do with the meta rows
    def _count_received(self, edge_key, counts):
        if edge_key is not None:
            tot = self.recv_totals.setdefault(edge_key, [0] * counts.shape[1])
            for d in range(len(tot)):
                tot[d] += int(counts[:, d].sum())

    def _agree(self, m: _Meta, mine, cached, edge_key, share) -> list | None:
        """The schema the rows are sent and decoded with (None: this rank neither sends nor receives).  Every rank
        published a checksum of its table's schema and of the schema it has cached for this edge; the schemas themselves
        travel -- `share(obj)` returns every rank's object -- only when the checksums disagree (a dictionary grew) or when
        a rank that will RECEIVE rows has neither a table nor a matching cached schema.  Dictionaries are merged into
        their sorted union."""
        hashes = set(h for h in m.hash if h != 0)
        negotiate = len(hashes) != 1
        if not negotiate:
            common = next(iter(hashes))
            negotiate = any(m.hash[r] == 0 and m.n_recv[r] > 0 and m.cached[r] != common for r in range(len(m.hash)))
        if negotiate:
            known = [h for h in share(mine) if h is not None]
            schema = []
            for i, (name, dt, _, atype, _) in enumerate(known[0]):
                dicts = [h[i][2] for h in known if h[i][2] is not None]
                union = sorted(set().union(*[set(d_) for d_ in dicts])) if dicts else None
                schema.append((name, dt, union, atype, any(h[i][4] for h in known)))
        else:
            schema = mine if mine is not None else (cached if _checksum(cached) == common else None)
        if edge_key is not None and schema is not None:
            self.schemas[edge_key] = schema
        return schema

    # ------------------------------------------------------------------ transport 1: the peer-memory link (csrc/exchange.cu)
    def _share_objects(self, ch, obj):
        """Every rank's `obj` (pickled) to every rank over the link: used only when schemas disagree."""
        w, me = ch.world, ch.rank
        blob = pickle.dumps(obj)
        buf = torch.frombuffer(bytearray(blob), dtype=torch.uint8).to(self.device)
        m = ch.meta([len(blob)] * w)
        sizes = [int(m[s_, 0]) for s_ in range(w)]
        if sum(sizes) > ch.mailbox_bytes:
            raise L.QkError("exchange: schema negotiation does not fit the mailbox")
        off = [sum(sizes[:s_]) for s_ in range(w)]
        ch.push([buf], [0] * w, [len(blob)] * w, [[off[me]] for _ in range(w)])
        out = torch.empty(sum(sizes), dtype=torch.uint8, device=self.device)
        ch.recv([0], [out])
        host = out.cpu().numpy().tobytes()
        ch.meta([0])        # the objects used this channel's epoch and mailbox: the payload gets a fresh epoch (and the barrier)
        return [pickle.loads(host[off[s_]:off[s_] + sizes[s_]]) for s_ in range(w)]

    def _native_call(self, link, parts, single_owner, edge_key) -> list:
        """One exchange over the link.  Host round trips: ONE (the meta matrix); collectives: none.  A hash partition's
        counts go into the meta row from the device (qk_xchg_meta) and its rows are scattered while they are sent."""
        ch = link.channels[lane_channel()]
        w, me = ch.world, ch.rank
        plan = _SendPlan(parts, single_owner, w)
        self.calls += 1
        cached = self.schemas.get(edge_key)
        m = _Meta(ch.meta(_Meta.row(plan.counts, plan.schema, cached, L.MAX_PEERS), plan.doffs), w, L.MAX_PEERS)
        self._count_received(edge_key, m.counts)
        if m.total == 0:
            return []
        schema = self._agree(m, plan.schema, cached, edge_key, lambda obj: self._share_objects(ch, obj))
        bases = []                                                       # bases[d][c]: column c in rank d's mailbox
        for d in range(w):
            row, off = [], 0
            for wd in m.widths:
                row.append(off)
                off += (m.n_recv[d] * wd + 255) // 256 * 256
            bases.append(row)
            if off > ch.mailbox_bytes:
                self._count_received(edge_key, -m.counts)                # the rounds count their own rows
                return self._native_oversize(link, plan, edge_key, off, ch.mailbox_bytes)
        if len(m.widths) > L.XCHG_MAX_BUFS:
            raise L.QkError(f"exchange: {len(m.widths)} buffers on one edge (columns + validity masks); the link moves at most "
                            f"{L.XCHG_MAX_BUFS} in one push")
        send = _send_columns(plan.table, schema, m.col_valid) if plan.table is not None else []
        row_off = [int(m.counts[:me, d].sum()) for d in range(w)]
        dst_off = [[bases[d][c] + row_off[d] * m.widths[c] for c in range(len(send))] for d in range(w)]
        if plan.dest is not None:
            ch.push_scatter(send, plan.dest, plan.doffs, dst_off)
        else:
            ch.push(send, plan.lo, plan.hi, dst_off)
        self.peer_calls += 1
        self.bytes_sent += m.sent_bytes(me)
        if m.n_recv[me] == 0 or schema is None:
            ch.recv([], [])
            return []
        outs = _recv_buffers(m.n_recv[me], schema, m.col_valid, self.device)
        ch.recv(bases[me], outs)
        return _split(outs, schema, m.col_valid, m.counts[:, me])

    def _native_oversize(self, link, plan: _SendPlan, edge_key, need, have) -> list:
        """Somebody's share does not fit its mailbox (every rank sees that in the same meta matrix): the rows go in R
        rounds, each a complete exchange of a slice of every sender's rows.  Returns what one exchange returns: the tables
        per source rank in rank order, each source's in round order (consumers fed through the graph depend on it)."""
        R = -(-int(need) // int(have)) * 2
        out = []
        w = len(plan.lo)
        if plan.dest is not None:
            # an unmaterialised hash partition: every round is the fused scatter push of a slice of the INPUT rows; the
            # slice's own plan comes from the destinations the full plan already assigned (no local scatter, no copy)
            n = len(plan.table)
            inner = plan.doffs[1:w].contiguous()
            for r in range(R):
                a, b = n * r // R, n * (r + 1) // R
                if b > a:
                    which = torch.bucketize(plan.dest[a:b].long(), inner, right=True).to(torch.int32)
                    d_r, o_r = ops.partition_plan(which, w, L.PART_CODE)
                    sub = Parts(None, None, (plan.table.slice(a, b), d_r, o_r))
                else:
                    sub = {}
                out += self._native_call(link, sub, None, edge_key)
            return sorted(out, key=lambda t: t.src_rank)          # stable: rounds stay in order within a source
        for r in range(R):
            sub = {}
            if plan.table is not None:
                for d in range(w):
                    n_d = plan.hi[d] - plan.lo[d]
                    a, b = plan.lo[d] + n_d * r // R, plan.lo[d] + n_d * (r + 1) // R
                    if b > a:
                        sub[d] = plan.table.slice(a, b)
            out += self._native_call(link, sub, None, edge_key)
        return sorted(out, key=lambda t: t.src_rank)

    # ------------------------------------------------------------------ transport 2: torch.distributed collectives
    @staticmethod
    def _gather_objects(obj):
        out = [None] * world_size()
        dist.all_gather_object(out, obj)
        return out

    def _collective_call(self, parts, single_owner, edge_key) -> list:
        """One exchange over torch.distributed: an all-gather of the meta rows, then one variable-split all_to_all_single
        per column, which takes each destination's rows as one contiguous run of the send buffer, in rank order."""
        w, me = world_size(), rank()
        plan = _SendPlan(parts, single_owner, w)
        self.calls += 1
        counts = plan.counts
        if plan.dest is not None:
            offs = plan.doffs.cpu().tolist()
            counts = [offs[d + 1] - offs[d] for d in range(w)]
        head = max(L.MAX_PEERS, w)
        cached = self.schemas.get(edge_key)
        row = torch.tensor(_Meta.row(counts, plan.schema, cached, head), dtype=torch.int64, device=self.device)
        allm = torch.empty(w * row.numel(), dtype=torch.int64, device=self.device)
        dist.all_gather_into_tensor(allm, row)
        m = _Meta(allm.cpu().view(w, -1).numpy(), w, head)
        self._count_received(edge_key, m.counts)
        if m.total == 0:
            return []
        schema = self._agree(m, plan.schema, cached, edge_key, self._gather_objects)
        nothing = torch.empty(0, dtype=torch.uint8, device=self.device)
        send = [nothing] * len(m.widths)
        if plan.table is not None:
            send = _send_columns(plan.table, schema, m.col_valid)
            if plan.dest is not None:                            # the hash partition, grouped locally
                send = ops.scatter(send, plan.dest)
            elif any(n and lo != sum(counts[:d]) for d, (lo, n) in enumerate(zip(plan.lo, counts))):
                send = [torch.cat([c[lo:hi] for lo, hi in zip(plan.lo, plan.hi)]) for c in send]     # a broadcast: one copy per rank
            else:
                send = [c[:sum(counts)] for c in send]
        n_recv = m.n_recv[me]
        recv = _recv_buffers(n_recv, schema, m.col_valid, self.device) if schema is not None else [nothing] * len(m.widths)
        recv_counts = [int(x) for x in m.counts[:, me]]
        for s_b, r_b, wd in zip(send, recv, m.widths):
            dist.all_to_all_single(r_b.reshape(-1).view(torch.uint8), s_b.reshape(-1).view(torch.uint8),
                                   [c_ * wd for c_ in recv_counts], [c_ * wd for c_ in counts])
        self.bytes_sent += m.sent_bytes(me)
        if n_recv == 0 or schema is None:
            return []
        return _split(recv, schema, m.col_valid, recv_counts)


# ------------------------------------------------------------------ the graph
def _takes_device_tables(executor) -> bool:
    """The Executor protocol hands `execute` a list of pyarrow.Table (pyquokka/executors/base_executor.py:26-32,
    core.py:624-632).  The executors of this package take the device-resident batches directly; any other class (a
    user's plug-in, written against the reference) gets Arrow tables on the host unless it opts in with
    `device_tables = True`.  Either kind may return a DeviceTable, a pyarrow.Table, a pandas frame or None."""
    flag = getattr(executor, "device_tables", None)
    return bool(flag) if flag is not None else type(executor).__module__.startswith("quokka_b200.")


class _Actor:
    def __init__(self, aid, kind, obj, stage, single):
        self.id, self.kind, self.obj, self.stage, self.single = aid, kind, obj, stage, single
        self.targets = []          # (target actor id, stream_id, TargetInfo)
        self.sources = {}          # stream_id -> source actor id
        self.blocking = False
        self.done = False
        self.instance = None       # this rank's executor instance (one per (actor, channel): core.py:526-527)
        self.results = []
        self.ordered = False
        self.lock = threading.Lock()   # one execute() at a time per executor instance (core.py:493), whatever the lane
        self.tail = None               # CUDA event after the last execute(): the next caller's stream waits for it


class TaskGraph:
    """Same construction calls as the reference's TaskGraph (quokka_runtime.py:118,314,370,383,394)."""

    def __init__(self, context=None) -> None:
        self.context = context
        self.actors: dict[int, _Actor] = {}
        self.current_actor = 0
        self.device = getattr(context, "device", None) or _default_device()
        self.exchange = Exchange(self.device)
        self.profile = bool(os.environ.get("QK_PROFILE"))      # like the reference's PROFILE flag (core.py:20-30)
        self.timings = {}
        self._bind_lock = threading.Lock()
        self._lane_streams = None
        self.lanes_used = 0

    def _timed(self, label, fn, *a, **kw):
        if not self.profile:
            return fn(*a, **kw)
        import time
        if self.device.type == "cuda":
            torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn(*a, **kw)
        if self.device.type == "cuda":
            torch.cuda.synchronize()
        self.timings[label] = self.timings.get(label, 0.0) + (time.perf_counter() - t0)
        return out

    def report(self):
        return {k: round(v * 1e3, 3) for k, v in sorted(self.timings.items(), key=lambda kv: -kv[1])}

    # -- construction
    def new_input_reader_node(self, reader, stage=0, placement_strategy=None):
        a = _Actor(self.current_actor, "input", reader, stage, False)
        a.ordered = hasattr(reader, "sorted_by")
        self.actors[a.id] = a
        self.current_actor += 1
        return a.id

    def _new_exec(self, streams, functionObject, stage, placement_strategy, source_target_info, blocking):
        single = isinstance(placement_strategy, SingleChannelStrategy)
        a = _Actor(self.current_actor, "exec", functionObject, stage, single)
        a.blocking = blocking
        a.ordered = bool(getattr(functionObject, "ordered_output", False))     # a sort: rank r's output precedes rank r + 1's
        for stream_id, src in streams.items():
            ti = source_target_info.get(stream_id) if source_target_info else None
            if ti is None:
                ti = TargetInfo(PassThroughPartitioner(), None, None, [])
            a.sources[stream_id] = src
            self.actors[src].targets.append((a.id, stream_id, ti))
        self.actors[a.id] = a
        self.current_actor += 1
        return a.id

    def new_non_blocking_node(self, streams, functionObject, stage=0, placement_strategy=CustomChannelsStrategy(1),
                              source_target_info={}, assume_sorted={}):
        return self._new_exec(streams, functionObject, stage, placement_strategy, source_target_info, False)

    def new_blocking_node(self, streams, functionObject, stage=0, placement_strategy=CustomChannelsStrategy(1),
                          source_target_info={}, transform_fn=None, assume_sorted={}):
        return self._new_exec(streams, functionObject, stage, placement_strategy, source_target_info, True)

    def create(self):
        for a in self.actors.values():
            if a.kind == "exec":
                a.instance = copy.deepcopy(a.obj)
            else:
                a.obj.device = self.device
                if self.context is not None and getattr(a.obj, "dictionaries", None) is None:
                    a.obj.dictionaries = self.context.dictionaries
        return self

    # -- execution
    def _owns(self, actor: _Actor) -> bool:
        return (not actor.single) or rank() == 0

    def _push(self, actor: _Actor, table):
        for tgt_id, stream_id, ti in actor.targets:
            tgt = self.actors[tgt_id]
            n = 1 if tgt.single else world_size()
            if table is not None and len(table.columns) > 0:
                with self._bind_lock:
                    ti.bind(table.column_names)
                parts = self._timed(f"edge {actor.id}->{tgt_id} partition_fn", partition_fn, ti, table, rank(), n)
            else:
                parts = {}
            if n > 1 and isinstance(ti.partitioner, PassThroughPartitioner) and isinstance(parts, dict):
                # channel c feeds channel c: nothing crosses ranks, and every rank knows that from the plan alone, so
                # the whole exchange (metadata all-gather, host sync, all-to-all) is skipped -- by all ranks alike
                received = [p for _, p in sorted(parts.items()) if p is not None and len(p) > 0]
            else:
                received = self._timed(f"edge {actor.id}->{tgt_id} exchange", self.exchange, parts, n,
                                       single_owner=0 if tgt.single else None, edge_key=(actor.id, tgt_id, stream_id))
            out = None
            if self._owns(tgt) and received:
                if not _takes_device_tables(tgt.instance):      # a user's Executor: the reference protocol, list[pyarrow.Table]
                    received = [b.to_arrow() for b in received]
                with tgt.lock:
                    cuda = self.device.type == "cuda"
                    if cuda and tgt.tail is not None:           # state last touched on another lane's stream
                        torch.cuda.current_stream().wait_event(tgt.tail)
                    out = self._timed(f"actor {tgt_id} {type(tgt.instance).__name__}.execute[{stream_id}]", tgt.instance.execute, received, stream_id, rank())
                    out = as_device_table(out) if out is not None else None
                    if cuda:
                        tgt.tail = torch.cuda.Event()
                        tgt.tail.record()
            # An executor whose execute() never returns rows for this stream (the build side of a join, an aggregate that
            # answers in done(): `silent_streams` on the class, the same on every rank) sends nothing downstream: no rank
            # starts the (empty) exchanges a None would otherwise cascade through -- one meta round trip each at > 1 rank
            quiet = _is_silent(tgt.instance, stream_id)
            if quiet and out is not None and len(out) > 0:
                raise L.QkError(f"{type(tgt.instance).__name__}.execute returned rows on stream {stream_id}, which it declares silent")
            self._emit(tgt, out, quiet)

    def _emit(self, actor: _Actor, out, quiet: bool = False):
        if actor.blocking:
            if out is not None and len(out) > 0:
                actor.results.append(out)
        elif not quiet:
            self._push(actor, out)

    def _publish_bloom(self, actor: _Actor):
        """`actor` just delivered the last build batch of every join it feeds on stream 1: where the planner
        asked for it, build the Bloom filter of each channel's build keys, all-gather the filters and hand them
        to the probe edge, so the probe-side scan drops non-joining rows BEFORE they are partitioned and sent."""
        for tgt_id, stream_id, edge in actor.targets:
            tgt = self.actors[tgt_id]
            if stream_id != 1 or not hasattr(tgt.instance, "make_bloom") or tgt.single:
                continue
            replicated = isinstance(edge.partitioner, BroadcastPartitioner)     # every rank holds ALL build keys
            sinks = [ti for a in self.actors.values() for _, _, ti in a.targets
                     if ti.bloom_key is not None and ti.bloom_source == tgt_id]
            if not sinks:
                continue
            w, me = world_size(), rank()
            n_local = tgt.instance.build_rows()
            no_filter = 0 if tgt.instance.bloom_ok() else 1      # string keys: codes of unrelated dictionaries
            if w > 1:
                ekey = (actor.id, tgt_id, stream_id)
                tot, sch = self.exchange.recv_totals.get(ekey), self.exchange.schemas.get(ekey)
                if tot is not None and (sch is not None or sum(tot) == 0) and native_link(self.device) is not None:
                    # every rank already knows how many build rows every rank holds (the exchanges' count matrices) and
                    # whether the key is a string column (the agreed schema): no extra agreement round
                    n_local = max(tot)
                    right = getattr(tgt.instance, "right_on", None)
                    # (string keys: codes of unrelated dictionaries; fp64 keys are matched on their bit pattern, not filtered)
                    no_filter = 1 if (sch is not None and any(name == right and (dic is not None or "float" in dt) for name, dt, dic, _, _ in sch)) else 0
                else:
                    n_local, no_filter = self.exchange.max_over_ranks([n_local, no_filter])
            if no_filter:
                continue
            words = ops.Bloom.words_for(-(-n_local // w) if replicated else n_local)
            local = self._timed(f"actor {tgt_id} bloom build", tgt.instance.make_bloom, words, w)
            bits = local.bits
            if w > 1 and not replicated:            # a replicated build side yields the complete filter on every rank
                mine = bits[me * words:(me + 1) * words].contiguous()
                if native_link(self.device) is not None:     # my slice to every rank over the peer-memory link
                    got = self.exchange.to_ranks(DeviceTable({"bits": DeviceColumn(mine)}), ("bloom", tgt_id))
                    bits = torch.cat([g["bits"].data for g in got]) if len(got) > 1 else got[0]["bits"].data
                else:
                    allbits = torch.empty(w * words, dtype=bits.dtype, device=self.device)
                    dist.all_gather_into_tensor(allbits, mine)
                    bits = allbits
            for ti in sinks:
                ti.bloom = ops.Bloom(bits, words, w)

    def _publish_left_template(self, actor: _Actor):
        """`actor` just delivered the last build batch of every join it feeds on stream 1.  A left join's probe rows on a rank
        that owns no build rows still need the build columns' types: every rank sends one of its build rows (if it has one) to
        every rank, and each join keeps the first it receives.  Nothing to do where the build side is replicated (every rank
        holds all of it), at one rank, or for a single-channel join; the decision depends on the plan alone, so all ranks
        take it alike."""
        w = world_size()
        for tgt_id, stream_id, edge in actor.targets:
            tgt = self.actors[tgt_id]
            if (w == 1 or stream_id != 1 or tgt.single or isinstance(edge.partitioner, BroadcastPartitioner)
                    or getattr(tgt.instance, "how", None) != "left" or not hasattr(tgt.instance, "set_left_template")):
                continue
            got = self.exchange.to_ranks(tgt.instance.left_template_row(), ("left-template", tgt_id))
            tgt.instance.set_left_template(got[0] if got else None)

    def _finish(self, actor: _Actor):
        actor.done = True
        self._publish_bloom(actor)
        self._publish_left_template(actor)
        for tgt_id, _, _ in actor.targets:
            tgt = self.actors[tgt_id]
            if tgt.done or not all(self.actors[s].done for s in tgt.sources.values()):
                continue
            out = None
            if self._owns(tgt):
                out = self._timed(f"actor {tgt_id} {type(tgt.instance).__name__}.done", tgt.instance.done, rank())
                out = as_device_table(out) if out is not None else None
            # An executor whose done() never emits (joins, pass-through sinks: `emits_on_done = False` on the class, the
            # same on every rank) sends nothing downstream: no rank starts the exchange for it.
            if out is not None or getattr(tgt.instance, "emits_on_done", True):
                self._emit(tgt, out)
            self._finish(tgt)

    def run(self):
        w, me = world_size(), rank()
        inputs = sorted((a for a in self.actors.values() if a.kind == "input"), key=lambda a: (a.stage, a.id))
        for a in inputs:
            state = a.obj.get_own_state(w)
            if a.ordered and w > 1:
                # ordered stream: batches enter in global order, one source channel after the other
                for ch in sorted(state):
                    for lineage in state[ch]:
                        batch = a.obj.execute(ch, lineage)[1] if ch == me else None
                        self._push(a, as_device_table(batch, self.device) if batch is not None else None)
            else:
                mine = state.get(me, [])
                rounds = len(mine)
                fixed = getattr(a.obj, "fixed_rounds", None)
                if fixed is not None:
                    rounds = fixed                              # the same on every rank by construction: no agreement round
                elif w > 1:
                    rounds = self.exchange.max_over_ranks([rounds])[0]
                if not self._run_laned(a, mine, rounds):
                    for i in range(rounds):
                        batch = a.obj.execute(me, mine[i])[1] if i < len(mine) else None
                        self._push(a, as_device_table(batch, self.device) if batch is not None else None)
            self._finish(a)
        return self

    def _run_laned(self, a: _Actor, mine: list, rounds: int) -> bool:
        """Chunk-pipelined execution of one reader: chunk i runs depth-first through the graph (scan -> partition ->
        exchange -> the consumer's execute -> ... ) on lane i % L, each lane a host thread with its own CUDA stream and
        its own exchange channel.  While one lane waits for the one host round trip of an exchange (or for a row count),
        the other has already enqueued the scan of the next chunk: exchange(i) overlaps scan(i+1) and build / probe(i-1),
        and partitions are consumed as they arrive (the reference pushes batches as produced, core.py:654,946).
        Executors see one execute() at a time (per-actor lock + event chain).  Needs: a reader whose execute() is
        re-entrant (`concurrent`), an unordered stream, and -- across ranks -- the peer-memory link (channels make the
        order of exchanges per lane the same on every rank; library collectives from several threads would not be)."""
        lanes = min(N_LANES, rounds)
        if lanes < 2 or self.device.type != "cuda" or not getattr(a.obj, "concurrent", False) or a.ordered:
            return False
        if world_size() > 1 and native_link(self.device) is None:
            return False
        if self._lane_streams is None:
            self._lane_streams = lane_streams(self.device)
        main = torch.cuda.current_stream()
        me = rank()
        errors = []

        def work(li):
            try:
                torch.cuda.set_device(self.device)
                _lane.index = li
                st = self._lane_streams[li]
                st.wait_stream(main)
                with torch.cuda.stream(st):
                    for i in range(li, rounds, lanes):
                        batch = a.obj.execute(me, mine[i])[1] if i < len(mine) else None
                        self._push(a, as_device_table(batch, self.device) if batch is not None else None)
            except BaseException as e:                          # surfaces on the driver thread
                errors.append(e)

        threads = [threading.Thread(target=work, args=(li,), name=f"qk-lane-{li}") for li in range(lanes)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        for st in self._lane_streams[:lanes]:
            main.wait_stream(st)
        if errors:
            raise errors[0]
        self.lanes_used = max(self.lanes_used, lanes)
        return True

    def results(self, actor_id) -> list:
        return self.actors[actor_id].results

    def describe(self) -> str:
        """The physical plan: actors in execution order with their stage, and every edge with its partitioner,
        predicate, folded batch functions and semi-join (Bloom) reduction."""
        lines = []
        for a in sorted(self.actors.values(), key=lambda a: (a.stage if a.kind == "input" else 1 << 30, a.id)):
            what = type(a.obj).__name__ + (" [single channel]" if a.single else "") + (" [sink]" if a.blocking else "")
            what += " [ordered]" if a.kind == "exec" and a.ordered else ""
            lines.append(f"actor {a.id}: {what}" + (f"  stage {a.stage}" if a.kind == "input" else ""))
            for tgt, sid, ti in a.targets:
                e = ti.edge_ops
                bits = [f"partitioner={ti.partitioner}"]
                if e.pred is not None:
                    bits.append(f"where {e.pred.sql()}")
                if e.defs is not None:
                    bits.append("cols=" + ",".join(n if d.kind == "col" and d.value == n else f"{n}:={d.sql()}" for n, d in e.defs.items()))
                if ti.batch_funcs:
                    bits.append("batch_funcs=" + ",".join(type(f).__name__ if not callable(f) or hasattr(f, "keys") else getattr(f, "__name__", "fn") for f in ti.batch_funcs))
                if ti.bloom_key is not None:
                    bits.append(f"bloom({ti.bloom_key} in build keys of actor {ti.bloom_source})")
                lines.append(f"    -> actor {tgt} stream {sid}: " + "; ".join(bits))
        return "\n".join(lines)


def _is_silent(instance, stream_id) -> bool:
    s = getattr(instance, "silent_streams", ())
    return s == "all" or stream_id in s


def gather_to_all(tables: list, device) -> list:
    """collect(): every rank receives every rank's sink batches (quokka_dataset.py:107-117: the result is
    the unordered concatenation of all sink batches)."""
    return Exchange(device).to_ranks(concat_tables(tables) if tables else None, None)
