"""Tensor-level wrappers over the C-ABI (include/qk.h).  torch is plumbing here: it owns the device
buffers and the stream; every computation below is a libqk.so kernel.  Inputs must be CUDA tensors --
there is no CPU path."""
from __future__ import annotations

import ctypes as C
from typing import Sequence

import torch

from . import _lib as L
from . import expr as E

_TORCH2QK = {torch.uint8: L.QK_U8, torch.bool: L.QK_U8, torch.int32: L.QK_I32, torch.int64: L.QK_I64,
             torch.float32: L.QK_F32, torch.float64: L.QK_F64}
_QK2TORCH = {L.QK_U8: torch.uint8, L.QK_I32: torch.int32, L.QK_I64: torch.int64, L.QK_F32: torch.float32,
             L.QK_F64: torch.float64}


def qk_dtype(t: torch.Tensor) -> int:
    try:
        return _TORCH2QK[t.dtype]
    except KeyError:
        raise L.QkError(f"unsupported column dtype {t.dtype}") from None


def _require_cuda(t: torch.Tensor, what: str):
    if not t.is_cuda:
        raise L.QkError(f"{what}: expected a CUDA tensor (quokka_b200 has no CPU path)")
    if not t.is_contiguous():
        raise L.QkError(f"{what}: column buffers must be contiguous")


def col(t: torch.Tensor, what: str = "column") -> L.qk_column:
    _require_cuda(t, what)
    return L.qk_column(t.data_ptr() if t.numel() else None, None, t.numel(), qk_dtype(t), 0)


def cols(ts: Sequence[torch.Tensor], what: str = "column"):
    arr = (L.qk_column * max(1, len(ts)))()
    for i, t in enumerate(ts):
        arr[i] = col(t, what)
    return arr


def _stream() -> int:
    # the raw handle of torch's current stream: one C call (torch.cuda.current_stream() builds a Stream object through
    # four Python layers -- ~140 of them per Q3 query were 10 % of the driver's host time)
    return torch._C._cuda_getCurrentRawStream(torch._C._cuda_getDevice())


def _ws(nbytes: int, device) -> torch.Tensor:
    return torch.empty(max(int(nbytes), 16), dtype=torch.uint8, device=device)


# ------------------------------------------------------------------ expression programs
Program = Sequence[tuple]      # (op, a0, a1, imm, imm_i)


_SET_BITMAPS: dict = {}      # (device, nbits, bitmap) -> uint32 device words of a QK_OP_IN_SET wider than 64 bits


def _set_bitmap_ptr(nbits: int, bitmap: int, device) -> int:
    """Device copy of a set-membership bitmap (uploaded once per distinct set and kept for the life of the process: the
    programs that point at it are compiled per batch but name the same few dictionary subsets)."""
    key = (str(device), int(nbits), int(bitmap))
    t = _SET_BITMAPS.get(key)
    if t is None:
        nwords = (nbits + 31) // 32
        words = [(bitmap >> (32 * i)) & 0xffffffff for i in range(nwords)]
        t = torch.tensor(words, dtype=torch.int64).to(torch.int32).to(device)     # two's-complement wrap of the high words
        if len(_SET_BITMAPS) > 4096:
            _SET_BITMAPS.clear()
        _SET_BITMAPS[key] = t
    return t.data_ptr()


def _i64(v: int) -> int:
    v &= (1 << 64) - 1
    return v - (1 << 64) if v >> 63 else v


class _Progs:
    """Keeps the ctypes node arrays alive for the duration of a call."""

    def __init__(self, programs: Sequence[Program | None], device=None):
        self.keep = []
        self.arr = (L.qk_expr * max(1, len(programs)))()
        for i, prog in enumerate(programs):
            prog = prog or []
            nodes = (L.qk_expr_node * max(1, len(prog)))()
            for j, (op, a0, a1, imm, imm_i) in enumerate(prog):
                if op == L.OP_IN_SET:
                    imm_i = _i64(imm_i) if a1 <= 64 else _set_bitmap_ptr(a1, imm_i, device)
                nodes[j] = L.qk_expr_node(int(op), int(a0), int(a1), 0, float(imm), int(imm_i))
            self.keep.append(nodes)
            self.arr[i] = L.qk_expr(C.cast(nodes, C.POINTER(L.qk_expr_node)), len(prog), 0)


def is_passthrough(prog: Program) -> bool:
    return len(prog) == 1 and prog[0][0] == L.OP_COL


# ------------------------------------------------------------------ K1
class Bloom:
    """Blocked Bloom filters over join build keys: `nparts` filters of `words` uint32 words each, filter p
    covering the keys with key % nparts == p (what an all-gather of per-rank filters yields)."""

    BITS_PER_KEY = int(__import__('os').environ.get('QK_BLOOM_BITS', '12'))

    def __init__(self, bits: torch.Tensor, words: int, nparts: int):
        self.bits, self.words, self.nparts = bits, int(words), int(nparts)

    @staticmethod
    def words_for(n_keys: int) -> int:
        return max(8, (int(n_keys) * Bloom.BITS_PER_KEY // 32 + 7) // 8 * 8)

    @staticmethod
    def build(keys: torch.Tensor | None, words: int, nparts: int, device) -> "Bloom":
        bits = torch.zeros(nparts * words, dtype=torch.int32, device=device)
        if keys is not None and keys.numel():
            kc = col(keys, "bloom key")
            L.check(L.lib().qk_bloom_build(C.byref(kc), bits.data_ptr(), words, nparts, _stream()), "qk_bloom_build")
        return Bloom(bits, words, nparts)


def scan_filter_project(columns: Sequence[torch.Tensor], pred: Program | None, projs: Sequence[Program],
                        stable: bool = False, bloom: "tuple[Bloom, int] | None" = None):
    """Returns (list of output tensors trimmed to the surviving rows, row count).  One device->host
    read of the row count (the only sync) sizes the result views.  bloom = (Bloom, index into projs of the
    join-key column): fuse the semi-join reduction into the scan (TMA compaction shape only)."""
    if not columns:
        raise L.QkError("scan_filter_project: no input columns")
    n = columns[0].numel()
    dev = columns[0].device
    outs = []
    for p in projs:
        if is_passthrough(p) and not 0 <= p[0][1] < len(columns):
            raise L.QkError(f"scan_filter_project: column slot {p[0][1]} out of range")
        dt = columns[p[0][1]].dtype if is_passthrough(p) else torch.float64
        outs.append(torch.empty(n, dtype=torch.uint8 if dt == torch.bool else dt, device=dev))
    out_rows = torch.zeros(1, dtype=torch.int64, device=dev)
    ws = _ws(L.lib().qk_scan_workspace_bytes(n), dev)
    E.check_call(len(columns), pred, projs, "scan_filter_project")
    pr = _Progs([pred], dev)
    pj = _Progs(list(projs), dev)
    if bloom is not None:
        bf, key_proj = bloom
        desc = L.qk_bloom(bf.bits.data_ptr(), bf.words, bf.nparts, int(key_proj))
        L.check(L.lib().qk_scan_filter_project_sj(cols(columns), len(columns), n, pr.arr, pj.arr, len(projs),
                                                  cols(outs, "output"), out_rows.data_ptr(), C.byref(desc),
                                                  ws.data_ptr(), ws.numel(), _stream()), "qk_scan_filter_project_sj")
    else:
        L.check(L.lib().qk_scan_filter_project(cols(columns), len(columns), n, pr.arr, pj.arr, len(projs),
                                               cols(outs, "output"), out_rows.data_ptr(), 1 if stable else 0,
                                               ws.data_ptr(), ws.numel(), _stream()), "qk_scan_filter_project")
    m = int(out_rows.item())
    return [o[:m] for o in outs], m


# ------------------------------------------------------------------ K1+K2 dense aggregate
DENSE_MAX_GROUPS = 4096            # csrc/scan.cu qk_scan_filter_agg_dense: more groups is QK_ERR_UNSUPPORTED
DENSE_GENERIC_SMEM = 200 * 1024    # csrc/scan.cu: the interpreter's lane-private states, ng * (nagg * 8 + 4) * 256 B


def dense_agg_fits(n_groups: int, nagg: int) -> bool:
    """Whether qk_scan_filter_agg_dense takes `n_groups` groups x `nagg` value aggregates whatever the expressions are:
    the bound of its postfix interpreter (variant 1), the one path that runs every program.  Under the default variant a
    fused plan that does not fit falls back to the interpreter, so a grouping inside this bound never fails for lack of
    shared memory.  Deliberately conservative: some groupings only the runtime-described plan could hold (about 67-140
    groups for one SUM) fail here too; they belong to the hash aggregate, like every grouping outside the bound."""
    n_groups, nagg = int(n_groups), int(nagg)
    return (1 <= n_groups <= DENSE_MAX_GROUPS and 0 <= nagg <= L.MAX_AGGS
            and n_groups * (nagg * 8 + 4) * 256 <= DENSE_GENERIC_SMEM)


class DenseAggState:
    """Running state of a dense (dictionary-key) aggregate: acc[n_groups, nagg] fp64 + cnt[n_groups]."""

    def __init__(self, group_card: Sequence[int], agg_ops: Sequence[int], device):
        self.group_card = [int(c) for c in group_card]
        self.agg_ops = [int(o) for o in agg_ops]
        self.n_groups = 1
        for c in self.group_card:
            self.n_groups *= c
        self.acc = torch.zeros(self.n_groups, max(1, len(self.agg_ops)), dtype=torch.float64, device=device)
        self.cnt = torch.zeros(self.n_groups, dtype=torch.int64, device=device)
        self.ws = _ws(L.lib().qk_scan_agg_workspace_bytes(self.n_groups, len(self.agg_ops)), device)

    def update(self, columns: Sequence[torch.Tensor], pred: Program | None, group_cols: Sequence[int],
               agg_exprs: Sequence[Program], variant: int = 0):
        n = columns[0].numel() if columns else 0
        gc = (C.c_int32 * max(1, len(group_cols)))(*group_cols)
        gk = (C.c_int32 * max(1, len(group_cols)))(*self.group_card)
        ops = (C.c_int32 * max(1, len(self.agg_ops)))(*self.agg_ops)
        E.check_call(len(columns), pred, agg_exprs, "scan_filter_agg_dense")
        dev = self.acc.device
        pr = _Progs([pred], dev)
        ag = _Progs(list(agg_exprs), dev)
        L.check(L.lib().qk_scan_filter_agg_dense(cols(columns), len(columns), n, pr.arr, gc, gk, len(group_cols),
                                                 ag.arr, ops, len(self.agg_ops), self.acc.data_ptr(),
                                                 self.cnt.data_ptr(), self.ws.data_ptr(), self.ws.numel(),
                                                 int(variant), _stream()), "qk_scan_filter_agg_dense")

    def merge_(self, other_acc: torch.Tensor, other_cnt: torch.Tensor):
        """Fold another partial state (e.g. from a peer rank) into this one (SUM only)."""
        self.acc += other_acc
        self.cnt += other_cnt


def last_variant() -> str:
    return L.lib().qk_last_variant().decode()


def last_variant_config() -> str:
    return L.lib().qk_last_variant_config().decode()


# ------------------------------------------------------------------ K2 hash aggregate
class HashAggState:
    def __init__(self, key_dtypes: Sequence[torch.dtype], agg_ops: Sequence[int], capacity: int, device):
        cap = 1
        while cap < max(16, capacity):
            cap <<= 1
        self.desc = L.qk_hashagg_desc()
        self.desc.capacity = cap
        self.desc.nkeys = len(key_dtypes)
        for i, d in enumerate(key_dtypes):
            self.desc.key_dtype[i] = _TORCH2QK[d]
        self.desc.nagg = len(agg_ops)
        for i, o in enumerate(agg_ops):
            self.desc.agg_op[i] = int(o)
        self.key_dtypes = list(key_dtypes)
        self.device = device
        nbytes = L.lib().qk_hashagg_state_bytes(C.byref(self.desc))
        if nbytes == 0:
            raise L.QkError("qk_hashagg_state_bytes: bad descriptor")
        self.state = _ws(nbytes, device)
        self._flags = torch.zeros(2, dtype=torch.int64, device=device)      # [overflow (int32 in the low half), group count]: ONE read-back
        self.overflow = self._flags[:1].view(torch.int32)[:1]
        self.rows_seen = 0
        L.check(L.lib().qk_hashagg_init(C.byref(self.desc), self.state.data_ptr(), _stream()), "qk_hashagg_init")

    @property
    def capacity(self) -> int:
        return int(self.desc.capacity)

    def update(self, keys: Sequence[torch.Tensor], vals: Sequence[torch.Tensor]):
        if len(keys) != self.desc.nkeys or len(vals) != self.desc.nagg:       # the C side reads nkeys / nagg columns
            raise L.QkError(f"hash aggregate: {len(keys)} key / {len(vals)} value columns for a state of "
                            f"{self.desc.nkeys} / {self.desc.nagg}")
        n = keys[0].numel()
        self.rows_seen += n
        L.check(L.lib().qk_hashagg_update(C.byref(self.desc), self.state.data_ptr(), cols(keys, "key"),
                                          cols(vals, "value"), n, self.overflow.data_ptr(), _stream()),
                "qk_hashagg_update")

    def finalize(self, max_groups: int | None = None):
        cap = min(self.capacity, max_groups if max_groups is not None else min(self.capacity, max(self.rows_seen, 1)))
        ok = [torch.empty(cap, dtype=d, device=self.device) for d in self.key_dtypes]
        ov = [torch.empty(cap, dtype=torch.float64, device=self.device) for _ in range(self.desc.nagg)]
        oc = torch.empty(cap, dtype=torch.int64, device=self.device)
        ng = self._flags[1:]
        ng.zero_()
        L.check(L.lib().qk_hashagg_finalize(C.byref(self.desc), self.state.data_ptr(), cols(ok, "key out"),
                                            cols(ov, "value out"), oc.data_ptr(), cap, ng.data_ptr(), _stream()),
                "qk_hashagg_finalize")
        flags = self._flags.cpu()                                            # the one host round trip of a finalize
        if int(flags[0].item()) & 0xffffffff:
            raise L.QkError("hash aggregate table overflowed: raise the capacity")
        g = int(flags[1].item())
        if g > cap:
            raise L.QkError(f"hash aggregate produced {g} groups but the output was sized for {cap}")
        return [k[:g] for k in ok], [v[:g] for v in ov], oc[:g]


# ------------------------------------------------------------------ K3 partition / movers
def partition_plan(key: torch.Tensor, nparts: int, mode: int = L.PART_MOD):
    """dest (int32 per row) and part_offsets (int64[nparts+1]) of the stable partition of `key`."""
    n = key.numel()
    dest = torch.empty(n, dtype=torch.int32, device=key.device)
    offs = torch.empty(nparts + 1, dtype=torch.int64, device=key.device)
    ws = _ws(L.lib().qk_partition_workspace_bytes(n, nparts), key.device)
    kc = col(key, "partition key")
    L.check(L.lib().qk_partition_plan(C.byref(kc), nparts, mode, dest.data_ptr(), offs.data_ptr(), ws.data_ptr(),
                                      ws.numel(), _stream()), "qk_partition_plan")
    return dest, offs


def scatter(columns: Sequence[torch.Tensor], dest: torch.Tensor):
    outs = [torch.empty_like(c) for c in columns]
    for lo in range(0, len(columns), L.MAX_COLS):
        part = list(columns[lo:lo + L.MAX_COLS])
        L.check(L.lib().qk_scatter(cols(part), len(part), dest.data_ptr(), cols(outs[lo:lo + L.MAX_COLS], "output"),
                                   _stream()), "qk_scatter")
    return outs


def scatter_peer(columns: Sequence[torch.Tensor], dest: torch.Tensor, part_offsets: torch.Tensor, peer_col_ptrs: Sequence[Sequence[int]],
                 peer_row_off: Sequence[int]):
    """Partition-scatter straight into the peers' mailboxes (qk_scatter_peer)."""
    nparts, ncols = len(peer_col_ptrs), len(columns)
    flat = (C.c_uint64 * (nparts * ncols))(*[int(p) for row in peer_col_ptrs for p in row])
    roff = (C.c_int64 * nparts)(*[int(x) for x in peer_row_off])
    L.check(L.lib().qk_scatter_peer(cols(columns), ncols, dest.data_ptr(), part_offsets.data_ptr(), nparts, flat, roff, _stream()),
            "qk_scatter_peer")


class XchgChannel:
    """One channel of the peer-memory shuffle (include/qk.h "K6"): this rank's control block + mailbox and the
    peer-mapped addresses of everybody else's.  All ranks call meta / push / recv in the same order on a channel."""

    META = L.XCHG_META_WORDS

    def __init__(self, world: int, rank: int, ctrl_ptrs: Sequence[int], mailbox_ptrs: Sequence[int], mailbox_bytes: int, device,
                 timeout_ms: int = 30000):
        self.world, self.rank, self.device, self.mailbox_bytes = int(world), int(rank), device, int(mailbox_bytes)
        self.desc = L.qk_xchg()
        self.desc.world, self.desc.rank = self.world, self.rank
        for p in range(self.world):
            self.desc.ctrl[p] = int(ctrl_ptrs[p])
            self.desc.mailbox[p] = int(mailbox_ptrs[p])
        self.desc.mailbox_bytes, self.desc.timeout_ms = self.mailbox_bytes, int(timeout_ms)
        self.epoch = 0
        self.meta_host = torch.zeros(self.world * self.META + 1, dtype=torch.int64).pin_memory()
        self.event = torch.cuda.Event()
        self.tail = None            # end of the channel's last recv / push: the next epoch's post must come after it

    def meta(self, words: Sequence[int], part_offsets: torch.Tensor | None = None):
        """Starts a new epoch: posts `words` (the first `world` of them replaced by the partition plan's per-destination
        row counts when part_offsets, a device int64[world+1], is given) and returns everybody's rows as a
        [world][META] int64 numpy array -- after ONE host wait on the stream (the exchange's only round trip)."""
        if len(words) > self.META:
            raise L.QkError("exchange: too many meta words")
        self.epoch += 1
        if self.tail is not None:   # a channel normally lives on one stream; if the caller switched streams, order them
            torch.cuda.current_stream().wait_event(self.tail)
        arr = (C.c_int64 * self.META)(*[int(x) for x in words], *([0] * (self.META - len(words))))
        L.check(L.lib().qk_xchg_meta(C.byref(self.desc), self.epoch, part_offsets.data_ptr() if part_offsets is not None else None,
                                     arr, None, self.meta_host.data_ptr(), _stream()), "qk_xchg_meta")
        self.event.record()
        self.event.synchronize()
        m = self.meta_host.numpy()
        if int(m[-1]) != 0:
            raise L.QkError(f"exchange: a wait for a peer timed out (status {int(m[-1]):#x}): a rank died or fell behind")
        return m[:-1].reshape(self.world, self.META).copy()

    def _off(self, dst_byte_off, ncols):
        flat = [int(x) for row in dst_byte_off for x in row]
        return (C.c_int64 * max(1, len(flat)))(*flat)

    def push(self, columns: Sequence[torch.Tensor], send_lo: Sequence[int], send_hi: Sequence[int], dst_byte_off):
        """Contiguous rows [send_lo[d], send_hi[d]) of every column -> rank d's mailbox (dst_byte_off[d][c])."""
        n = len(columns)
        lo = (C.c_int64 * self.world)(*[int(x) for x in send_lo])
        hi = (C.c_int64 * self.world)(*[int(x) for x in send_hi])
        L.check(L.lib().qk_xchg_push(C.byref(self.desc), self.epoch, cols(columns) if n else None, n, lo, hi,
                                     self._off(dst_byte_off, n), _stream()), "qk_xchg_push")

    def push_scatter(self, columns: Sequence[torch.Tensor], dest: torch.Tensor, part_offsets: torch.Tensor, dst_byte_off):
        """The fused partition scatter + all-to-all (dest / part_offsets from partition_plan)."""
        n = len(columns)
        L.check(L.lib().qk_xchg_push_scatter(C.byref(self.desc), self.epoch, cols(columns), n, dest.data_ptr(), part_offsets.data_ptr(),
                                             self._off(dst_byte_off, n), _stream()), "qk_xchg_push_scatter")

    def recv(self, src_byte_off: Sequence[int], outs: Sequence[torch.Tensor]):
        n = len(outs)
        so = (C.c_int64 * max(1, n))(*[int(x) for x in src_byte_off])
        L.check(L.lib().qk_xchg_recv(C.byref(self.desc), self.epoch, so, cols(outs, "output") if n else None, n, _stream()), "qk_xchg_recv")
        if self.tail is None:
            self.tail = torch.cuda.Event()
        self.tail.record()


def gather(columns: Sequence[torch.Tensor], idx: torch.Tensor):
    n = idx.numel()
    outs = [torch.empty(n, dtype=c.dtype, device=c.device) for c in columns]
    if n == 0:
        return outs
    for lo in range(0, len(columns), L.MAX_COLS):
        part = list(columns[lo:lo + L.MAX_COLS])
        L.check(L.lib().qk_gather(cols(part), len(part), idx.data_ptr(), n, cols(outs[lo:lo + L.MAX_COLS], "output"),
                                  _stream()), "qk_gather")
    return outs


# ------------------------------------------------------------------ K4 / K5 join
class JoinTable:
    """Persistent open-addressing table over int64 build keys; build rows are numbered in arrival order."""

    def __init__(self, capacity_rows: int, device):
        cap = 16
        while cap < 2 * max(1, capacity_rows):
            cap <<= 1
        self.capacity = cap
        self.device = device
        self.table = _ws(L.lib().qk_join_table_bytes(cap), device)
        self.flags = torch.zeros(1, dtype=torch.int32, device=device)
        self.rows = 0
        L.check(L.lib().qk_join_init(self.table.data_ptr(), cap, _stream()), "qk_join_init")

    def build(self, key: torch.Tensor):
        kc = col(key, "build key")
        L.check(L.lib().qk_join_build(self.table.data_ptr(), self.capacity, C.byref(kc), self.rows,
                                      self.flags.data_ptr(), _stream()), "qk_join_build")
        self.rows += key.numel()

    def check_flags(self):
        f = int(self.flags.item())
        if f & 1:
            raise L.QkError("join table overflowed")
        if f & 2:
            raise L.QkError("join key INT64_MIN is reserved")
        return f

    def probe(self, key: torch.Tensor, how: int = L.JOIN_INNER, expect: int | None = None):
        """(probe_idx, build_idx | None) as int32 tensors.  Retries once with the exact size when the
        first output buffer was too small (duplicate build keys)."""
        n = key.numel()
        cap = max(1, expect if expect is not None else n)
        kc = col(key, "probe key")
        while True:
            pi = torch.empty(cap, dtype=torch.int32, device=key.device)
            bi = torch.empty(cap, dtype=torch.int32, device=key.device) if how in (L.JOIN_INNER, L.JOIN_LEFT) else None
            cnt = torch.zeros(1, dtype=torch.int64, device=key.device)
            L.check(L.lib().qk_join_probe(self.table.data_ptr(), self.capacity, C.byref(kc), how, pi.data_ptr(),
                                          bi.data_ptr() if bi is not None else None, cap, cnt.data_ptr(), _stream()),
                    "qk_join_probe")
            m = int(cnt.item())
            if m <= cap:
                return pi[:m], (bi[:m] if bi is not None else None)
            cap = m


# ------------------------------------------------------------------ K7 as-of
def asof_backward(l_time: torch.Tensor, l_by: torch.Tensor, r_time: torch.Tensor, r_by: torch.Tensor, n_by: int):
    out = torch.empty(l_time.numel(), dtype=torch.int32, device=l_time.device)
    ws = _ws(L.lib().qk_asof_workspace_bytes(r_time.numel(), n_by), l_time.device)
    a, b, c, d = col(l_time), col(l_by), col(r_time), col(r_by)
    L.check(L.lib().qk_asof_backward(C.byref(a), C.byref(b), C.byref(c), C.byref(d), n_by, out.data_ptr(),
                                     ws.data_ptr(), ws.numel(), _stream()), "qk_asof_backward")
    return out


def asof_merge(l_time: torch.Tensor, l_by: torch.Tensor, r_time: torch.Tensor, r_by: torch.Tensor, n_by: int,
               carry_in: torch.Tensor | None = None, r_base: int = 0, want_carry: bool = False):
    """Sorted-merge as-of join (qk_asof_merge): out[i] = r_base + (row of the newest right row with the same key and
    r_time <= l_time[i]) or carry_in[key] (or -1).  Returns (out, carry_out | None); None, None when n_by is too large
    for the shared-memory table (the caller then uses asof_backward)."""
    ws_bytes = L.lib().qk_asof_merge_workspace_bytes(l_time.numel(), r_time.numel(), n_by)
    if ws_bytes == 0:
        return None, None
    out = torch.empty(l_time.numel(), dtype=torch.int32, device=l_time.device)
    carry_out = torch.empty(n_by, dtype=torch.int32, device=l_time.device) if want_carry else None
    ws = _ws(ws_bytes, l_time.device)
    a, b, c, d = col(l_time), col(l_by), col(r_time), col(r_by)
    L.check(L.lib().qk_asof_merge(C.byref(a), C.byref(b), C.byref(c), C.byref(d), n_by,
                                  carry_in.data_ptr() if carry_in is not None else None, int(r_base),
                                  carry_out.data_ptr() if carry_out is not None else None, out.data_ptr(), ws.data_ptr(), ws.numel(),
                                  _stream()), "qk_asof_merge")
    return out, carry_out


# ------------------------------------------------------------------ time-series windows
def window_sliding(time: torch.Tensor, by: torch.Tensor, seg: torch.Tensor, n_by: int, size: int, vals: Sequence[torch.Tensor],
                   aggs: Sequence[tuple]):
    """aggs = [(QK_WIN_*, index into vals)]; inputs in key-segmented order.  Returns one fp64 column per aggregate."""
    n = time.numel()
    outs = [torch.empty(n, dtype=torch.float64, device=time.device) for _ in aggs]
    t, b = col(time), col(by)
    opv = (C.c_int32 * max(1, len(aggs)))(*[int(a[0]) for a in aggs])
    srcv = (C.c_int32 * max(1, len(aggs)))(*[int(a[1]) for a in aggs])
    L.check(L.lib().qk_window_sliding(C.byref(t), C.byref(b), seg.data_ptr(), int(n_by), int(size), cols(vals) if vals else None, len(vals),
                                      opv, srcv, len(aggs), cols(outs, "output"), _stream()), "qk_window_sliding")
    return outs


def window_hop_expand(time: torch.Tensor, by: torch.Tensor, seg: torch.Tensor, n_by: int, size: int, hop: int):
    """(wstart int64, key int32, src int32) with ceil(size / hop) slots per row; src = -1 marks an unused slot."""
    slots = -(-int(size) // int(hop))
    n = time.numel()
    wstart = torch.empty(n * slots, dtype=torch.int64, device=time.device)
    key = torch.empty(n * slots, dtype=torch.int32, device=time.device)
    src = torch.empty(n * slots, dtype=torch.int32, device=time.device)
    t, b = col(time), col(by)
    L.check(L.lib().qk_window_hop_expand(C.byref(t), C.byref(b), seg.data_ptr(), int(n_by), int(size), int(hop), slots, wstart.data_ptr(),
                                         key.data_ptr(), src.data_ptr(), _stream()), "qk_window_hop_expand")
    return wstart, key, src


def window_session_ids(time: torch.Tensor, by: torch.Tensor, timeout: int) -> torch.Tensor:
    n = time.numel()
    ids = torch.empty(n, dtype=torch.int64, device=time.device)
    ws = _ws(L.lib().qk_window_session_workspace_bytes(n), time.device)
    t, b = col(time), col(by)
    L.check(L.lib().qk_window_session_ids(C.byref(t), C.byref(b), int(timeout), ids.data_ptr(), ws.data_ptr(), ws.numel(), _stream()),
            "qk_window_session_ids")
    return ids


# ------------------------------------------------------------------ K8 top-k
def topk_candidates(key: torch.Tensor, k: int, descending: bool):
    n = key.numel()
    idx = torch.empty(n, dtype=torch.int32, device=key.device)
    cnt = torch.zeros(1, dtype=torch.int64, device=key.device)
    ws = _ws(L.lib().qk_topk_workspace_bytes(n), key.device)
    kc = col(key, "top-k key")
    L.check(L.lib().qk_topk_candidates(C.byref(kc), int(k), 1 if descending else 0, idx.data_ptr(), cnt.data_ptr(),
                                       ws.data_ptr(), ws.numel(), _stream()), "qk_topk_candidates")
    return idx[:int(cnt.item())]


# ------------------------------------------------------------------ K9 Gram matrix
class GramState:
    """Running Gram matrix of a stream of k-column batches (qk_gram): gram = sum (X - c)^T (X - c) (fp64 [k, k]),
    sums = sum (X - c) (fp64 [k]) and n = rows seen.  The shift c is the caller's: pass the same one to every update."""

    def __init__(self, k: int, device):
        self.k = int(k)
        if self.k < 1:
            raise L.QkError("GramState: k must be >= 1")
        self.gram = torch.zeros(self.k, self.k, dtype=torch.float64, device=device)
        self.sums = torch.zeros(self.k, dtype=torch.float64, device=device)
        self.n = 0
        self.ws = None

    def update(self, columns: Sequence[torch.Tensor], shift: torch.Tensor | None = None, variant: int = 0):
        if len(columns) != self.k:
            raise L.QkError(f"GramState.update: {len(columns)} columns for a {self.k}-column state")
        n = columns[0].numel()
        if shift is not None:
            _require_cuda(shift, "gram shift")
            if shift.dtype != torch.float64 or shift.numel() != self.k:
                raise L.QkError("GramState.update: the shift must be fp64 with one value per column")
        need = int(L.lib().qk_gram_workspace_bytes(n, self.k))
        if self.ws is None or self.ws.numel() < need:
            self.ws = _ws(need, self.gram.device)
        L.check(L.lib().qk_gram(cols(columns, "gram column"), self.k, n, shift.data_ptr() if shift is not None else None,
                                self.gram.data_ptr(), self.sums.data_ptr(), int(variant), self.ws.data_ptr(), self.ws.numel(),
                                _stream()), "qk_gram")
        self.n += n


def gram_last_plan() -> str:
    return L.lib().qk_gram_last_plan().decode()


# ------------------------------------------------------------------ K10 quantile sketch
QSKETCH_SHIFT, QSKETCH_TILE, QSKETCH_MIN_CAPACITY = 42, 2048, 4096          # include/qk.h QK_QSKETCH_*
_SIGN = -(1 << 63)                                                           # int64 with only the sign bit set


def _pow2_at_least(n: int) -> int:
    return 1 << max(0, int(n) - 1).bit_length()


def qsketch_quantiles(keys, counts, mins, maxs, k: int, qs) -> tuple[torch.Tensor, torch.Tensor]:
    """Quantiles `qs` of the k columns of a compacted sketch (any order of entries; min / max are raw images stored in int64):
    (fp64 [len(qs), k] values, bool [len(qs), k] valid).  Target rank of q among the n counted rows of a column:
    round-half-away((n - 1) q), the `nearest` rule of Polars' quantile.  The bucket that holds that rank answers: its min when
    the rank is the bucket's first, its max when it is the last, otherwise the bucket's middle image clamped to [min, max].
    A column with no counted row is not valid (NULL)."""
    dev = keys.device
    nq = len(qs)
    if keys.numel() == 0:
        return torch.full((nq, k), float("nan"), dtype=torch.float64, device=dev), torch.zeros(nq, k, dtype=torch.bool, device=dev)
    order = torch.argsort(keys)
    keys, counts = keys[order], counts[order]
    smin, smax = mins[order] ^ _SIGN, maxs[order] ^ _SIGN                  # order-preserving as signed int64
    col = keys >> 22
    cum = torch.cumsum(counts, 0)
    n = torch.zeros(k, dtype=torch.int64, device=dev).index_add_(0, col, counts)
    base = torch.cumsum(n, 0) - n
    q = torch.tensor([float(x) for x in qs], dtype=torch.float64, device=dev)
    x = (n.to(torch.float64) - 1)[None, :] * q[:, None]                       # (n - 1) q in fp64, as Polars computes it
    f = torch.floor(x)
    r = (f + (x - f >= 0.5).to(torch.float64)).to(torch.int64)               # x - floor(x) is exact: round half away from zero
    valid = (n > 0)[None, :].expand(nq, k)
    target = torch.where(valid, base[None, :] + r, torch.zeros_like(r))
    idx = torch.searchsorted(cum, target, right=True).clamp_max(keys.numel() - 1)
    hi = cum[idx] - 1
    lo = hi - counts[idx] + 1
    mn, mx = smin[idx], smax[idx]
    mid = ((keys[idx] & ((1 << 22) - 1)) - (1 << 21)) * (1 << QSKETCH_SHIFT) + (1 << (QSKETCH_SHIFT - 1))
    s = torch.where(target == lo, mn, torch.where(target == hi, mx, torch.minimum(torch.maximum(mid, mn), mx)))
    bits = torch.where(s >= 0, s, (~s) ^ _SIGN)
    return torch.where(valid, bits.view(torch.float64), float("nan")), valid.clone()


class QuantileSketch:
    """Device quantile sketch of k columns (qk_qsketch_update / qk_qsketch_merge): an open-addressed table of
    [capacity, 4] int64 slots (key, count, min image, max image) and its control words.  update() folds a batch in, growing
    the table and re-running the tiles the kernel deferred until every tile is counted; entries() compacts the occupied
    slots; quantiles(qs) answers from them.  rounds / grows count the deferral rounds and table growths."""

    def __init__(self, k: int, device, capacity: int = 1 << 16):
        self.k = int(k)
        if self.k < 1:
            raise L.QkError("QuantileSketch: k must be >= 1")
        self.device = torch.device(device)
        self.ctrl = torch.zeros(4, dtype=torch.int64, device=self.device)
        self._alloc(max(QSKETCH_MIN_CAPACITY, _pow2_at_least(capacity)))
        self.ws = _ws(L.lib().qk_qsketch_workspace_bytes(self.k), self.device)
        self.rounds = self.grows = 0
        self.ctas = 2 * torch.cuda.get_device_properties(self.device).multi_processor_count   # CTAs resident at once

    def _alloc(self, capacity: int):
        self.capacity = capacity
        self.table = torch.empty(capacity, 4, dtype=torch.int64, device=self.device)
        self.table[:, 0] = -1                                                  # QK_QSKETCH_EMPTY
        self.table[:, 1] = 0
        self.table[:, 2] = -1                                                  # min image ~0
        self.table[:, 3] = 0
        self.ctrl[0] = 0

    def _run(self, columns, valid, n, tiles, ntiles):
        deferred = torch.empty(max(1, ntiles), dtype=torch.int32, device=self.device)
        vp = None
        if valid is not None:
            vp = C.cast((C.c_void_p * self.k)(*[None if v is None else v.data_ptr() for v in valid]), C.c_void_p)
        L.check(L.lib().qk_qsketch_update(cols(columns, "quantile column"), vp, self.k, n, self.table.data_ptr(), self.capacity,
                                          self.ctrl.data_ptr(), None if tiles is None else tiles.data_ptr(), ntiles,
                                          deferred.data_ptr(), self.ws.data_ptr(), self.ws.numel(), _stream()), "qk_qsketch_update")
        occupied, ndef, overflow, _ = self.ctrl.tolist()                      # the one read of the batch
        if overflow:
            raise L.QkError("qk_qsketch_update: a probe ran through the whole table")
        return occupied, ndef, deferred

    def update(self, columns: Sequence[torch.Tensor], valid: Sequence[torch.Tensor | None] | None = None):
        if len(columns) != self.k:
            raise L.QkError(f"QuantileSketch.update: {len(columns)} columns for a {self.k}-column sketch")
        if valid is not None:
            if len(valid) != self.k:
                raise L.QkError("QuantileSketch.update: one row mask (or None) per column")
            for v in valid:
                if v is not None:
                    _require_cuda(v, "quantile row mask")
                    if v.dtype != torch.uint8 or v.numel() != columns[0].numel():
                        raise L.QkError("QuantileSketch.update: a row mask is uint8 with one byte per row")
        n = columns[0].numel()
        if n == 0:
            return
        ntiles = self.k * ((n + QSKETCH_TILE - 1) // QSKETCH_TILE)
        occupied, ndef, deferred = self._run(columns, valid, n, None, ntiles)
        while ndef:
            self.rounds += 1
            pending = deferred[:ndef].clone()
            need = occupied + min(ndef, self.ctas) * QSKETCH_TILE               # room for one wave of new tiles
            if 2 * need > self.capacity:
                self.grow(_pow2_at_least(4 * need))
            occupied, ndef, deferred = self._run(columns, valid, n, pending, ndef)

    def grow(self, capacity: int):
        """Re-insert every entry into a table of `capacity` slots."""
        keys, counts, mins, maxs = self.entries()
        self._alloc(capacity)
        self.merge(keys, counts, mins, maxs)
        self.grows += 1

    def merge(self, keys, counts, mins, maxs):
        """Fold compacted entries (int64 tensors, raw images) in: the final merge of the ranks."""
        n = keys.numel()
        if 2 * (int(self.ctrl[0]) + n) > self.capacity:
            self.grow(_pow2_at_least(4 * (int(self.ctrl[0]) + n)))
        if n == 0:
            return
        ks, cs, lo, hi = (t.contiguous() for t in (keys, counts, mins, maxs))
        L.check(L.lib().qk_qsketch_merge(ks.data_ptr(), cs.data_ptr(), lo.data_ptr(), hi.data_ptr(), n, self.table.data_ptr(),
                                         self.capacity, self.ctrl.data_ptr(), _stream()), "qk_qsketch_merge")

    def entries(self):
        """(key, count, min image, max image) of the occupied slots, int64 tensors in table order."""
        t = self.table[self.table[:, 0] != -1]
        return t[:, 0].contiguous(), t[:, 1].contiguous(), t[:, 2].contiguous(), t[:, 3].contiguous()

    def quantiles(self, qs):
        return qsketch_quantiles(*self.entries(), self.k, qs)


# ------------------------------------------------------------------ Parquet column chunks -> Arrow-layout columns
PQ_PAD = 16      # readable bytes the decoder may touch past the last encoded byte (aligned 8-byte windows)


def parquet_decode(raw: torch.Tensor, runs: torch.Tensor, n_runs: int, n_values: int, dictionary: torch.Tensor | None,
                   out: torch.Tensor, status: torch.Tensor | None = None):
    """raw: uint8 device buffer holding the chunk bytes + PQ_PAD; runs: uint8 view of (n_runs + 1) qk_pq_run
    records (sentinel last); dictionary: entries as wide as `out`'s elements (or None); out: n_values elements."""
    for t, what in ((raw, "parquet bytes"), (runs, "parquet runs"), (out, "parquet output")):
        _require_cuda(t, what)
    if dictionary is not None:
        _require_cuda(dictionary, "parquet dictionary")
        if dictionary.element_size() != out.element_size():
            raise L.QkError("parquet_decode: dictionary entries and output elements differ in width")
    if out.numel() < n_values or runs.numel() < (n_runs + 1) * C.sizeof(L.qk_pq_run) or raw.numel() < PQ_PAD:
        raise L.QkError("parquet_decode: buffer too small")
    L.check(L.lib().qk_parquet_decode(raw.data_ptr(), raw.numel() - PQ_PAD, runs.data_ptr(), n_runs, n_values,
                                      dictionary.data_ptr() if dictionary is not None and dictionary.numel() else None,
                                      dictionary.numel() if dictionary is not None else 0, out.element_size(), out.data_ptr(),
                                      status.data_ptr() if status is not None else None, _stream()), "qk_parquet_decode")
    return out


def parquet_inflate_workspace(n_zstd_pages: int, device) -> torch.Tensor | None:
    """Workspace for the ZSTD / GZIP pages of one inflate call: one slot (decoding tables + literals buffer) per page in flight,
    at most 8 per SM, in whole CTAs.  None when the call has no ZSTD page."""
    if n_zstd_pages <= 0:
        return None
    slot = int(L.lib().qk_parquet_inflate_slot_bytes())
    slots = min(n_zstd_pages, 8 * int(L.lib().qk_sm_count()))
    slots = (slots + L.PQ_INFLATE_WARPS - 1) // L.PQ_INFLATE_WARPS * L.PQ_INFLATE_WARPS
    return torch.empty(slots * slot, dtype=torch.uint8, device=device)


def parquet_inflate(raw: torch.Tensor, pages: torch.Tensor, n_pages: int, scratch: torch.Tensor, work: torch.Tensor | None = None):
    """pages: uint8 view of n_pages qk_pq_page records (device).  Writes every page's uncompressed image to `scratch`."""
    for t, what in ((raw, "parquet bytes"), (pages, "parquet pages"), (scratch, "parquet scratch")):
        _require_cuda(t, what)
    if work is not None:
        _require_cuda(work, "parquet inflate workspace")
    if pages.numel() < n_pages * C.sizeof(L.qk_pq_page):
        raise L.QkError("parquet_inflate: page table too small")
    L.check(L.lib().qk_parquet_inflate(raw.data_ptr(), raw.numel(), pages.data_ptr(), n_pages, scratch.data_ptr(), scratch.numel(),
                                       work.data_ptr() if work is not None else None, work.numel() if work is not None else 0,
                                       _stream()), "qk_parquet_inflate")


def parquet_page_runs(scratch: torch.Tensor, pages: torch.Tensor, n_pages: int, physical_type: int,
                      run_offsets: torch.Tensor | None = None, runs: torch.Tensor | None = None, runs_cap: int = 0):
    """Count pass (run_offsets None: fills pages[i].n_runs / .status) or fill pass of the device-side run walk."""
    for t, what in ((scratch, "parquet scratch"), (pages, "parquet pages")):
        _require_cuda(t, what)
    if run_offsets is not None:
        _require_cuda(run_offsets, "run offsets")
        _require_cuda(runs, "parquet runs")
        if run_offsets.dtype != torch.int64 or run_offsets.numel() < n_pages or runs.numel() < runs_cap * C.sizeof(L.qk_pq_run):
            raise L.QkError("parquet_page_runs: run_offsets must be int64[n_pages] and runs hold runs_cap records")
    L.check(L.lib().qk_parquet_page_runs(scratch.data_ptr(), scratch.numel(), pages.data_ptr(), n_pages, physical_type,
                                         run_offsets.data_ptr() if run_offsets is not None else None,
                                         runs.data_ptr() if runs is not None else None, runs_cap, _stream()), "qk_parquet_page_runs")


def launch_count() -> int:
    return int(L.lib().qk_launch_count())
