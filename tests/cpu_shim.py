"""TEST-ONLY stand-in for quokka_b200.ops so that the HOST logic (expression compiler, planner, edge
functions, executors' protocol handling, the SPMD driver and the gloo exchange) can be exercised in the
CPU build container.  Every function mirrors the signature of its quokka_b200.ops counterpart and is
implemented with the numpy oracle; nothing here ships -- the product has no CPU path, and the same tests
run against the real kernels on the GPU box (tests/test_gpu_api.py)."""
from __future__ import annotations

import numpy as np
import torch

from oracle import relops as R
from quokka_b200 import _lib as L
from quokka_b200 import expr as E
from quokka_b200 import ops as real_ops
from quokka_b200.executors import order_image

qk_dtype = real_ops.qk_dtype
is_passthrough = real_ops.is_passthrough


def _t(a, like=None):
    return torch.from_numpy(np.ascontiguousarray(a))


def _cmp(a, c, b):
    return [a < b, a <= b, a > b, a >= b, a == b, a != b][c]


def eval_prog(prog, cols, n):
    st = []
    for op, a0, a1, imm, imm_i in prog:
        if op == L.OP_COL:
            st.append(cols[a0].astype(np.float64))
        elif op == L.OP_CONST:
            st.append(np.full(n, imm, dtype=np.float64))
        elif op in (L.OP_ADD, L.OP_SUB, L.OP_MUL, L.OP_DIV):
            b, a = st.pop(), st.pop()
            with np.errstate(all="ignore"):
                st.append({L.OP_ADD: a + b, L.OP_SUB: a - b, L.OP_MUL: a * b, L.OP_DIV: a / b}[op])
        elif op == L.OP_NEG:
            st.append(-st.pop())
        elif op in (L.OP_LT, L.OP_LE, L.OP_GT, L.OP_GE, L.OP_EQ, L.OP_NE):
            b, a = st.pop(), st.pop()
            st.append(_cmp(a, op - L.OP_LT, b).astype(np.float64))
        elif op in (L.OP_AND, L.OP_OR):
            b, a = st.pop(), st.pop()
            st.append(((a != 0) & (b != 0) if op == L.OP_AND else (a != 0) | (b != 0)).astype(np.float64))
        elif op == L.OP_NOT:
            st.append((st.pop() == 0).astype(np.float64))
        elif op == L.OP_RINT:
            st.append(np.rint(st.pop()))
        elif op == L.OP_EXTRACT:
            d = st.pop().astype("int64").astype("datetime64[D]")
            part = [d.astype("datetime64[Y]").astype(np.int64) + 1970, d.astype("datetime64[M]").astype(np.int64) % 12 + 1,
                    (d - d.astype("datetime64[M]")).astype(np.int64) + 1][a1]
            st.append(part.astype(np.float64))
        elif op == L.OP_SELECT:
            b, a, c = st.pop(), st.pop(), st.pop()
            st.append(np.where(c != 0, a, b))
        elif op == L.OP_IN_SET:
            code = cols[a0].astype(np.int64)
            lut = np.array([(int(imm_i) >> i) & 1 for i in range(a1)] + [0], dtype=bool)
            st.append(lut[np.where((code >= 0) & (code < a1), code, a1)].astype(np.float64))
        elif op == L.OP_CMP_COL_IMM:
            st.append(_cmp(cols[a0].astype(np.int64), a1, np.int64(imm_i)).astype(np.float64))
        elif op == L.OP_RANGE_COL_IMM:
            x = cols[a0].astype(np.int64)
            st.append((((x >= np.int64(imm_i)) & (x <= np.int64(imm))) != bool(a1)).astype(np.float64))
        elif op == L.OP_CMP_COL_COL:
            st.append(_cmp(cols[a0].astype(np.int64), a1 & 0xff, cols[a1 >> 8].astype(np.int64)).astype(np.float64))
        else:
            raise ValueError(op)
    assert len(st) == 1
    return st[0]


class Bloom:
    """One-hash Bloom filter in numpy with the geometry of quokka_b200.ops.Bloom (nparts x words)."""
    BITS_PER_KEY = 12

    def __init__(self, bits, words, nparts):
        self.bits, self.words, self.nparts = bits, int(words), int(nparts)

    @staticmethod
    def words_for(n_keys):
        return max(8, (int(n_keys) * Bloom.BITS_PER_KEY // 32 + 7) // 8 * 8)

    @staticmethod
    def _slots(keys, words, nparts):
        k = keys.astype(np.int64)
        bit = (k.astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15) >> np.uint64(20)) % np.uint64(words * 32)
        return (k % nparts) * words + (bit // np.uint64(32)).astype(np.int64), (bit % np.uint64(32)).astype(np.int64)

    @staticmethod
    def build(keys, words, nparts, device):
        if keys is not None and keys.dtype not in (torch.uint8, torch.int32, torch.int64):
            raise L.QkError("qk_bloom_build: keys must be integer columns")       # csrc/scan.cu qk_bloom_build
        bits = np.zeros(nparts * words, dtype=np.int64)
        if keys is not None and keys.numel():
            w, b = Bloom._slots(keys.numpy(), words, nparts)
            np.bitwise_or.at(bits, w, np.int64(1) << b)
        return Bloom(_t(bits.astype(np.uint32).view(np.int32)), words, nparts)

    def test(self, keys):
        w, b = Bloom._slots(keys, self.words, self.nparts)
        return ((self.bits.numpy().view(np.uint32)[w].astype(np.int64) >> b) & 1) != 0


def scan_filter_project(columns, pred, projs, stable=False, bloom=None):
    E.check_call(len(columns), pred, projs, "scan_filter_project")          # the limits csrc/scan.cu enforces
    cols = [c.numpy() for c in columns]
    n = len(cols[0])
    mask = eval_prog(pred, cols, n) != 0 if pred else np.ones(n, bool)
    if bloom is not None:
        bf, key_proj = bloom
        _last["variant"] = "shim-bloom"
        mask &= bf.test(cols[projs[key_proj][0][1]])
    outs = []
    for p in projs:
        if is_passthrough(p):
            if not 0 <= p[0][1] < len(cols):
                raise L.QkError("column slot out of range")
            outs.append(_t(cols[p[0][1]][mask]))
        else:
            outs.append(_t(eval_prog(p, cols, n)[mask]))
    return outs, int(mask.sum())


_last = {"variant": "shim"}


def last_variant():
    return _last["variant"]


def last_variant_config():
    return "cpu-shim"


def launch_count():
    return 0


class DenseAggState:
    def __init__(self, group_card, agg_ops, device):
        self.group_card, self.agg_ops = [int(c) for c in group_card], [int(o) for o in agg_ops]
        self.n_groups = int(np.prod(self.group_card)) if self.group_card else 1
        self.acc = torch.zeros(self.n_groups, max(1, len(self.agg_ops)), dtype=torch.float64)
        self.cnt = torch.zeros(self.n_groups, dtype=torch.int64)

    def update(self, columns, pred, group_cols, agg_exprs, variant=0):
        E.check_call(len(columns), pred, agg_exprs, "scan_filter_agg_dense")
        if len(group_cols) > 4 or len(self.agg_ops) > L.MAX_AGGS or self.n_groups > real_ops.DENSE_MAX_GROUPS:
            raise L.QkError("scan_filter_agg_dense: ngroup_cols / nagg / groups out of range")
        if not real_ops.dense_agg_fits(self.n_groups, len(self.agg_ops)):
            raise L.QkError("scan_filter_agg_dense: groups x aggregates exceed the shared-memory dense path")
        cols = [c.numpy() for c in columns]
        n = len(cols[0]) if cols else 0
        mask = eval_prog(pred, cols, n) != 0 if pred else np.ones(n, bool)
        g = np.zeros(n, dtype=np.int64)
        for k, gc in enumerate(group_cols):
            g = g * self.group_card[k] + cols[gc].astype(np.int64)
        g = np.clip(g[mask], 0, self.n_groups - 1)            # the kernels clamp a group id outside the dense range
        seen = self.cnt.numpy() > 0
        self.cnt += _t(np.bincount(g, minlength=self.n_groups).astype(np.int64))
        acc = self.acc.numpy()
        for j, (op, prog) in enumerate(zip(self.agg_ops, agg_exprs)):
            v = eval_prog(prog, cols, n)[mask]
            if op == L.AGG_SUM:
                acc[:, j] += np.bincount(g, weights=v, minlength=self.n_groups)
            else:
                # the kernels combine with fmin / fmax (csrc/scan.cu agg_combine): a NaN value is skipped, not propagated
                f = np.fmin if op == L.AGG_MIN else np.fmax
                cur = np.full(self.n_groups, np.inf if op == L.AGG_MIN else -np.inf)
                f.at(cur, g, v)
                acc[:, j] = np.where(seen, f(acc[:, j], cur), cur)
        _last["variant"] = "shim-dense"


class HashAggState:
    def __init__(self, key_dtypes, agg_ops, capacity, device):
        self.key_dtypes, self.agg_ops = list(key_dtypes), [int(o) for o in agg_ops]
        self.capacity, self.device, self.rows_seen = max(16, int(capacity)), device, 0
        self.keys, self.vals = [], []

    def update(self, keys, vals):
        if any(v.dtype != torch.float64 or v.numel() != keys[0].numel() for v in vals):      # csrc/hashagg.cu: values are fp64 columns
            raise L.QkError("qk_hashagg_update: value columns must be fp64 with as many rows as the keys")
        self.rows_seen += keys[0].numel()
        self.keys.append([k.numpy().copy() for k in keys])
        self.vals.append([v.numpy().copy() for v in vals])

    def finalize(self, max_groups=None):
        nk = len(self.key_dtypes)
        keys = [np.concatenate([b[i] for b in self.keys]) if self.keys else np.zeros(0) for i in range(nk)]
        gid, uniq = R.group_ids(keys)
        ng = len(uniq[0])
        if max_groups is not None and ng > max_groups:
            raise L.QkError(f"hash aggregate produced {ng} groups but the output was sized for {max_groups}")
        ov = []
        for j, op in enumerate(self.agg_ops):
            v = np.concatenate([b[j] for b in self.vals]) if self.vals else np.zeros(0)
            if op == L.AGG_SUM:
                ov.append(_t(np.bincount(gid, weights=v, minlength=ng)))
                continue
            # csrc/hashagg.cu atomic_minmax: a NaN value never replaces the accumulator, which starts at +inf / -inf
            acc = np.full(ng, np.inf if op == L.AGG_MIN else -np.inf)
            (np.fmin if op == L.AGG_MIN else np.fmax).at(acc, gid, v)
            ov.append(_t(acc))
        ok = [_t(u.astype(k.dtype)) for u, k in zip(uniq, keys)]
        return ok, ov, _t(np.bincount(gid, minlength=ng).astype(np.int64))


PART_MOD_MAX_PARTS = 16_384              # csrc/partition.cu: MOD partitions keep their per-chunk histogram in shared memory
MERGE_MAX_KEYS = 40_960                  # csrc/asof.cu: the merge kernel's per-key table is at most 160 KB of int32


def partition_plan(key, nparts, mode=L.PART_MOD):
    if nparts < 1 or (mode == L.PART_MOD and nparts > PART_MOD_MAX_PARTS):
        raise L.QkError(f"qk_partition_plan: nparts must be in [1, {PART_MOD_MAX_PARTS}] in MOD mode")
    k = key.numpy().astype(np.int64)
    p = k % nparts if mode == L.PART_MOD else np.clip(k, 0, nparts - 1)
    order = np.argsort(p, kind="stable")
    dest = np.empty(len(k), dtype=np.int32)
    dest[order] = np.arange(len(k), dtype=np.int32)
    offs = np.concatenate([[0], np.cumsum(np.bincount(p, minlength=nparts))]).astype(np.int64)
    return _t(dest), _t(offs)


def scatter(columns, dest):
    d = dest.numpy()
    outs = []
    for c in columns:
        o = np.empty_like(c.numpy())
        o[d] = c.numpy()
        outs.append(_t(o))
    return outs


def gather(columns, idx):
    i = idx.numpy().astype(np.int64)
    outs = []
    for c in columns:
        a = c.numpy()
        if len(a) == 0:
            outs.append(_t(np.zeros(len(i), dtype=a.dtype)))
            continue
        o = a[np.maximum(i, 0)]
        o[i < 0] = 0
        outs.append(_t(o))
    return outs


class JoinTable:
    def __init__(self, capacity_rows, device):
        self.keys, self.rows, self.device = [], 0, device

    def build(self, key):
        self.keys.append(key.numpy().astype(np.int64))
        self.rows += key.numel()

    def check_flags(self):
        return 0

    def probe(self, key, how=L.JOIN_INNER, expect=None):
        bk = np.concatenate(self.keys) if self.keys else np.zeros(0, np.int64)
        name = {L.JOIN_INNER: "inner", L.JOIN_LEFT: "left", L.JOIN_SEMI: "semi", L.JOIN_ANTI: "anti"}[how]
        li, ri = R.join_indices(key.numpy().astype(np.int64), bk, name)
        return _t(li.astype(np.int32)), (None if ri is None else _t(ri.astype(np.int32)))


def asof_backward(l_time, l_by, r_time, r_by, n_by):
    return _t(R.asof_backward(l_time.numpy(), l_by.numpy(), r_time.numpy(), r_by.numpy()).astype(np.int32))


def asof_merge(l_time, l_by, r_time, r_by, n_by, carry_in=None, r_base=0, want_carry=False):
    if n_by > MERGE_MAX_KEYS:
        return None, None
    lb, rb = l_by.numpy().astype(np.int64), r_by.numpy().astype(np.int64)
    idx = R.asof_backward(l_time.numpy(), lb, r_time.numpy(), rb).astype(np.int64)
    cin = carry_in.numpy().astype(np.int64) if carry_in is not None else np.full(n_by, -1, np.int64)
    ok = (lb >= 0) & (lb < n_by)
    fallback = np.where(ok, cin[np.clip(lb, 0, n_by - 1)], -1)
    out = np.where(idx >= 0, idx + r_base, fallback)
    carry = None
    if want_carry:
        carry = cin.copy()
        good = (rb >= 0) & (rb < n_by)
        last = np.full(n_by, -1, np.int64)
        np.maximum.at(last, rb[good], np.nonzero(good)[0])
        carry = np.where(last >= 0, last + r_base, carry)
        carry = _t(carry.astype(np.int32))
    return _t(out.astype(np.int32)), carry


def window_sliding(time, by, seg, n_by, size, vals, aggs):
    t, b = time.numpy(), by.numpy()
    names = {L.WIN_SUM: "sum", L.WIN_MIN: "min", L.WIN_MAX: "max", L.WIN_COUNT: "count", L.WIN_AVG: "avg"}
    res = R.sliding_window(t, b, size, {str(i): (names[op], None if op == L.WIN_COUNT else vals[src].numpy()) for i, (op, src) in enumerate(aggs)})
    return [_t(res[str(i)].astype(np.float64)) for i in range(len(aggs))]


def window_hop_expand(time, by, seg, n_by, size, hop):
    t, b, sg = time.numpy(), by.numpy().astype(np.int64), seg.numpy()
    slots = -(-int(size) // int(hop))
    n = len(t)
    first = (t[np.clip(sg[np.clip(b, 0, n_by - 1)], 0, max(n - 1, 0))] // hop) * hop if n else np.zeros(0, np.int64)
    kmax, kmin = t // hop, (t - size) // hop + 1
    k = kmax[:, None] - np.arange(slots)[None, :]
    valid = (k >= kmin[:, None]) & (k * hop >= first[:, None])
    src = np.where(valid, np.arange(n)[:, None], -1)
    return _t((k * hop).reshape(-1).astype(np.int64)), _t(np.repeat(b, slots).astype(np.int32)), _t(src.reshape(-1).astype(np.int32))


def window_session_ids(time, by, timeout):
    t, b = time.numpy(), by.numpy()
    flag = np.ones(len(t), dtype=np.int64)
    if len(t) > 1:
        flag[1:] = (b[1:] != b[:-1]) | ((t[1:] - t[:-1]) > timeout)
    return _t(np.cumsum(flag))


def topk_candidates(key, k, descending):
    if k <= 0:
        raise L.QkError("qk_topk_candidates: k must be positive")
    v = key.numpy()
    if len(v) <= k:
        return _t(np.arange(len(v), dtype=np.int32))
    img = order_image(v, not descending)                   # csrc/topk.cu image_of: the best rows have the largest image
    kth = np.sort(img)[-k]
    return _t(np.nonzero(img >= kth)[0].astype(np.int32))


PQ_PAD = real_ops.PQ_PAD
_pq_native = None


def _pq_check_lib():
    """g++ build of tests/native/pq_core_check.cpp: the decoder core of quokka_b200/csrc/parquet_core.h on the host."""
    global _pq_native
    if _pq_native is None:
        import ctypes, os, subprocess
        here = os.path.dirname(os.path.abspath(__file__))
        out_dir = os.path.join(here, "_native")
        os.makedirs(out_dir, exist_ok=True)
        so = os.path.join(out_dir, "pq_core_check.so")
        srcs = [os.path.join(here, "native", "pq_core_check.cpp"), os.path.join(here, "..", "quokka_b200", "csrc", "parquet_core.h"),
                os.path.join(here, "..", "quokka_b200", "csrc", "zstd_core.h"), os.path.join(here, "..", "quokka_b200", "csrc", "deflate_core.h"),
                os.path.join(here, "..", "include", "qk.h")]
        if not os.path.exists(so) or any(os.path.getmtime(f) > os.path.getmtime(so) for f in srcs):
            subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so + ".tmp", srcs[0]], check=True)
            os.replace(so + ".tmp", so)
        _pq_native = ctypes.CDLL(so)
        _pq_native.pq_check_decode.restype = ctypes.c_int
        _pq_native.pq_check_decode.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int64, ctypes.c_void_p,
                                               ctypes.c_int64, ctypes.c_int, ctypes.c_void_p]
        _pq_native.pq_check_inflate.restype = None
        _pq_native.pq_check_inflate.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64]
        _pq_native.pq_check_slot_bytes.restype = ctypes.c_size_t
        _pq_native.pq_check_zstd.restype = ctypes.c_int
        _pq_native.pq_check_zstd.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64]
        _pq_native.pq_check_gzip.restype = ctypes.c_int
        _pq_native.pq_check_gzip.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64]
        _pq_native.pq_check_page_runs.restype = None
        _pq_native.pq_check_page_runs.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_void_p,
                                                  ctypes.c_void_p, ctypes.c_int64]
    return _pq_native


def parquet_decode(raw, runs, n_runs, n_values, dictionary, out, status=None):
    if dictionary is not None and dictionary.element_size() != out.element_size():
        raise L.QkError("parquet_decode: dictionary entries and output elements differ in width")
    bad = _pq_check_lib().pq_check_decode(raw.data_ptr(), runs.data_ptr(), n_runs, n_values,
                                          dictionary.data_ptr() if dictionary is not None else None,
                                          dictionary.numel() if dictionary is not None else 0, out.element_size(), out.data_ptr())
    if bad and status is not None:
        status |= 1
    return out


def parquet_inflate_workspace(n_zstd_pages, device):
    if n_zstd_pages <= 0:
        return None
    slots = (min(n_zstd_pages, 6) + 3) // 4 * 4            # few slots: pages must queue up behind them, as on a busy GPU
    return torch.empty(slots * _pq_check_lib().pq_check_slot_bytes(), dtype=torch.uint8)


def parquet_inflate(raw, pages, n_pages, scratch, work=None):
    lib = _pq_check_lib()
    lib.pq_check_inflate(raw.data_ptr(), pages.data_ptr(), n_pages, scratch.data_ptr(), work.data_ptr() if work is not None else None,
                         work.numel() // lib.pq_check_slot_bytes() if work is not None else 0)


def parquet_page_runs(scratch, pages, n_pages, physical_type, run_offsets=None, runs=None, runs_cap=0):
    elem = {L.PQ_BOOLEAN: 0, L.PQ_INT32: 4, L.PQ_FLOAT: 4, L.PQ_INT64: 8, L.PQ_DOUBLE: 8, L.PQ_BYTE_ARRAY: -1}[physical_type]
    _pq_check_lib().pq_check_page_runs(scratch.data_ptr(), pages.data_ptr(), n_pages, elem,
                                       run_offsets.data_ptr() if run_offsets is not None else None,
                                       runs.data_ptr() if runs is not None else None, runs_cap)


def install(monkeypatch):
    """Route quokka_b200's kernel calls to this shim and let QuokkaContext run on CPU tensors."""
    import quokka_b200.columns as C
    import quokka_b200.df as D
    import quokka_b200.edge as ED
    import quokka_b200.executors as X
    import quokka_b200.runtime as RT
    import sys
    shim = sys.modules[__name__]
    import quokka_b200.parquet as PQ
    for mod in (C, ED, X, RT, PQ):
        monkeypatch.setattr(mod, "ops", shim)
    monkeypatch.setattr(C, "_default_device", lambda: torch.device("cpu"))
