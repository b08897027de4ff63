"""Exact numpy reference and seeded plan generator for the dense aggregate (csrc/scan.cu qk_scan_filter_agg_dense), the
grammar of its runtime-described plan (`match_dyn`):

    predicate  = AND of 0..6 terms, each optionally negated: integer column <cmp> constant | fp column <cmp> constant |
                 code column IN set | integer column <cmp> integer column
    group keys = 0..4 code columns (row-major group id, first key most significant)
    aggregate  = SUM / MIN / MAX of f1 * f2 * f3 (left to right), f = k | c | k + c | k - c | c - k | -c,
                 SUM optionally gated: CASE WHEN term THEN product ELSE 0 END

A plan is built from `Term`, `Factor` and `Agg` objects, each of which carries its SQL text and its numpy evaluation, so
the text goes through `expr.parse` / `expr.compile_expr` like every query, and the reference computes the mask, the group
id and every per-row value with the same fp64 operations in the same order as the kernels.  The library is built with
-fmad=false, so each per-row value is bit-identical to the kernel's.  From those values the reference takes counts,
MIN / MAX (fmin / fmax: a NaN value is skipped, as `agg_combine` does) and SUMs as exact sums (math.fsum per group, or a
plain sum where every partial sum is exact).

Data modes:
- "dyadic": factor columns hold integers in [-256, 256] times 2^-4 and factor constants are such numbers too, so a
  product of three factors is an integer multiple of 2^-12 below 2^27 in magnitude and any SUM of fewer than 2^26 rows
  is exact in every summation order: every kernel path must then match the reference bit for bit (±0 compare equal).
- "tpch": the fp64 measures, ship date and flags of oracle/tpch_gen.py's lineitem: SUMs within
  n_g * 2^-53 * sum|x| of the exact sum (n_g = the group's row count), MIN / MAX and counts exact.

Importable without a GPU: tests/test_dense_agg_cpu.py checks the reference against a per-row Python evaluation and the
CPU shim against the reference; tests/test_gpu_dense_agg.py runs the kernels."""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import numpy as np

from oracle import tpch_gen as G
from quokka_b200 import _lib as L

I32_MIN, I32_MAX = -(1 << 31), (1 << 31) - 1
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
DY_MAXTERMS, DY_MAXCOLS, DY_MAXFACT = 6, 10, 3          # csrc/scan.cu
CMPS = ("<", "<=", ">", ">=", "=", "!=")
_NP_CMP = {"<": np.less, "<=": np.less_equal, ">": np.greater, ">=": np.greater_equal, "=": np.equal, "!=": np.not_equal}
QK_DTYPE = {np.dtype(np.uint8): L.QK_U8, np.dtype(np.int32): L.QK_I32, np.dtype(np.int64): L.QK_I64,
            np.dtype(np.float32): L.QK_F32, np.dtype(np.float64): L.QK_F64}
AGG_OP = {"sum": L.AGG_SUM, "min": L.AGG_MIN, "max": L.AGG_MAX}


def fmt(c) -> str:
    """SQL literal of a number: shortest round-trip decimal; ±inf as ±1e400 (which the tokenizer reads back as ±inf)."""
    if isinstance(c, (int, np.integer)):
        return str(int(c))
    c = float(c)
    if math.isinf(c):
        return "1e400" if c > 0 else "-1e400"
    return repr(c)


# ------------------------------------------------------------------ plan objects
@dataclass
class Term:
    sql: str
    cols: tuple
    fn: object                      # data dict -> bool array
    kind: str = ""

    def mask(self, d):
        return np.asarray(self.fn(d), dtype=bool)

    def negate(self) -> "Term":
        return Term(f"not ({self.sql})", self.cols, lambda d, f=self.fn: ~np.asarray(f(d), dtype=bool), self.kind)


def irange(c, cmp, k) -> Term:
    """integer column <cmp> integer constant (any int64 constant: range_of clamps it to the column's width)"""
    return Term(f"{c} {cmp} {fmt(int(k))}", (c,), lambda d: _NP_CMP[cmp](d[c].astype(np.int64), np.int64(k)), "irange")


def between(c, lo, hi) -> Term:
    return Term(f"{c} between {fmt(int(lo))} and {fmt(int(hi))}", (c,),
                lambda d: (d[c].astype(np.int64) >= lo) & (d[c].astype(np.int64) <= hi), "irange")


def fcmp(c, cmp, k) -> Term:
    """fp column (f64 or f32, widened exactly) <cmp> fp64 constant"""
    return Term(f"{c} {cmp} {fmt(float(k))}", (c,), lambda d: _errfree(_NP_CMP[cmp], d[c].astype(np.float64), np.float64(k)), "fcmp")


def inset(c, codes) -> Term:
    """code column IN (non-negative integer codes): one bitmap node of max(codes) + 1 bits"""
    codes = sorted(set(int(x) for x in codes))
    return Term(f"{c} in ({', '.join(map(str, codes))})", (c,), lambda d: np.isin(d[c].astype(np.int64), codes), "inset")


def colcol(a, cmp, b) -> Term:
    return Term(f"{a} {cmp} {b}", (a, b), lambda d: _NP_CMP[cmp](d[a].astype(np.int64), d[b].astype(np.int64)), "colcol")


def _errfree(f, *a):
    with np.errstate(all="ignore"):
        return f(*a)


@dataclass
class Factor:
    sql: str
    col: str | None
    fn: object                      # data dict -> fp64 array
    key: tuple = ()                 # (k0, k1, column) as match_dyn sees it: equal keys share a product prefix

    def values(self, d, n):
        return np.broadcast_to(np.asarray(self.fn(d), dtype=np.float64), (n,))


def f_col(c) -> Factor:
    return Factor(c, c, lambda d: d[c].astype(np.float64), (0.0, 1.0, c))


def f_const(k) -> Factor:
    k = float(k)
    return Factor(fmt(k), None, lambda d: np.float64(k), (k, 0.0, None))


def f_kplus(k, c) -> Factor:          # k + c
    k = float(k)
    return Factor(f"({fmt(k)} + {c})", c, lambda d: _errfree(np.add, np.float64(k), d[c].astype(np.float64)), (k, 1.0, c))


def f_kminus(k, c) -> Factor:         # k - c
    k = float(k)
    return Factor(f"({fmt(k)} - {c})", c, lambda d: _errfree(np.subtract, np.float64(k), d[c].astype(np.float64)), (k, -1.0, c))


def f_minusk(c, k) -> Factor:         # c - k
    k = float(k)
    return Factor(f"({c} - {fmt(k)})", c, lambda d: _errfree(np.subtract, d[c].astype(np.float64), np.float64(k)), (-k, 1.0, c))


def f_neg(c) -> Factor:               # -c
    return Factor(f"(-{c})", c, lambda d: -d[c].astype(np.float64), (-0.0, -1.0, c))


@dataclass
class Agg:
    op: str                          # sum | min | max
    factors: list
    gate: Term | None = None

    @property
    def sql(self) -> str:
        body = " * ".join(f.sql for f in self.factors)
        return f"case when {self.gate.sql} then {body} else 0 end" if self.gate is not None else body

    @property
    def cols(self):
        return tuple(f.col for f in self.factors if f.col is not None) + (self.gate.cols if self.gate is not None else ())

    def values(self, d, n):
        x = self.factors[0].values(d, n).copy()
        with np.errstate(all="ignore"):
            for f in self.factors[1:]:
                x = x * f.values(d, n)                    # left to right, like the postfix program and the tile walk
        if self.gate is not None:
            x = np.where(self.gate.mask(d), x, 0.0)
        return x


@dataclass
class Plan:
    terms: list = field(default_factory=list)
    keys: list = field(default_factory=list)          # [(column, cardinality)]
    aggs: list = field(default_factory=list)

    @property
    def pred_sql(self):
        return " and ".join(t.sql for t in self.terms) if self.terms else None

    @property
    def columns(self):
        """the columns a call passes, in first-use order: predicate, keys, aggregates"""
        out = []
        for c in [c for t in self.terms for c in t.cols] + [k for k, _ in self.keys] + [c for a in self.aggs for c in a.cols]:
            if c not in out:
                out.append(c)
        return out

    @property
    def cards(self):
        return [int(c) for _, c in self.keys]

    @property
    def n_groups(self):
        return int(np.prod(self.cards)) if self.keys else 1

    @property
    def agg_ops(self):
        return [AGG_OP[a.op] for a in self.aggs]

    def describe(self):
        return f"pred={self.pred_sql!r} keys={self.keys} aggs={[(a.op, a.sql) for a in self.aggs]}"


# ------------------------------------------------------------------ compiling a plan the product's way
def compile_plan(plan: Plan, data: dict):
    """-> (column names, predicate program or None, group slots, aggregate programs), through expr.parse / compile_expr"""
    from quokka_b200 import expr as E
    names = plan.columns or [next(iter(data))]
    sch = {c: E.ColumnInfo(i, QK_DTYPE[np.dtype(data[c].dtype)]) for i, c in enumerate(names)}
    pred = E.compile_expr(E.parse(plan.pred_sql), sch) if plan.terms else None
    progs = [E.compile_expr(E.parse(a.sql), sch) for a in plan.aggs]
    E.check_call(len(names), pred, progs, "dense_agg_cases")
    return names, pred, [sch[k].slot for k, _ in plan.keys], progs


# ------------------------------------------------------------------ the reference
def group_ids(plan: Plan, d: dict, n: int) -> np.ndarray:
    g = np.zeros(n, dtype=np.int64)
    for k, card in plan.keys:
        g = g * card + d[k].astype(np.int64)
    return np.clip(g, 0, plan.n_groups - 1)              # the kernels clamp an id outside the dense range


def exact_group_sums(g, v, ng):
    """Exact per-group sums of fp64 values (then rounded once): a plain sum where every partial sum is exact (all values
    integer multiples of 2^-12 whose magnitudes add up to less than 2^53 of them), math.fsum per group otherwise; IEEE
    rules for groups holding inf / NaN."""
    out = np.zeros(ng)
    if len(v) == 0:
        return out
    fin = np.isfinite(v)
    s = v * 4096.0
    if fin.all() and np.all(s == np.trunc(s)) and np.abs(s).sum() < 2.0 ** 53:
        return np.bincount(g, weights=v, minlength=ng)
    order = np.argsort(g, kind="stable")
    gs, vs = g[order], v[order]
    bounds = np.searchsorted(gs, np.arange(ng + 1))
    vl = vs.tolist()
    for j in range(ng):
        lo, hi = bounds[j], bounds[j + 1]
        if lo == hi:
            continue
        part = vs[lo:hi]
        if np.isfinite(part).all():
            out[j] = math.fsum(vl[lo:hi])
        elif np.isnan(part).any() or (np.isposinf(part).any() and np.isneginf(part).any()):
            out[j] = np.nan
        else:
            out[j] = np.inf if np.isposinf(part).any() else -np.inf
    return out


@dataclass
class Reference:
    acc: np.ndarray                  # [n_groups, max(1, nagg)]: what a fresh DenseAggState holds after one update
    cnt: np.ndarray                  # [n_groups] int64
    abs_sum: np.ndarray              # [n_groups, max(1, nagg)]: sum |x| of the SUM arguments (error bound)
    mask: np.ndarray
    gid: np.ndarray


def reference(plan: Plan, d: dict, n: int | None = None) -> Reference:
    n = len(next(iter(d.values()))) if n is None else n
    ng = plan.n_groups
    mask = np.ones(n, dtype=bool)
    for t in plan.terms:
        mask &= t.mask(d)
    gid = group_ids(plan, d, n)
    g = gid[mask]
    cnt = np.bincount(g, minlength=ng).astype(np.int64)
    acc = np.zeros((ng, max(1, len(plan.aggs))))
    abs_sum = np.zeros_like(acc)
    for j, a in enumerate(plan.aggs):
        v = a.values(d, n)[mask]
        if a.op == "sum":
            acc[:, j] = exact_group_sums(g, v, ng)
            with np.errstate(all="ignore"):
                abs_sum[:, j] = np.bincount(g, weights=np.abs(v), minlength=ng)
        else:
            f = np.fmin if a.op == "min" else np.fmax                 # agg_combine: a NaN value is skipped
            cur = np.full(ng, np.inf if a.op == "min" else -np.inf)    # the identity stays for a group without rows
            f.at(cur, g, v)
            acc[:, j] = cur
    return Reference(acc, cnt, abs_sum, mask, gid)


def check(plan: Plan, acc, cnt, ref: Reference, exact: bool, tag="") -> None:
    """Counts always bit-equal, MIN / MAX equal (±0 equal, NaN = NaN), SUMs equal when `exact` else within
    n_g * 2^-53 * sum |x| of the exact sum."""
    acc, cnt = np.asarray(acc), np.asarray(cnt)
    where = f"{tag} {plan.describe()}"
    bad = np.flatnonzero(cnt != ref.cnt)
    assert len(bad) == 0, f"counts differ in groups {bad[:8]}: got {cnt[bad[:8]]} want {ref.cnt[bad[:8]]}; {where}"
    for j, a in enumerate(plan.aggs):
        got, want = acc[:, j], ref.acc[:, j]
        same = (got == want) | (np.isnan(got) & np.isnan(want))
        if a.op == "sum" and not exact:
            tol = ref.cnt * 2.0 ** -53 * ref.abs_sum[:, j]
            with np.errstate(all="ignore"):
                same |= np.isfinite(want) & (np.abs(got - want) <= tol)
        bad = np.flatnonzero(~same)
        assert len(bad) == 0, (f"aggregate {j} ({a.op} {a.sql}) differs in groups {bad[:8]}: got {got[bad[:8]].tolist()} "
                               f"want {want[bad[:8]].tolist()}; {where}")


# ------------------------------------------------------------------ data
FACTOR_COLS = ("fa", "fb", "fc", "g32")          # f64, f64, f64, f32
KEY_COLS = {"k8a": (np.uint8, 3), "k8b": (np.uint8, 2), "k32": (np.int32, 4), "k64": (np.int64, 3)}


def dyadic(rng, n, dtype=np.float64):
    return (rng.integers(-256, 257, n) / 16.0).astype(dtype)


def make_data(n: int, seed: int, mode: str = "dyadic") -> dict:
    """Columns every generated plan draws from.  fa, fb, fc, fd: fp64 factors / compare columns; g32: float32; i32a, i32b:
    int32 (i32a holds INT32_MIN / MAX in a few rows); i64a, i64b: int64 (INT64_MIN / MAX in a few rows); u8: uint8 codes
    0..255; c32: int32 codes -5..79 (negative and beyond any 64-bit set); keys k8a, k8b (uint8), k32 (int32), k64 (int64)
    with the cardinalities of KEY_COLS.  mode "tpch" takes fa, fb, fc, fd, g32 and i32a from lineitem (extended price,
    discount, tax, quantity, quantity as float32, ship date)."""
    rng = np.random.default_rng(seed)
    d = {}
    if mode == "dyadic":
        d["fa"], d["fb"], d["fc"], d["fd"] = dyadic(rng, n), dyadic(rng, n), dyadic(rng, n), dyadic(rng, n)
        d["g32"] = dyadic(rng, n, np.float32)
        d["i32a"] = rng.integers(-1000, 1000, n).astype(np.int32)
    else:
        lo = int(rng.integers(0, 5_000_000))
        li = G.gen_lineitem(1, lo, lo + n, ["l_extendedprice", "l_discount", "l_tax", "l_quantity", "l_shipdate"])
        d["fa"], d["fb"], d["fc"], d["fd"] = li["l_extendedprice"], li["l_discount"], li["l_tax"], li["l_quantity"]
        d["g32"] = li["l_quantity"].astype(np.float32)
        d["i32a"] = li["l_shipdate"].astype(np.int32)
    d["i32b"] = rng.integers(-1000, 1000, n).astype(np.int32)
    d["i64a"] = rng.integers(-1000, 1000, n).astype(np.int64)
    d["i64b"] = rng.integers(-1000, 1000, n).astype(np.int64)
    d["u8"] = rng.integers(0, 256, n).astype(np.uint8)
    d["c32"] = rng.integers(-5, 80, n).astype(np.int32)
    for k, (dt, card) in KEY_COLS.items():
        d[k] = rng.integers(0, card, n).astype(dt)
    if n >= 8:
        at = rng.choice(n, 4, replace=False)
        d["i32a"][at[:2]] = [I32_MIN, I32_MAX]
        d["i64a"][at[2:]] = [I64_MIN, I64_MAX]
    return d


# ------------------------------------------------------------------ the random plan generator
def _constant(rng, d, c):
    """a compare constant that often equals a value of the column (boundary rows)"""
    if len(d[c]) and rng.random() < 0.7:
        return d[c][int(rng.integers(0, len(d[c])))]
    return rng.integers(-256, 257) / 16.0


def random_term(rng, d, fast: bool) -> Term:
    kinds = ["irange32", "fcmp64", "inset8"] if fast else \
        ["irange32", "irange64", "irange8", "fcmp64", "fcmp32", "inset8", "inset32", "cc32", "cc64", "ccmix"]
    if fast:
        kinds += ["irange64", "cc32", "cc64"]       # int64 ranges and same-width column pairs are typed-walk terms too
    kind = kinds[int(rng.integers(0, len(kinds)))]
    cmp = CMPS[int(rng.integers(0, 6))]
    if kind.startswith("irange"):
        c = {"irange32": "i32a", "irange64": "i64a", "irange8": "u8"}[kind]
        r = rng.random()
        if r < 0.15:
            k = int(rng.choice([I32_MIN - 5, I32_MAX + 5, -(1 << 40), 1 << 40, I64_MIN, I64_MAX]))
        elif r < 0.3:
            lo, hi = sorted(int(x) for x in rng.integers(-300, 300, 2))
            t = between(c, lo, hi) if rng.random() < 0.8 else between(c, hi + 1, lo)      # sometimes empty
            return t.negate() if rng.random() < 0.3 else t
        else:
            k = int(d[c][int(rng.integers(0, len(d[c])))]) if len(d[c]) and rng.random() < 0.6 else int(rng.integers(-300, 300))
        t = irange(c, cmp, k)
    elif kind.startswith("fcmp"):
        c = ["fa", "fb", "fc"][int(rng.integers(0, 3))] if kind == "fcmp64" else "g32"
        t = fcmp(c, cmp, _constant(rng, d, c))
    elif kind.startswith("inset"):
        c = "u8" if kind == "inset8" else "c32"
        hi = int(rng.choice([3, 63, 64, 65, 70] if c == "c32" else [3, 63, 64, 65, 200]))
        # at least two codes: a one-code set compiles to `c = code`, an integer range term on the code column
        codes = set(int(x) for x in rng.integers(0, hi, int(rng.integers(2, 12)))) | {0, hi - 1}
        t = inset(c, codes)
    else:
        a, b = {"cc32": ("i32a", "i32b"), "cc64": ("i64a", "i64b"), "ccmix": ("i32b", "i64b")}[kind]
        t = colcol(a, cmp, b)
    return t.negate() if rng.random() < 0.25 else t


def random_factor(rng, fast: bool) -> Factor:
    cols = ["fa", "fb", "fc"] if fast else ["fa", "fb", "fc", "g32"]
    c = cols[int(rng.integers(0, len(cols)))]
    k = int(rng.integers(-256, 257)) / 16.0
    r = rng.random()
    return (f_col(c) if r < 0.4 else f_kminus(k, c) if r < 0.55 else f_kplus(k, c) if r < 0.7 else
            f_minusk(c, k) if r < 0.8 else f_neg(c) if r < 0.9 else f_const(k))


def random_plan(rng, d, fast: bool = False, max_terms: int = DY_MAXTERMS) -> Plan:
    """0..6 terms, 0..4 keys, 0..8 aggregates; every plan stays inside the runtime-described plan's limits (at most 6
    terms, 10 staged columns, 3 factors) and inside ops.dense_agg_fits, so the fused path and the interpreter both take it."""
    from quokka_b200 import expr as E, ops
    for _ in range(1000):
        terms = [random_term(rng, d, fast) for _ in range(int(rng.integers(0, max_terms + 1)))]
        kc = list(KEY_COLS) if not fast else ["k8a", "k8b", "k32"]
        nk = int(rng.integers(0, 5))
        keys = [(k, KEY_COLS[k][1]) for k in rng.permutation(kc)[:nk]]
        aggs = []
        for j in range(int(rng.integers(0, 9))):
            op = ["sum", "sum", "min", "max"][int(rng.integers(0, 4))]
            if aggs and len(aggs[-1].factors) < DY_MAXFACT and rng.random() < 0.4:
                fs = list(aggs[-1].factors) + [random_factor(rng, fast)]                   # extends the previous product
            else:
                fs = [random_factor(rng, fast) for _ in range(int(rng.integers(1, DY_MAXFACT + 1)))]
            gate = random_term(rng, d, fast) if op == "sum" and rng.random() < 0.25 else None
            aggs.append(Agg(op, fs, gate))
        plan = Plan(terms, keys, aggs)
        if not plan.columns or len(plan.columns) > DY_MAXCOLS or not ops.dense_agg_fits(plan.n_groups, len(aggs)):
            continue
        try:
            compile_plan(plan, d)
        except E.ExprError:
            continue                              # over the per-call node limits: draw again
        return plan
    raise AssertionError("no plan drawn")


# ------------------------------------------------------------------ the dynamic plan's shared-memory rule (host mirror)
DYN_SHAPES = [(128, 4), (256, 4), (256, 2), (128, 8), (128, 2), (128, 1)]       # csrc/scan.cu launch_dyn, preference order
SMEM_CAP = 227 * 1024 - 64


def dyn_ctas_per_sm(row_bytes: int, n_groups: int, nagg: int, nt: int, v: int) -> int:
    """csrc/scan.cu dyn_ctas_per_sm"""
    smem = 3 * row_bytes * nt * v + n_groups * (nagg * 8 + 4) * nt
    if smem > SMEM_CAP:
        return 0
    return min((227 * 1024) // (smem + 1024), 2048 // nt, 6)


def dyn_pick(row_bytes: int, n_groups: int, nagg: int):
    """the (threads, rows) shape launch_dyn picks without QK_DYN_SHAPE, or None when none fits"""
    for nt, v in DYN_SHAPES:
        if dyn_ctas_per_sm(row_bytes, n_groups, nagg, nt, v) >= 2:
            return nt, v
    best, pick = 0, None
    for nt, v in DYN_SHAPES:
        rows = dyn_ctas_per_sm(row_bytes, n_groups, nagg, nt, v) * nt * v
        if rows > best:
            best, pick = rows, (nt, v)
    return pick


def dyn_max_groups(row_bytes: int, nagg: int, nt: int, v: int) -> int:
    """the largest group count shape (nt, v) accepts: dyn_ctas_per_sm > 0 needs smem + 1024 <= 227 KB"""
    ng = (227 * 1024 - 1024 - 3 * row_bytes * nt * v) // ((nagg * 8 + 4) * nt)
    assert dyn_ctas_per_sm(row_bytes, ng, nagg, nt, v) > 0 and dyn_ctas_per_sm(row_bytes, ng + 1, nagg, nt, v) == 0
    return ng


# ------------------------------------------------------------------ routing of dictionary groupings (edge.PartialAgg)
ROUTING_GROUPS = (66, 67, 150, 1024)
ROUTING_AGGS = (0, 1, 2, 4)                      # number of SUMs; 0 = COUNT(*) only
ROUTING_PREDS = ("x > 0.1 and y < 0.9", "x > 0.1 or y > 0.5")       # dyn grammar; an OR tree (interpreter only)


def routing_case(qc, monkeypatch, n_groups: int, nsum: int, pred: str, n: int = 20_000, seed: int = 0):
    """`groupby(<dictionary string column>)` with `n_groups` values and `nsum` SUMs (or COUNT(*) only) behind `pred`,
    collected through the DataStream API and compared with pandas.  Returns the paths edge.PartialAgg took."""
    import pandas as pd
    import pyarrow as pa
    from quokka_b200 import edge
    rng = np.random.default_rng(seed * 7919 + n_groups * 31 + nsum)
    names = [f"t{i:04d}" for i in range(n_groups)]
    codes = np.concatenate([np.arange(n_groups), rng.integers(0, n_groups, n - n_groups)])    # every value occurs
    x, y = rng.random(n), rng.random(n)
    t = pa.table({"k": pa.array([names[i] for i in codes]).dictionary_encode(), "x": x, "y": y})
    paths = []
    call = edge.PartialAgg.__call__

    def spy(self, tbl, e=None):
        out = call(self, tbl, e)
        paths.append(self.last_path)
        return out
    monkeypatch.setattr(edge.PartialAgg, "__call__", spy)
    sql = ", ".join([f"sum(x * {j + 1}) as s{j}" for j in range(nsum)] or ["count(*) as c"])
    got = qc.from_arrow(t).filter_sql(pred).groupby("k").agg_sql(sql).collect().to_pandas()
    df = pd.DataFrame({"k": [names[i] for i in codes], "x": x, "y": y})
    m = (x > 0.1) & (y < 0.9) if " and " in pred else (x > 0.1) | (y > 0.5)
    g = df[m].groupby("k")
    want = pd.DataFrame({f"s{j}": g["x"].apply(lambda s, j=j: math.fsum(s * (j + 1))) for j in range(nsum)}) if nsum \
        else g.size().rename("c").to_frame()
    got = got.assign(k=got["k"].astype(str)).set_index("k").sort_index()
    want = want.sort_index()
    assert list(got.index) == list(want.index), (n_groups, nsum, pred)
    for c in want.columns:
        if nsum:
            np.testing.assert_allclose(got[c].to_numpy(np.float64), want[c].to_numpy(), rtol=1e-12, err_msg=f"{c} {n_groups} {pred}")
        else:
            assert np.array_equal(got[c].to_numpy(np.int64), want[c].to_numpy(np.int64)), (n_groups, pred)
    assert paths, "the partial aggregate never ran"
    return paths
