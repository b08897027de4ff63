"""OrderedStream.pattern_recognize: a brute-force restatement of its specification and the API cases that the CPU (shim), gloo and
GPU runs share.

The oracle enumerates EVERY tuple r0 < r1 < ... < r(m-1) of a key's rows (in time order) whose rows satisfy their events'
row-local parts, keeps the tuples that meet the whole specification, and reports per start the smallest time vector -- no pruning,
no resume rule, nothing of the kernel's search."""
from __future__ import annotations

import datetime
import itertools
import os

import numpy as np
import pyarrow as pa

from quokka_b200 import expr as E

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


class _Null(Exception):
    pass


def _value(arrs, name, r):
    v = arrs[name][r]
    if v is None:
        raise _Null()
    return v


def _eval(n, env):
    """fp64 / string value of an expression node; env(col) gives a column's value in the current binding."""
    k = n.kind
    if k == "col":
        return env(n.value)
    if k in ("num", "date"):
        return np.float64(n.value)
    if k == "str":
        return n.value
    if k == "un":
        v = _eval(n.args[0], env)
        return -v if n.value == "neg" else np.float64(v == 0)
    if k == "func" and n.value == "case":
        c = _eval(n.args[0], env)
        return _eval(n.args[1], env) if c != 0 else _eval(n.args[2], env)
    if k == "bin":
        a, b = _eval(n.args[0], env), _eval(n.args[1], env)
        if isinstance(a, str) or isinstance(b, str):
            return np.float64({"=": a == b, "!=": a != b}[n.value])
        with np.errstate(all="ignore"):
            a, b = np.float64(a), np.float64(b)
            return {"+": lambda: a + b, "-": lambda: a - b, "*": lambda: a * b, "/": lambda: a / b,
                    "<": lambda: np.float64(a < b), "<=": lambda: np.float64(a <= b), ">": lambda: np.float64(a > b),
                    ">=": lambda: np.float64(a >= b), "=": lambda: np.float64(a == b), "!=": lambda: np.float64(a != b),
                    "and": lambda: np.float64(a != 0 and b != 0), "or": lambda: np.float64(a != 0 or b != 0)}[n.value]()
    raise ValueError(f"oracle cannot evaluate {n.sql()}")


def pattern_recognize(table: pa.Table, time_col, events, maxspan, by):
    """Sorted list of (key, t0, ..., t(m-1)): one per start row with a match, the match with the smallest (t1 .. t(m-1))."""
    names = [n for n, _ in events]
    m = len(events)
    preds = [None if p is None else E.parse(p) for _, p in events]
    arrs = {c: table[c].to_pylist() for c in table.column_names}
    tvals = table[time_col].cast(pa.int64()) if not pa.types.is_date32(table[time_col].type) else \
        table[time_col].cast(pa.int32()).cast(pa.int64())
    times = tvals.to_pylist()
    if isinstance(maxspan, datetime.timedelta):
        t = table[time_col].type
        per_s = {"s": 1, "ms": 10 ** 3, "us": 10 ** 6, "ns": 10 ** 9}[t.unit] if pa.types.is_timestamp(t) else None
        maxspan = int(maxspan / datetime.timedelta(days=1)) if per_s is None else int(round(maxspan.total_seconds() * per_s))
    keys = arrs[by]

    def holds(e, rows):
        """Event e's whole predicate with rows[0..e] bound; False when it reads a NULL."""
        if preds[e] is None:
            return True

        def where(c):
            q, col = c.split(".", 1) if "." in c else (names[e], c)
            return rows[names.index(q)], col
        try:
            for c in preds[e].columns():                  # a predicate that reads a NULL is false, whatever else it says
                _value(arrs, where(c)[1], where(c)[0])
            return _eval(preds[e], lambda c: _value(arrs, where(c)[1], where(c)[0])) != 0
        except _Null:
            return False

    def local_only(e):
        return preds[e] is None or not any("." in c and c.split(".", 1)[0] != names[e] for c in preds[e].columns())

    out = []
    groups = {}
    for r in range(table.num_rows):
        groups.setdefault(keys[r], []).append(r)
    for key, rows in groups.items():
        rows = sorted(rows, key=lambda r: times[r])            # stable: equal times keep their input order
        for i0, r0 in enumerate(rows):
            if not holds(0, [r0]):
                continue
            t0 = times[r0]
            span = [r for r in rows[i0 + 1:] if times[r] <= t0 + maxspan]
            # the rows each later event could bind on its own (all rows of the span for an event with a link predicate)
            can = [{r for r in span if not local_only(e) or holds(e, [r0] * e + [r])} for e in range(1, m)]
            pool = [r for r in span if any(r in c for c in can)]
            best = None
            for tup in itertools.combinations(pool, m - 1):          # every increasing tuple of rows
                if not all(r in c for r, c in zip(tup, can)):
                    continue
                bound = [r0] + list(tup)
                ts = [times[r] for r in bound]
                if any(ts[j + 1] <= ts[j] for j in range(m - 1)) or ts[-1] > t0 + maxspan:
                    continue
                if not all(holds(e, bound[:e + 1]) for e in range(1, m)):
                    continue
                if best is None or ts[1:] < best[1:]:
                    best = ts
            if best is not None:
                out.append((key, *best))
    return sorted(out, key=lambda x: (str(x[0]), *x[1:]))


def rows_of(res: pa.Table, by, names):
    cols = [res[by].to_pylist()] + [res[n].cast(pa.int64()).to_pylist() if not pa.types.is_date32(res[n].type)
                                    else res[n].cast(pa.int32()).cast(pa.int64()).to_pylist() for n in names]
    return sorted(zip(*cols), key=lambda x: (str(x[0]), *x[1:]))


# ------------------------------------------------------------------ the kernel's inputs
def search(fn, tab, time_col, events, maxspan, by, budget=1 << 30, device="cpu", rows_tested=None):
    """The executor's host path in numpy -- segment by key, row-local candidate bits, link programs -- then the search `fn`
    (ops.pattern_search or the shim's) on `device`; the result in the oracle's form."""
    import torch

    import cpu_shim
    preds = E.split_pattern(events, tab.column_names, by)
    keys = np.asarray(tab[by].to_numpy(zero_copy_only=False))
    uniq, codes = np.unique(keys, return_inverse=True)
    order = np.argsort(codes, kind="stable")
    time = tab[time_col].to_numpy().astype(np.int64)[order]
    codes = codes[order].astype(np.int32)
    seg = np.searchsorted(codes, np.arange(len(uniq) + 1)).astype(np.int64)
    cols = {c: np.asarray(tab[c].to_numpy(zero_copy_only=False))[order] for c in preds.columns}
    valid = {c: np.asarray(tab[c].is_valid().to_numpy(zero_copy_only=False))[order].astype(np.uint8) for c in preds.columns
             if tab[c].null_count}
    vals = {c: np.nan_to_num(np.asarray(v, dtype=np.float64)) if c in valid else v for c, v in cols.items()}
    n, m = len(time), len(events)
    cand = np.zeros(n, np.uint8)
    from quokka_b200.columns import DeviceColumn, DeviceTable
    sch = DeviceTable({c: DeviceColumn(torch.from_numpy(np.ascontiguousarray(v))) for c, v in vals.items()}).schema_info()
    for e, node in enumerate(preds.local):
        if node is None:
            cand |= np.uint8(1 << e)
            continue
        ok = cpu_shim.eval_prog(E.compile_expr(node, sch), [vals[c] for c in sch], n) != 0
        for c in node.columns():
            if c in valid:
                ok &= valid[c].astype(bool)
        cand |= (ok.astype(np.uint8) << e)
    lcols, links = E.compile_links(preds, sch)
    starts = np.nonzero(cand & 1)[0].astype(np.int32)
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(device)
    out = fn(d(time), d(codes), d(seg), len(uniq), d(cand), d(starts), m, maxspan, [d(vals[c]) for c in lcols],
             [d(valid[c]) if c in valid else None for c in lcols], links, budget, rows_tested).cpu().numpy()
    got = [(uniq[codes[b[0]]].item(), *[int(time[r]) for r in b]) for b in out if b[0] >= 0]
    return sorted(got, key=lambda x: (str(x[0]), *x[1:]))


# ------------------------------------------------------------------ generators
def random_stream(seed, n=60, keys=3, tmax=40, m=3, nulls=False):
    """Dense ties: few keys, times drawn from a small range, integer-valued prices."""
    rng = np.random.default_rng(seed)
    t = np.sort(rng.integers(0, tmax, n)).astype(np.int64)
    tab = {"time": t, "sym": rng.integers(0, keys, n).astype(np.int64), "px": rng.integers(0, 10, n).astype(np.float64),
           "sz": rng.integers(0, 5, n).astype(np.int64)}
    tab = pa.table(tab)
    if nulls:
        px = tab["px"].to_pylist()
        px = [None if rng.random() < 0.15 else v for v in px]
        tab = tab.set_column(2, "px", pa.array(px, pa.float64()))
    return tab


def random_events(seed, m):
    rng = np.random.default_rng(seed)
    names = ["a", "b", "c", "d", "e", "f", "g", "h"][:m]
    ev = [("a", None if rng.random() < 0.3 else f"px >= {int(rng.integers(0, 6))}")]
    for i in range(1, m):
        opts = [f"px < {int(rng.integers(3, 10))}", f"sz != {int(rng.integers(0, 5))}",
                f"{names[i]}.px > {names[int(rng.integers(0, i))]}.px", f"px + sz >= {names[int(rng.integers(0, i))]}.px",
                f"px * 2 <= {names[i - 1]}.px + 6", f"case when {names[0]}.sz > 2 then px > 3 else px <= 5 end"]
        k = int(rng.integers(1, 3))
        ev.append((names[i], " and ".join(rng.choice(opts, size=k, replace=False))))
    return ev


def tie_stream(seed, n=24, tmax=10):
    """One key, many rows per timestamp, values that make tied rows lead to different completions."""
    rng = np.random.default_rng(seed)
    return pa.table({"time": np.sort(rng.integers(0, tmax, n)).astype(np.int64), "sym": np.zeros(n, np.int64),
                     "px": rng.integers(0, 6, n).astype(np.float64), "sz": rng.integers(0, 3, n).astype(np.int64)})


def tie_events(seed, m):
    """Chained link programs (each event reads the one before), so that no level is independent and the caps matter."""
    rng = np.random.default_rng(seed)
    names = ["a", "b", "c", "d", "e", "f", "g", "h"][:m]
    ev = [("a", None)]
    for i in range(1, m):
        p = names[i - 1]
        ev.append((names[i], str(rng.choice([f"{names[i]}.px > {p}.px", f"px < {p}.px + 2 and px != {p}.px",
                                               f"px + {p}.sz >= {p}.px", f"px = {p}.px + 1"]))))
    return ev


# ------------------------------------------------------------------ API cases
def _quotes():
    g = np.load(os.path.join(GOLDEN, "asof2.npz"))
    syms = np.array([f"S{i:04d}" for i in range(int(g["q_sym"].max()) + 1)], dtype=object)
    return pa.table({"time": g["q_time"], "symbol": pa.array(list(syms[g["q_sym"]])), "asize": g["q_asize"]})


def check(qc, table, time_col, events, maxspan, by, chunks=(1 << 26,), expect=None):
    """The API result for every batch size in `chunks` equals the oracle (and `expect` when given)."""
    want = pattern_recognize(table, time_col, events, maxspan, by)
    if expect is not None:
        assert want == expect, (want, expect)
    names = [n for n, _ in events]
    for chunk in chunks:
        qc.set_config("chunk_rows", chunk)
        try:
            res = qc.from_arrow_sorted(table, time_col).pattern_recognize(time_col, events, maxspan, by).collect()
        finally:
            qc.set_config("chunk_rows", 1 << 26)
        assert res.column_names == [by] + names, res.column_names
        assert rows_of(res, by, names) == want, (chunk, rows_of(res, by, names)[:5], want[:5])
    return want


def case_blog_asize(qc):
    """The announcement's three-event pattern (blog/orderedstreams.md:76-102) on the as-of fixture's quotes, with thresholds from
    the data's quantiles, batched three ways."""
    q = _quotes()
    hi, lo = (float(np.quantile(q["asize"].to_numpy(), x)) for x in (0.8, 0.2))
    ev = [("a", f"asize > {hi}"), ("b", f"asize < {lo}"), ("c", f"asize > {hi}")]
    got = check(qc, q, "time", ev, 300, "symbol", chunks=(1 << 26, 500, 97))
    assert len(got) > 10


def case_link_predicates(qc):
    q = _quotes()
    ev = [("a", "asize > 0"), ("b", "b.asize > a.asize * 1.005"), ("c", "asize < a.asize - b.asize and c.asize + a.asize > 0")]
    got = check(qc, q, "time", ev, 400, "symbol", chunks=(1 << 26, 333))
    assert got


def case_first_event_any_row(qc):
    q = _quotes()
    check(qc, q, "time", [("a", None), ("b", "asize > 1.5")], 50, "symbol")


def case_maxspan_boundary(qc):
    t = pa.table({"t": np.array([0, 5, 10, 20], np.int64), "k": np.zeros(4, np.int64), "v": np.array([1.0, 2.0, 3.0, 4.0])})
    ev = [("a", "v = 1"), ("b", "v = 3")]
    check(qc, t, "t", ev, 10, "k", expect=[(0, 0, 10)])            # t(b) = t0 + maxspan is in
    check(qc, t, "t", ev, 9, "k", expect=[])                       # one tick less: out


def case_equal_times(qc):
    """Equal timestamps never chain (strictly increasing times), and among tied rows the lexicographic rule decides, not row
    order: of the two b rows at time 2, v = 10 leads to a c at 5 (v = 15) and v = 20 only to a c at 9 (v = 25).  A search that
    kept the first match it finds would answer (2, 9) when the v = 20 row comes first."""
    t = pa.table({"t": np.array([1, 1, 2, 2, 5, 9], np.int64), "k": np.zeros(6, np.int64),
                  "v": np.array([1.0, 2.0, 10.0, 20.0, 15.0, 25.0])})
    ev = [("a", "v = 1"), ("b", "v >= 2"), ("c", "c.v > b.v")]
    got = check(qc, t, "t", ev, 100, "k", chunks=(1 << 26, 2), expect=[(0, 1, 2, 5)])
    rev = t.take(pa.array([0, 1, 3, 2, 4, 5]))                     # the tied rows in the other order: the same answer
    check(qc, rev, "t", ev, 100, "k", chunks=(1 << 26, 2), expect=got)


CAP_TABLE = dict(t=[1, 2, 2, 3, 5, 9, 12], v=[100.0, 10.0, 0.0, 5.0, 15.0, 16.0, 6.0])
CAP_EVENTS = [("a", "v = 100"), ("b", "v < 50"), ("c", "c.v > b.v and c.v < 50"), ("d", "d.v = c.v + 1")]


def case_lexicographic_cap(qc):
    """The caps of the best match hold only while the levels above equal it.  The first b (t = 2, v = 10) gives (2, 5, 9); the
    tied b (t = 2, v = 0) binds c at 3 < 5, and from there d may lie beyond the best's d: (2, 3, 12) is smaller.  Capping d at 9
    anyway would keep (2, 5, 9)."""
    t = pa.table({"t": np.array(CAP_TABLE["t"], np.int64), "k": np.zeros(7, np.int64), "v": np.array(CAP_TABLE["v"])})
    got = check(qc, t, "t", CAP_EVENTS, 20, "k", chunks=(1 << 26, 3), expect=[(0, 1, 2, 3, 12)])
    rev = t.take(pa.array([0, 2, 1, 3, 4, 5, 6]))
    check(qc, rev, "t", CAP_EVENTS, 20, "k", expect=got)


def case_string_by(qc):
    q = _quotes()
    check(qc, q, "time", [("x", "asize < -1"), ("y", "asize > 1"), ("z", "asize < z.asize")], 200, "symbol")


def case_timestamp_timedelta(qc):
    q = _quotes()
    ts = pa.array(q["time"].to_numpy() * 1000, pa.timestamp("ms"))
    t = pa.table({"ts": ts, "symbol": q["symbol"], "asize": q["asize"]})
    ev = [("a", "asize > 1"), ("b", "asize < 0")]
    got = check(qc, t, "ts", ev, datetime.timedelta(seconds=40), "symbol")
    assert got == pattern_recognize(t, "ts", ev, 40_000, "symbol")


def case_asof_nulls(qc):
    """An as-of join's unmatched rows carry NULL quote columns; a predicate that reads one is false, in the row itself or in a
    row bound earlier."""
    g = np.load(os.path.join(GOLDEN, "asof2.npz"))
    syms = np.array([f"S{i:04d}" for i in range(int(max(g["t_sym"].max(), g["q_sym"].max())) + 1)], dtype=object)
    trades = pa.table({"time": g["t_time"], "symbol": pa.array(list(syms[g["t_sym"]])), "size": g["t_size"]})
    quotes = pa.table({"time": g["q_time"], "symbol": pa.array(list(syms[g["q_sym"]])), "asize": g["q_asize"]})
    joined = qc.from_arrow_sorted(trades, "time").join_asof(qc.from_arrow_sorted(quotes, "time"), on="time", by="symbol").collect()
    assert joined["asize"].null_count > 0
    ev = [("a", "size > 0"), ("b", "asize > 0 and size < a.size"), ("c", "c.asize < b.asize")]
    want = pattern_recognize(joined, "time", ev, 500, "symbol")
    res = qc.from_arrow_sorted(trades, "time").join_asof(qc.from_arrow_sorted(quotes, "time"), on="time", by="symbol") \
        .pattern_recognize("time", ev, 500, "symbol").collect()
    assert rows_of(res, "symbol", ["a", "b", "c"]) == want and want


def case_no_match(qc):
    q = _quotes()
    res = qc.from_arrow_sorted(q, "time").pattern_recognize("time", [("a", "asize > 100"), ("b", "asize < 0")], 10, "symbol").collect()
    assert res.num_rows == 0 and res.column_names == ["symbol", "a", "b"]


def case_empty_stream(qc):
    t = pa.table({"t": pa.array([], pa.int64()), "k": pa.array([], pa.int64()), "v": pa.array([], pa.float64())})
    res = qc.from_arrow_sorted(t, "t").pattern_recognize("t", [("a", "v > 0"), ("b", "v < 0")], 10, "k").collect()
    assert res.num_rows == 0 and res.column_names == ["k", "a", "b"]


def case_ragged_batches(qc):
    tab = random_stream(11, n=400, keys=4, tmax=200)
    ev = [("a", "px >= 5"), ("b", "b.px < a.px"), ("c", "px > b.px and sz != 0")]
    want = check(qc, tab, "time", ev, 20, "sym", chunks=(1 << 26, 1, 7, 64, 399))
    assert want


def case_unsorted_raises(qc):
    import pytest
    from quokka_b200 import _lib as L
    t = pa.table({"t": np.array([3, 1, 2], np.int64), "k": np.zeros(3, np.int64), "v": np.ones(3)})
    with pytest.raises(L.QkError, match="not sorted"):
        qc.from_arrow_sorted(t, "t").pattern_recognize("t", [("a", "v > 0"), ("b", "v > 0")], 10, "k").collect()


API_CASES = [case_blog_asize, case_link_predicates, case_first_event_any_row, case_maxspan_boundary, case_equal_times,
             case_lexicographic_cap,
             case_string_by, case_timestamp_timedelta, case_asof_nulls, case_no_match, case_empty_stream, case_ragged_batches]
# one rank alone: the error is raised on the rank that holds the unsorted key, and the other ranks would wait for it
SINGLE_RANK_CASES = [case_unsorted_raises]
