"""numpy restatement of the reference's relational operators on the hot path.
TEST INFRASTRUCTURE -- see oracle/__init__.py.  Reference paths are relative to a checkout of the reference.

Each function cites the reference code whose observable behaviour it restates.  The reference
delegates the arithmetic to Polars / DuckDB / Arrow (absent here); what is restated is the
*relational semantics at the Executor / partitioner boundary*, with numpy doing the arithmetic:
integer keys bit-exact, fp64 in IEEE double like the reference engines.
"""
from __future__ import annotations

import numpy as np


# ------------------------------------------------------------------ partitioner
def hash_partition(key: np.ndarray, n: int) -> np.ndarray:
    """Target channel of every row.  pyquokka/quokka_runtime.py:217-231 (`partition_key_str`):
    integer keys go to channel `key % num_target_channels`."""
    assert np.issubdtype(key.dtype, np.integer), "only integer keys are pinned by the reference"
    return (key.astype(np.int64) % n).astype(np.int32)


def partition_table(cols: dict, key: str, n: int) -> dict:
    """{channel: cols} with row order preserved inside a channel (Polars partition_by keeps order;
    quokka_runtime.py:222,226-228).  Channels that receive no rows are absent from the dict."""
    p = hash_partition(cols[key], n)
    out = {}
    for ch in range(n):
        m = p == ch
        if m.any():
            out[ch] = {c: v[m] for c, v in cols.items()}
    return out


# ------------------------------------------------------------------ join
def join_indices(left_key: np.ndarray, right_key: np.ndarray, how: str = "inner"):
    """Row-index form of `batch.join(state, left_on, right_on, how)` --
    pyquokka/executors/sql_executors.py:371 (probe = left = stream 0, build = right = stream 1).
    Returns (left_idx, right_idx); right_idx is -1 for unmatched rows of a left join and None for
    semi / anti.  Duplicate build keys multiply rows (Polars semantics).  Output is ordered by
    left row, then by build row order among equal keys."""
    assert how in {"inner", "left", "semi", "anti"}            # sql_executors.py:341
    order = np.argsort(right_key, kind="stable")
    rk = right_key[order]
    lo = np.searchsorted(rk, left_key, side="left")
    hi = np.searchsorted(rk, left_key, side="right")
    cnt = hi - lo
    if how == "semi":
        return np.nonzero(cnt > 0)[0], None
    if how == "anti":
        return np.nonzero(cnt == 0)[0], None
    emit = cnt.copy()
    if how == "left":
        emit = np.maximum(cnt, 1)
    total = int(emit.sum())
    left_idx = np.repeat(np.arange(len(left_key)), emit)
    starts = np.cumsum(emit) - emit
    within = np.arange(total) - np.repeat(starts, emit)
    pos = np.repeat(lo, emit) + within
    right_idx = np.full(total, -1, dtype=np.int64)
    matched = np.repeat(cnt > 0, emit)
    right_idx[matched] = order[pos[matched]]
    return left_idx, right_idx


def join_tables(left: dict, right: dict, left_on: str, right_on: str, how: str = "inner",
                suffix: str = "_2", key_to_keep: str = "left") -> dict:
    """Column-level join result: left columns, then right columns minus the right key, clashing
    names get `suffix` (pyquokka/datastream.py:1506-1519); `key_to_keep == "right"` renames the
    surviving key (sql_executors.py:372-373).  Empty build side: anti passes the probe through,
    everything else emits nothing (sql_executors.py:362-366) -- falls out of join_indices."""
    li, ri = join_indices(left[left_on], right[right_on], how)
    out = {c: v[li] for c, v in left.items()}
    if ri is not None:
        for c, v in right.items():
            if c == right_on:
                continue
            name = c + suffix if c in out else c
            g = v[np.maximum(ri, 0)]
            if how == "left" and (ri < 0).any():
                g = np.ma.masked_array(g, mask=ri < 0)
            out[name] = g
    if key_to_keep == "right" and left_on != right_on:
        out = {(right_on if c == left_on else c): v for c, v in out.items()}
    return out


# ------------------------------------------------------------------ group-by aggregate
def group_ids(keys: list):
    """Dense group id per row + the unique key tuples, sorted lexicographically by key."""
    n = len(keys[0])
    if n == 0:
        return np.zeros(0, np.int64), [k[:0] for k in keys]
    order = np.lexsort(keys[::-1])
    sk = [k[order] for k in keys]
    new = np.zeros(n, dtype=bool)
    new[0] = True
    for k in sk:
        new[1:] |= k[1:] != k[:-1]
    gid_sorted = np.cumsum(new) - 1
    gid = np.empty(n, dtype=np.int64)
    gid[order] = gid_sorted
    uniq = [k[new] for k in sk]
    return gid, uniq


def group_aggregate(keys: dict, aggs: dict) -> dict:
    """Two-phase aggregate of DataStream._grouped_aggregate_sql (pyquokka/datastream.py:1819-1856)
    collapsed to its result: `select keys, AGG(...) group by keys` (SQLAggExecutor,
    sql_executors.py:556-599).  `aggs` maps output name -> (op, values) with op in
    sum|min|max|count|avg; avg is SUM(x)/COUNT(*) as the reference rewrites it
    (pyquokka/sql_utils.py:337-351)."""
    names = list(keys)
    gid, uniq = group_ids([keys[k] for k in names])
    ng = len(uniq[0]) if names else (1 if len(gid) or not names else 0)
    if not names:
        n_rows = len(next(iter(aggs.values()))[1]) if aggs else 0
        gid = np.zeros(n_rows, np.int64)
        ng = 1
    out = {k: u for k, u in zip(names, uniq)}
    cnt = np.bincount(gid, minlength=ng).astype(np.int64)
    for name, (op, vals) in aggs.items():
        if op == "count":
            out[name] = cnt.copy()
        elif op == "sum":
            out[name] = np.bincount(gid, weights=vals.astype(np.float64), minlength=ng)
        elif op == "avg":
            out[name] = np.bincount(gid, weights=vals.astype(np.float64), minlength=ng) / cnt
        elif op in ("min", "max"):
            init = np.inf if op == "min" else -np.inf
            acc = np.full(ng, init)
            (np.minimum if op == "min" else np.maximum).at(acc, gid, vals.astype(np.float64))
            out[name] = acc
        else:
            raise ValueError(op)
    return out


def sum_exact_int(gid: np.ndarray, vals: np.ndarray, ng: int) -> np.ndarray:
    """Integer sums without fp rounding (for the as-of checksum, apps/tpc-h/range.py:15)."""
    acc = np.zeros(ng, dtype=np.int64)
    np.add.at(acc, gid, vals.astype(np.int64))
    return acc


# ------------------------------------------------------------------ top-k
def top_k(cols: dict, by: list, k: int, descending: list | None = None) -> dict:
    """`select * order by ... limit k` -- DataStream.top_k, pyquokka/datastream.py:1702-1767
    (per batch, then once more on one channel; the composition equals one global top-k)."""
    descending = descending or [False] * len(by)
    keys = []
    for c, d in zip(by, descending):
        v = cols[c]
        keys.append(-v.astype(np.float64) if d and v.dtype.kind == "f" else (-v if d else v))
    order = np.lexsort(keys[::-1])[:k]
    return {c: v[order] for c, v in cols.items()}


# ------------------------------------------------------------------ as-of join
def asof_backward(l_time: np.ndarray, l_by: np.ndarray, r_time: np.ndarray, r_by: np.ndarray):
    """Backward as-of match per `by` key: for every left row the index of the LAST right row with
    the same `by` and r_time <= l_time, else -1.  Polars `join_asof(strategy="backward", by=...)`
    as called by SortedAsofExecutor (pyquokka/executors/ts_executors.py:369,383); among equal right
    timestamps the last row wins (pandas / Polars behaviour, SURVEY.md section 4)."""
    out = np.full(len(l_time), -1, dtype=np.int64)
    r_order = np.lexsort((np.arange(len(r_time)), r_time, r_by))      # by, time, original order
    rb, rt = r_by[r_order], r_time[r_order]
    # segment of each by-key in the sorted right side
    keys, starts = np.unique(rb, return_index=True)
    ends = np.append(starts[1:], len(rb))
    pos = np.searchsorted(keys, l_by)
    pos_c = np.minimum(pos, len(keys) - 1) if len(keys) else pos
    has = (pos < len(keys)) & (keys[pos_c] == l_by) if len(keys) else np.zeros(len(l_by), bool)
    for s in np.unique(pos_c[has]) if len(keys) else []:
        rows = np.nonzero(has & (pos_c == s))[0]
        seg_t = rt[starts[s]:ends[s]]
        j = np.searchsorted(seg_t, l_time[rows], side="right") - 1
        ok = j >= 0
        out[rows[ok]] = r_order[starts[s] + j[ok]]
    return out


# ------------------------------------------------------------------ aggregate decomposition strings
def decompose_aggregations(aggs: list):
    """Restates parse_multiple_aggregations (pyquokka/sql_utils.py:379-413) for the plain
    `FUNC(arg) as alias` forms: returns (partial list, final list, aliases) as the reference names
    them (`e{i}_agg_{j}`), avg -> SUM + COUNT(*).  `aggs` = [(func, arg_sql, alias)]."""
    partial, final, aliases = [], [], []
    for i, (func, arg, alias) in enumerate(aggs):
        p = f"e{i}_"
        f = func.lower()
        if f == "avg":
            partial += [f"SUM({arg}) as {p}agg_0", f"COUNT(*) as {p}agg_1"]
            final.append(f"(SUM({p}agg_0) / SUM({p}agg_1)) AS {alias}")
        elif f == "count":
            partial.append(f"COUNT({arg}) as {p}agg_0")
            final.append(f"SUM({p}agg_0) AS {alias}")
        else:
            partial.append(f"{f.upper()}({arg}) as {p}agg_0")
            final.append(f"{f.upper()}({p}agg_0) AS {alias}")
        aliases.append(alias)
    return ",".join(partial), ",".join(final), aliases


# ------------------------------------------------------------------ time-series windows (ts_executors.py:12-288)
def _agg(op, v):
    return {"sum": np.sum, "min": np.min, "max": np.max, "avg": np.mean, "count": len}[op](v)


def sliding_window(time, by, size, aggs):
    """Polars groupby_rolling(time, period=size, by=by) as SlidingWindowExecutor uses it (ts_executors.py:183): for every
    row, aggregates over the rows of the same key with time in (t - size, t].  aggs = {name: (op, values | None)}.
    Returns {name: array aligned with the input rows}."""
    time, by = np.asarray(time), np.asarray(by)
    out = {k: np.zeros(len(time)) for k in aggs}
    for key in np.unique(by):
        idx = np.nonzero(by == key)[0]
        t = time[idx]
        lo = np.searchsorted(t, t - size, side="right")
        hi = np.searchsorted(t, t, side="right")
        for name, (op, v) in aggs.items():
            vv = None if v is None else np.asarray(v)[idx]
            out[name][idx] = [(_agg(op, vv[a:b]) if vv is not None else b - a) for a, b in zip(lo, hi)]
    return out


def hopping_window(time, by, size, hop, aggs):
    """Polars groupby_dynamic(time, every=hop, period=size, by=by) as HoppingWindowExecutor uses it (ts_executors.py:62):
    windows [k * hop, k * hop + size), closed left, labelled by their start; per key the first window starts at the key's
    first timestamp truncated to `hop`; empty windows are not reported.  Returns {"by", "start", name...} (one row per window)."""
    time, by = np.asarray(time), np.asarray(by)
    rows = {"by": [], "start": [], **{k: [] for k in aggs}}
    for key in np.unique(by):
        idx = np.nonzero(by == key)[0]
        t = time[idx]
        first = (t[0] // hop) * hop
        last = (t[-1] // hop) * hop
        for start in range(int(first), int(last) + 1, int(hop)):
            a, b = np.searchsorted(t, start, side="left"), np.searchsorted(t, start + size, side="left")
            if b <= a:
                continue
            rows["by"].append(key); rows["start"].append(start)
            for name, (op, v) in aggs.items():
                rows[name].append(_agg(op, np.asarray(v)[idx][a:b]) if v is not None else b - a)
    return {k: np.array(v) for k, v in rows.items()}


def session_window(time, by, timeout, aggs):
    """SessionWindowExecutor (ts_executors.py:215-236): per key, consecutive rows belong to one session while their gap is
    <= timeout.  Returns {"by", "start", name...} (one row per session)."""
    time, by = np.asarray(time), np.asarray(by)
    rows = {"by": [], "start": [], **{k: [] for k in aggs}}
    for key in np.unique(by):
        idx = np.nonzero(by == key)[0]
        t = time[idx]
        cuts = np.concatenate([[0], np.nonzero(np.diff(t) > timeout)[0] + 1, [len(t)]])
        for a, b in zip(cuts[:-1], cuts[1:]):
            rows["by"].append(key); rows["start"].append(t[a])
            for name, (op, v) in aggs.items():
                rows[name].append(_agg(op, np.asarray(v)[idx][a:b]) if v is not None else b - a)
    return {k: np.array(v) for k, v in rows.items()}
