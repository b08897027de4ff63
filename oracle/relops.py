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


def asof_backward_fast(l_time, l_by, r_time, r_by):
    """asof_backward without the per-key loop, for many keys: (by, time) packed into one int64 (by < 2^22, 0 <= time < 2^40),
    the right side sorted by it (input order among equals), one searchsorted for all left rows."""
    l_time, r_time = np.asarray(l_time, dtype=np.int64), np.asarray(r_time, dtype=np.int64)
    l_by, r_by = np.asarray(l_by, dtype=np.int64), np.asarray(r_by, dtype=np.int64)
    for t, b in ((l_time, l_by), (r_time, r_by)):
        assert not len(t) or (t.min() >= 0 and t.max() < 2 ** 40 and b.min() >= 0 and b.max() < 2 ** 22), "outside the packed range"
    r_key = (r_by << 40) | r_time
    r_order = np.argsort(r_key, kind="stable")
    rk = r_key[r_order]
    j = np.searchsorted(rk, (l_by << 40) | l_time, side="right") - 1      # the last right row with key <= (by, t)
    jc = np.maximum(j, 0)
    ok = (j >= 0) & (rk[jc] >> 40 == l_by) if len(rk) else np.zeros(len(l_time), bool)
    return np.where(ok, r_order[jc] if len(rk) else -1, -1).astype(np.int64)


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


# ------------------------------------------------------------------ vectorised windows (same results as the three above)
# The functions above loop per row in Python.  These give the same answers at test sizes: the rows are put in (key, time)
# order, every window becomes a row range [lo, hi) of that order (searchsorted, one call per key at most), and the ranges
# are aggregated with prefix sums (SUM / COUNT / AVG) and a sparse table (MIN / MAX).  SUM is exact for values that are
# integer multiples of 2^-63 below 2^40 in magnitude (see range_sum_exact), so the references make no rounding error of
# their own beyond the final conversion to fp64.
def window_order(time, by):
    """(order, sorted time, sorted by, key values, segment starts [nkeys + 1]): the rows by key, then time, then input order."""
    time, by = np.asarray(time, dtype=np.int64), np.asarray(by)
    order = np.lexsort((time, by))
    ts, bs = time[order], by[order]
    keys, starts = np.unique(bs, return_index=True)
    return order, ts, bs, keys, np.append(starts, len(bs)).astype(np.int64)


def _per_key_searchsorted(ts, seg, key_pos, x, side):
    """For every query x[j] of key number key_pos[j] (queries grouped by key): seg start + searchsorted in that key's times."""
    out = np.empty(len(x), dtype=np.int64)
    if not len(x):
        return out
    cut = np.flatnonzero(np.diff(key_pos)) + 1
    for a, b in zip(np.concatenate([[0], cut]), np.concatenate([cut, [len(x)]])):
        s0, s1 = seg[key_pos[a]], seg[key_pos[a] + 1]
        out[a:b] = s0 + np.searchsorted(ts[s0:s1], x[a:b], side=side)
    return out


def sliding_window_ranges(time, by, size):
    """(order, lo, hi): sorted row r aggregates sorted rows [lo[r], hi[r]) -- its key's rows with time in (t - size, t]."""
    order, ts, bs, keys, seg = window_order(time, by)
    kp = np.searchsorted(keys, bs)
    return order, _per_key_searchsorted(ts, seg, kp, ts - np.int64(size), "right"), _per_key_searchsorted(ts, seg, kp, ts, "right")


def hopping_window_ranges(time, by, size, hop):
    """(order, key, start, lo, hi) of every non-empty window [start, start + size), start = k * hop >= the key's first time
    truncated to hop, ordered by key and start.  Candidates: for every row the windows k * hop <= t whose start is at most
    ceil(size / hop) hops back, which covers every window that holds a row; membership is then decided by searchsorted."""
    order, ts, bs, keys, seg = window_order(time, by)
    hop, size = np.int64(hop), np.int64(size)
    slots = int(-(-size // hop))
    kp = np.searchsorted(keys, bs)
    k = (ts // hop)[:, None] - np.arange(slots, dtype=np.int64)[None, :]
    kk = np.repeat(kp, slots)
    k = k.reshape(-1)
    first = (ts[seg[:-1]] // hop) if len(keys) else np.zeros(0, np.int64)
    keep = k >= first[kk]
    kk, k = kk[keep], k[keep]
    o = np.lexsort((k, kk))
    kk, k = kk[o], k[o]
    new = np.ones(len(k), bool)
    new[1:] = (kk[1:] != kk[:-1]) | (k[1:] != k[:-1])
    kk, start = kk[new], k[new] * hop
    lo = _per_key_searchsorted(ts, seg, kk, start, "left")
    hi = _per_key_searchsorted(ts, seg, kk, start + size, "left")
    ne = hi > lo
    return order, keys[kk[ne]], start[ne], lo[ne], hi[ne]


def session_window_ranges(time, by, timeout):
    """(order, key, start time, lo, hi) of every session, ordered by key and start: a key's rows split at gaps > timeout."""
    order, ts, bs, keys, seg = window_order(time, by)
    n = len(ts)
    new = np.ones(n, bool)
    new[1:] = (bs[1:] != bs[:-1]) | ((ts[1:] - ts[:-1]) > timeout)
    lo = np.flatnonzero(new).astype(np.int64)
    hi = np.append(lo[1:], n).astype(np.int64)
    return order, bs[lo], ts[lo], lo, hi


def range_sum_exact(v, lo, hi):
    """Sums of v[lo:hi] as np.longdouble, exact up to the final rounding to long double.  Every value is split into its
    integer part and its fraction scaled by 2^63 (two int64 limbs); int64 prefix sums of the three parts are exact.
    Requires |v| < 2^40 and v an integer multiple of 2^-63 (true of every fp64 with |v| >= 2^-11)."""
    v = np.asarray(v, dtype=np.float64)
    a = np.trunc(v)
    f = (v - a) * 2.0 ** 63                       # v - trunc(v) is exact; scaling by a power of two too
    assert np.all(np.abs(v) < 2.0 ** 40) and np.all(f == np.trunc(f)), "values outside the exact range of range_sum_exact"
    fi = f.astype(np.int64)
    fh = fi >> 31
    fl = fi - (fh << 31)
    sums = []
    for part in (a.astype(np.int64), fh, fl):
        p = np.concatenate([[0], np.cumsum(part)])
        sums.append((p[hi] - p[lo]).astype(np.longdouble))
    return sums[0] + sums[1] * np.longdouble(2.0 ** -32) + sums[2] * np.longdouble(2.0 ** -63)


def range_minmax(v, lo, hi, fn):
    """fn (np.minimum / np.maximum) over v[lo:hi] for non-empty ranges: sparse table, one level at a time (O(n) memory)."""
    v = np.asarray(v, dtype=np.float64)
    out = np.empty(len(lo), dtype=np.float64)
    if not len(lo):
        return out
    w = hi - lo
    assert np.all(w > 0)
    level = np.frexp(w.astype(np.float64))[1] - 1          # floor(log2(w))
    cur = v
    for j in range(int(level.max()) + 1):
        q = np.flatnonzero(level == j)
        out[q] = fn(cur[lo[q]], cur[hi[q] - (1 << j)])      # two overlapping blocks of 2^j rows
        cur = fn(cur[:len(cur) - (1 << j)], cur[(1 << j):])  # cur[i] = fn over v[i : i + 2^(j+1)]
    return out


def range_aggregate(op, v, lo, hi):
    """op over v[lo:hi] for every range (v in the order lo / hi index; None for COUNT): fp64, one rounding for SUM / AVG."""
    if op == "count":
        return (hi - lo).astype(np.float64)
    if op in ("min", "max"):
        return range_minmax(v, lo, hi, np.minimum if op == "min" else np.maximum)
    s = range_sum_exact(v, lo, hi).astype(np.float64)
    return s if op == "sum" else s / (hi - lo)


def sliding_window_fast(time, by, size, aggs):
    """sliding_window, vectorised: {name: fp64 array aligned with the input rows}."""
    order, lo, hi = sliding_window_ranges(time, by, size)
    out = {}
    for name, (op, v) in aggs.items():
        r = np.empty(len(order), dtype=np.float64)
        r[order] = range_aggregate(op, None if v is None else np.asarray(v)[order], lo, hi)
        out[name] = r
    return out


def _grouped(ranges, aggs):
    order, key, start, lo, hi = ranges
    out = {"by": key, "start": start}
    for name, (op, v) in aggs.items():
        out[name] = range_aggregate(op, None if v is None else np.asarray(v)[order], lo, hi)
    return out


def hopping_window_fast(time, by, size, hop, aggs):
    """hopping_window, vectorised: {"by", "start", name...}, one row per non-empty window, ordered by key and start."""
    return _grouped(hopping_window_ranges(time, by, size, hop), aggs)


def session_window_fast(time, by, timeout, aggs):
    """session_window, vectorised: {"by", "start", name...}, one row per session, ordered by key and start."""
    return _grouped(session_window_ranges(time, by, timeout), aggs)
