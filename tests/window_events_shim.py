"""Per-event (OnEventTrigger) tumbling and session windows in numpy: the references the kernel (csrc/window.cu qk_window_running)
is tested against, and the stand-in that window_sliding(..., run=...) of tests/cpu_shim.py calls.

The rows of a key, in time order, are cut into runs -- tumbling: one run per floor(t / size); session: a new run at the key's
first row and after every gap t - t_prev > timeout -- and every row aggregates the rows of its run with time <= its own
(DuckDB's RANGE UNBOUNDED PRECEDING, ts_executors.py:64-96, 109-136, 239-288)."""
from __future__ import annotations

import numpy as np
import torch

from oracle import relops as R

KINDS = ("tumbling", "session")


def run_breaks(prev, t, kind, param):
    """The run boundary between consecutive times of one key.  A session gap is taken as an unsigned difference: the times are
    sorted within a key, and t - prev overflows int64 from -2^62 to +2^62."""
    prev, t = np.asarray(prev, dtype=np.int64), np.asarray(t, dtype=np.int64)
    if kind == "tumbling":
        return (prev // np.int64(param)) != (t // np.int64(param))
    return (t.view(np.uint64) - prev.view(np.uint64)) > np.uint64(param)


def running_window(time, by, kind, param, aggs):
    """One row at a time: every row aggregates the rows of its key and run with time <= its own.  aggs = {name: (op,
    values | None)} as for relops.sliding_window; returns {name: array aligned with the input rows}."""
    time, by = np.asarray(time, dtype=np.int64), np.asarray(by)
    out = {k: np.zeros(len(time)) for k in aggs}
    for key in np.unique(by):
        idx = np.nonzero(by == key)[0]
        idx = idx[np.argsort(time[idx], kind="stable")]
        t = time[idx]
        run = np.concatenate([[0], np.cumsum(run_breaks(t[:-1], t[1:], kind, param))]) if len(t) else np.zeros(0, np.int64)
        for p in range(len(t)):
            m = (run == run[p]) & (t <= t[p])
            for name, (op, v) in aggs.items():
                out[name][idx[p]] = R._agg(op, np.asarray(v)[idx][m]) if v is not None else m.sum()
    return out


def running_window_ranges(time, by, kind, param):
    """(order, lo, hi), vectorised: sorted row r (relops.window_order) aggregates sorted rows [lo[r], hi[r]) -- from its run's
    first row to the last row of its key with its time."""
    order, ts, bs, keys, seg = R.window_order(time, by)
    n = len(ts)
    new = np.ones(n, bool)
    end = np.ones(n, bool)
    if n > 1:
        key_change = bs[1:] != bs[:-1]
        new[1:] = key_change | run_breaks(ts[:-1], ts[1:], kind, param)
        end[:-1] = key_change | (ts[1:] != ts[:-1])
    lo = np.flatnonzero(new)[np.cumsum(new) - 1].astype(np.int64)
    ends = np.flatnonzero(end)
    hi = (ends[np.searchsorted(ends, np.arange(n))] + 1).astype(np.int64)
    return order, lo, hi


def padded(v):
    """v followed by a copy of itself, for relops.range_aggregate over ranges of v: its MIN / MAX sparse table needs the array
    to be at least twice as long as the widest range, and a run can span the whole column.  The ranges never index the copy."""
    v = np.asarray(v, dtype=np.float64)
    return np.concatenate([v, v])


_ACC = {"sum": np.add, "avg": np.add, "min": np.fmin, "max": np.fmax}


def window_running(time, by, seg, n_by, kind, param, vals, aggs):
    """The per-event windows of ops.window_sliding(..., run=kind) with param = its `size`: the ranges above, each run's rows
    folded with ufunc.accumulate in row order."""
    from quokka_b200 import _lib as L
    names = {L.WIN_SUM: "sum", L.WIN_MIN: "min", L.WIN_MAX: "max", L.WIN_COUNT: "count", L.WIN_AVG: "avg"}
    if kind not in (L.WIN_RUN_TUMBLING, L.WIN_RUN_SESSION) or (param <= 0 if kind == L.WIN_RUN_TUMBLING else param < 0):
        raise L.QkError(f"qk_window_running: bad window kind {kind} / parameter {param}")
    t, b = time.numpy(), by.numpy()
    order, lo, hi = running_window_ranges(t, b, "tumbling" if kind == L.WIN_RUN_TUMBLING else "session", int(param))
    starts = np.unique(lo)
    stops = np.append(starts[1:], len(lo))
    outs = []
    for op, src in aggs:
        op = names[op]
        r = np.empty(len(order), dtype=np.float64)
        if op == "count":
            r[order] = hi - lo
        else:
            v = vals[src].numpy().astype(np.float64)[order]
            acc = np.empty(len(v), dtype=np.float64)
            for a, e in zip(starts, stops):
                acc[a:e] = _ACC[op].accumulate(v[a:e])
            got = acc[hi - 1] if len(hi) else acc
            r[order] = got / (hi - lo) if op == "avg" else got
        outs.append(torch.from_numpy(r))
    return outs

