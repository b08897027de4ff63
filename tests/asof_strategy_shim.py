"""TEST-ONLY numpy statements of the as-of strategies (csrc/asof.cu qk_asof_join, qk_asof_search_join).  `asof_join` is the
plain restatement of pandas.merge_asof(direction=strategy, tolerance=tolerance) that the other tests compare against;
`merge_join` states what the merge kernel returns with its carry tables.  The asof_merge and asof_backward of
tests/cpu_shim.py answer with them when given a `strategy=` / `tolerance=`, so OrderedStream.join_asof(strategy=...) runs
through the planner, the executors and the gloo exchange without a GPU.  The GPU tests compare both kernels with these, bit
for bit."""
from __future__ import annotations

import numpy as np

STRATEGIES = ("backward", "forward", "nearest")


def _dist(a, b):
    """|a - b| of int64 arrays, exact over the whole int64 range (as uint64)."""
    a, b = np.asarray(a, np.int64), np.asarray(b, np.int64)
    return np.where(a < b, b.view(np.uint64) - a.view(np.uint64), a.view(np.uint64) - b.view(np.uint64))


def candidates(l_time, l_by, r_time, r_by):
    """(back, fwd): per left row the LAST right row of its key with r_time <= l_time and the FIRST with r_time >= l_time (-1
    none), right rows in stream order.  Keys and times are ranked into one int64 composite, so one stable sort serves all."""
    lt, lb = np.asarray(l_time, np.int64), np.asarray(l_by, np.int64)
    rt, rb = np.asarray(r_time, np.int64), np.asarray(r_by, np.int64)
    times = np.unique(np.concatenate([lt, rt]))
    width = np.int64(len(times) + 1)
    lc = lb * width + np.searchsorted(times, lt)
    rc = rb * width + np.searchsorted(times, rt)
    order = np.argsort(rc, kind="stable")               # by key, then time, then stream order
    rs = rc[order]
    hi = np.searchsorted(rs, lc, side="right")
    lo = np.searchsorted(rs, lc, side="left")
    back = np.full(len(lt), -1, np.int64)
    fwd = np.full(len(lt), -1, np.int64)
    ok = hi > 0
    ok[ok] = rb[order[hi[ok] - 1]] == lb[ok]
    back[ok] = order[hi[ok] - 1]
    ok = lo < len(rs)
    ok[ok] = rb[order[lo[ok]]] == lb[ok]
    fwd[ok] = order[lo[ok]]
    return back, fwd


def pick(l_time, strategy, back, t_back, fwd, t_fwd, tolerance):
    """The answer from the two candidates (rows, -1 none) and their times: nearest takes the closer one, the backward one on a
    tie; then the tolerance (inclusive)."""
    lt = np.asarray(l_time, np.int64)
    if strategy == "backward":
        fwd = np.full_like(back, -1)
    elif strategy == "forward":
        back = np.full_like(fwd, -1)
    db, df = _dist(t_back, lt), _dist(t_fwd, lt)
    take_back = (back >= 0) & ((fwd < 0) | (db <= df))
    ans = np.where(take_back, back, fwd)
    if tolerance is not None:
        ans = np.where(np.where(take_back, db, df) <= np.uint64(tolerance), ans, -1)
    return ans


def asof_join(l_time, l_by, r_time, r_by, strategy="backward", tolerance=None):
    """Per left row the right row pandas.merge_asof(direction=strategy, tolerance=tolerance, by=...) matches, or -1.  Both
    sides time-sorted; ties: backward takes the last right row of equal time, forward the first, nearest the backward
    candidate on a distance tie."""
    if strategy not in STRATEGIES:
        raise ValueError(strategy)
    rt = np.asarray(r_time, np.int64)
    back, fwd = candidates(l_time, l_by, r_time, r_by)
    tb = rt[np.maximum(back, 0)] if len(rt) else np.zeros(len(back), np.int64)
    tf = rt[np.maximum(fwd, 0)] if len(rt) else np.zeros(len(fwd), np.int64)
    return pick(l_time, strategy, back, tb, fwd, tf, tolerance)


def merge_join(l_time, l_by, r_time, r_by, n_by, strategy, tolerance, carry_back=None, back_time=None, carry_fwd=None, fwd_time=None,
               r_base=0):
    """What qk_asof_join writes: local right rows numbered r_base + i; a key with no local candidate in a direction takes that
    direction's carry (rows and their times, per key)."""
    lt, lb = np.asarray(l_time, np.int64), np.asarray(l_by, np.int64)
    rt = np.asarray(r_time, np.int64)
    back, fwd = candidates(lt, lb, rt, r_by)
    key = np.clip(lb, 0, n_by - 1)
    inkey = (lb >= 0) & (lb < n_by)

    def side(local, carry, ctime):
        t = rt[np.maximum(local, 0)] if len(rt) else np.zeros(len(local), np.int64)
        row = np.where(local >= 0, local + r_base, -1)
        if carry is not None:
            c = np.where(inkey, np.asarray(carry, np.int64)[key], -1)
            row = np.where(local >= 0, row, c)
            t = np.where(local >= 0, t, np.asarray(ctime, np.int64)[key])
        return row, t

    rb_, tb = side(back, carry_back, back_time)
    rf_, tf = side(fwd, carry_fwd, fwd_time)
    return pick(lt, strategy, rb_, tb, rf_, tf, tolerance)


def table_pass(r_by, n_by, forward, carry=None, r_base=0):
    """carry_out of qk_asof_join / qk_asof_merge: the newest (forward: oldest) row of every key, local rows first, else carry."""
    rb = np.asarray(r_by, np.int64)
    good = (rb >= 0) & (rb < n_by)
    rows = np.nonzero(good)[0]
    out = np.full(n_by, -1, np.int64)
    if forward:
        first = np.full(n_by, len(rb), np.int64)
        np.minimum.at(first, rb[good], rows)
        out = np.where(first < len(rb), first + r_base, -1)
    else:
        last = np.full(n_by, -1, np.int64)
        np.maximum.at(last, rb[good], rows)
        out = np.where(last >= 0, last + r_base, -1)
    if carry is not None:
        out = np.where(out >= 0, out, np.asarray(carry, np.int64))
    return out

