"""OrderedStream.join_asof(strategy=..., tolerance=...) through the planner and the executors: the cases the CPU tests run on
the numpy shims (1 rank and 2 gloo ranks) and the GPU tests on the kernels.  Every rank passes its own contiguous slice of the
two sorted streams (cut points chosen per case, so quote times straddle the rank boundary, ranks hold no quotes or no trades,
and a symbol's only quotes sit on a later rank), and collect() is compared row for row with the numpy restatement of
pandas.merge_asof (asof_strategy_shim.asof_join) on the whole inputs."""
import datetime
import os

import numpy as np
import pyarrow as pa

import asof_strategy_shim as S

CASES_TOL = (None, 0, 3)


def _world():
    from quokka_b200.runtime import rank, world_size
    return world_size(), rank()


def _shard(table: pa.Table, cuts):
    w, me = _world()
    c = cuts(table.num_rows, w) if callable(cuts) else cuts
    return table.slice(c[me], c[me + 1] - c[me])


def even(n, w):
    return [n * r // w for r in range(w + 1)]


def _codes(a, b):
    va, vb = a.to_pylist(), b.to_pylist()
    index = {v: i for i, v in enumerate(dict.fromkeys(va + vb))}
    return np.array([index[v] for v in va], np.int64), np.array([index[v] for v in vb], np.int64)


def _time(c):
    c = c.combine_chunks() if hasattr(c, "combine_chunks") else c
    if pa.types.is_timestamp(c.type):
        c = c.cast(pa.int64())
    return c.to_numpy(zero_copy_only=False).astype(np.int64)


def check(qc, trades: pa.Table, quotes: pa.Table, strategy, tolerance, cuts_t=even, cuts_q=even, by="symbol", batch_rows=None,
          ticks=None):
    """trades need an int64 `it` column (row id), quotes an int64 `iq`; ticks = the tolerance in the time column's unit."""
    from quokka_b200.columns import DeviceTable
    t = qc.from_device(DeviceTable.from_arrow(_shard(trades, cuts_t)), sorted_by="time", batch_rows=batch_rows)
    q = qc.from_device(DeviceTable.from_arrow(_shard(quotes, cuts_q)), sorted_by="time", batch_rows=batch_rows)
    res = t.join_asof(q, on="time", by=by, strategy=strategy, tolerance=tolerance)
    got = res.collect()
    assert got.column_names == trades.column_names + [c for c in quotes.column_names if c not in ("time", by)], got.column_names
    lb, rb = _codes(trades[by].combine_chunks(), quotes[by].combine_chunks())
    exp = S.asof_join(_time(trades["time"]), lb, _time(quotes["time"]), rb, strategy, tolerance if ticks is None else ticks)
    iq = quotes["iq"].to_numpy()
    want = np.where(exp >= 0, iq[np.maximum(exp, 0)] if len(iq) else -1, -1)
    order = np.argsort(got["it"].to_numpy(), kind="stable")
    assert np.array_equal(got["it"].to_numpy()[order], trades["it"].to_numpy()), (strategy, tolerance)
    have = got["iq"].fill_null(-1).to_numpy()[order]
    bad = np.nonzero(have != want)[0]
    assert len(bad) == 0, (strategy, tolerance, by, bad[:5], have[bad[:5]], want[bad[:5]])
    return got


def _tables(nt, nq, nsym, span, seed, str_by=False):
    """Heavy time ties on both sides, duplicate (time, symbol) quotes, a symbol without quotes, trades before the first and
    after the last quote."""
    rng = np.random.default_rng(seed)
    tt = np.sort(rng.integers(-5, span + 5, nt)).astype(np.int64)
    qt = np.sort(rng.integers(0, span, nq)).astype(np.int64)
    ts, qs = rng.integers(0, nsym + 1, nt), rng.integers(0, nsym, nq)
    sym = (lambda a: pa.array([f"S{x}" for x in a])) if str_by else (lambda a: pa.array(a.astype(np.int64)))
    trades = pa.table({"time": tt, "symbol": sym(ts), "size": rng.standard_normal(nt), "it": np.arange(nt, dtype=np.int64)})
    quotes = pa.table({"time": qt, "symbol": sym(qs), "px": rng.standard_normal(nq), "iq": np.arange(nq, dtype=np.int64)})
    return trades, quotes


def case_strategies(qc):
    trades, quotes = _tables(700, 900, 6, 120, 0)
    for strategy in S.STRATEGIES:
        for tol in CASES_TOL:
            check(qc, trades, quotes, strategy, tol)
            check(qc, trades, quotes, strategy, tol, cuts_t=lambda n, w: [0] + [n // 3] * (w - 1) + [n])   # trades far from their quotes


def case_rank_boundaries(qc):
    """Quotes of one symbol at time 10 on both sides of the boundary and trades at exactly 10; a gap between the ranks' times;
    symbol 7 quoted only on the last rank; a rank without quotes, a rank without trades."""
    q_time = np.array([1, 4, 10, 10, 10, 10, 10, 30, 31, 40, 40, 50], np.int64)
    q_sym = np.array([1, 2, 1, 2, 1, 2, 1, 7, 1, 2, 7, 1], np.int64)
    t_time = np.array([0, 3, 10, 10, 10, 12, 20, 25, 30, 40, 45, 60], np.int64)
    t_sym = np.array([1, 1, 1, 2, 7, 2, 1, 7, 7, 2, 1, 1], np.int64)
    quotes = pa.table({"time": q_time, "symbol": q_sym, "iq": np.arange(len(q_time), dtype=np.int64)})
    trades = pa.table({"time": t_time, "symbol": t_sym, "it": np.arange(len(t_time), dtype=np.int64)})
    straddle = lambda n, w: [0] + [5] * (w - 1) + [n]                     # rank 0 ends with two of the five quotes at 10
    gap = lambda n, w: [0] + [7] * (w - 1) + [n]                          # rank 0 ends at 10, rank 1 starts at 30
    only_last = lambda n, w: [0] * w + [n]                                # ranks before the last have no quotes
    no_trades_first = lambda n, w: [0] * w + [n]
    for strategy in S.STRATEGIES:
        for tol in (None, 0, 5):
            for cq in (straddle, gap, only_last, even):
                for ct in (even, no_trades_first, lambda n, w: [0] + [n] * w):
                    check(qc, trades, quotes, strategy, tol, cuts_t=ct, cuts_q=cq)


def case_hash_plan(qc):
    trades, quotes = _tables(400, 500, 5, 80, 1)
    qc.set_config("asof_time_ranges", False)
    try:
        for strategy in S.STRATEGIES:
            for tol in (None, 2):
                check(qc, trades, quotes, strategy, tol)
    finally:
        qc.set_config("asof_time_ranges", True)


def case_many_symbols(qc):
    """More symbols than the merge kernel's shared-memory table holds: the partition + search path."""
    n = 50_000
    rng = np.random.default_rng(3)
    qs = rng.permutation(np.arange(n + 2000) % n)
    quotes = pa.table({"time": np.sort(rng.integers(0, 5000, len(qs))).astype(np.int64), "symbol": qs.astype(np.int64),
                       "iq": np.arange(len(qs), dtype=np.int64)})
    trades = pa.table({"time": np.sort(rng.integers(0, 5000, 20_000)).astype(np.int64), "symbol": rng.integers(0, n + 10, 20_000).astype(np.int64),
                       "it": np.arange(20_000, dtype=np.int64)})
    for strategy in S.STRATEGIES:
        for tol in (None, 4):
            check(qc, trades, quotes, strategy, tol)


def case_string_by(qc):
    trades, quotes = _tables(300, 400, 7, 60, 4, str_by=True)
    for strategy in S.STRATEGIES:
        for tol in (None, 1):
            check(qc, trades, quotes, strategy, tol)


def case_timestamp_timedelta(qc):
    trades, quotes = _tables(300, 400, 4, 60, 5)
    us = lambda t: t.set_column(0, "time", pa.array(t["time"].to_numpy() * 1_000_000, pa.timestamp("us")))
    for strategy in S.STRATEGIES:
        check(qc, us(trades), us(quotes), strategy, datetime.timedelta(seconds=2), ticks=2_000_000)
        check(qc, us(trades), us(quotes), strategy, 1_500_000)


def case_small_batches(qc):
    """Many small batches: backward with a tolerance streams with its carried table, forward and nearest hold."""
    trades, quotes = _tables(600, 800, 5, 150, 6)
    for strategy in S.STRATEGIES:
        for tol in (None, 2):
            check(qc, trades, quotes, strategy, tol, batch_rows=7)


def case_golden_reference(qc, golden_dir):
    """apps/time-series/test_trade2.csv x test_quote2.csv, forward and nearest as pandas.merge_asof computed them
    (tests/golden/make_golden_asof_strategy.py)."""
    g = np.load(os.path.join(golden_dir, "asof_strategy2.npz"))
    trades = pa.table({"time": g["t_time"], "symbol": g["t_sym"].astype(np.int64), "it": np.arange(len(g["t_time"]), dtype=np.int64)})
    quotes = pa.table({"time": g["q_time"], "symbol": g["q_sym"].astype(np.int64), "iq": np.arange(len(g["q_time"]), dtype=np.int64)})
    tol = int(g["tolerance"])
    for strategy in ("forward", "nearest"):
        for t, tag in ((None, ""), (tol, "_tol")):
            exp = S.asof_join(g["t_time"], g["t_sym"], g["q_time"], g["q_sym"], strategy, t)
            assert np.array_equal(exp, g[f"ridx_{strategy}{tag}"]), (strategy, t)       # the restatement against pandas
            got = check(qc, trades, quotes, strategy, t, batch_rows=500)
            order = np.argsort(got["it"].to_numpy(), kind="stable")
            assert np.array_equal(got["iq"].fill_null(-1).to_numpy()[order], g[f"ridx_{strategy}{tag}"])


def case_invalid_args(qc):
    trades, quotes = _tables(10, 10, 2, 10, 7)
    t, q = qc.from_arrow_sorted(trades, "time"), qc.from_arrow_sorted(quotes, "time")
    for kw in ({"strategy": "closest"}, {"strategy": None}, {"tolerance": -1}, {"tolerance": 1.5}, {"tolerance": True},
               {"tolerance": "1s"}, {"tolerance": datetime.timedelta(seconds=-1)}):
        try:
            t.join_asof(q, on="time", by="symbol", **kw)
        except ValueError:
            continue
        raise AssertionError(f"join_asof accepted {kw}")
    try:                                     # a timedelta needs a timestamp time column
        t.join_asof(q, on="time", by="symbol", tolerance=datetime.timedelta(seconds=1)).collect()
    except ValueError:
        return
    raise AssertionError("a timedelta tolerance on an integer time column was accepted")


API_CASES = [case_strategies, case_rank_boundaries, case_hash_plan, case_many_symbols, case_string_by, case_timestamp_timedelta,
             case_small_batches, case_golden_reference, case_invalid_args]
