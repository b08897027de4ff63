"""windowed_transform(TumblingWindow | SessionWindow, OnEventTrigger()) through the planner and the executors: the cases the CPU
tests run on the numpy shims (1 rank and 2 gloo ranks) and the GPU tests on the kernels (1 rank and in-process ranks).  Every
result is compared with the one-row-at-a-time reference (window_events_shim.running_window) and, for the reference's quote
fixture, with pandas; at the last row of every window it must also agree with the OnCompletionTrigger row of that window."""
import datetime

import numpy as np
import pyarrow as pa

import window_events_shim as S

RTOL = 1e-9
U = 2.0 ** -53
AGGD = {"avg_bid": "AVG(bid)", "max_spread": "MAX(ask - bid)", "n": "count(*)", "sum_ask": "SUM(ask)", "min_bid": "MIN(bid)"}


def _oaggs(bid, ask):
    return {"avg_bid": ("avg", bid), "max_spread": ("max", ask - bid), "n": ("count", None), "sum_ask": ("sum", ask), "min_bid": ("min", bid)}


def _ints(c):
    c = c.combine_chunks() if hasattr(c, "combine_chunks") else c
    if pa.types.is_timestamp(c.type):
        c = c.cast(pa.int64())
    return c.to_numpy(zero_copy_only=False).astype(np.int64)


def _keys(c):
    return np.asarray(c.to_pylist(), dtype=object)


def _codes(keys, universe):
    u = np.unique(universe)
    return np.searchsorted(u, keys)


def _run(qc, table, window, trigger, chunk=1 << 26):
    qc.set_config("chunk_rows", chunk)
    try:
        return qc.from_arrow_sorted(table, "time").windowed_transform(window, trigger).collect()
    finally:
        qc.set_config("chunk_rows", 1 << 26)


def _window(kind, length):
    from quokka_b200.windowtypes import SessionWindow, TumblingWindow
    return (TumblingWindow if kind == "tumbling" else SessionWindow)("time", "symbol", length, AGGD)


def check_events(res, time, key, bid, ask, kind, param):
    """res (collect() of a per-event window over rows time / key / bid / ask) against running_window: schema, one row per input
    row, int64 COUNT, rows of a key contiguous and in time order, every aggregate.  Returns res's (time, key codes) order."""
    names = (["time", "symbol"] if kind == "tumbling" else ["symbol", "time"]) + list(AGGD)
    assert res.column_names == names, res.column_names
    assert res.num_rows == len(time), (res.num_rows, len(time))
    assert res["n"].type == pa.int64(), res["n"].type
    t, k = _ints(res["time"]), _codes(_keys(res["symbol"]), key)
    kin = _codes(key, key)
    change = np.flatnonzero(np.diff(k) != 0)
    assert len(change) == len(np.unique(k)) - 1, "rows of one key are not contiguous"
    assert np.all((np.diff(t) >= 0) | (np.diff(k) != 0)), "rows of a key are not in time order"
    exp = S.running_window(time, kin, kind, param, _oaggs(bid, ask))
    og, oe = np.lexsort((t, k)), np.lexsort((time, kin))          # peers carry equal values: their order does not matter
    assert np.array_equal(t[og], time[oe]) and np.array_equal(k[og], kin[oe])
    for c in AGGD:
        got = res[c].to_numpy()[og]
        if c == "n":
            assert np.array_equal(got, exp[c][oe].astype(np.int64)), c
        else:
            np.testing.assert_allclose(got, exp[c][oe], rtol=RTOL, atol=1e-12, err_msg=c)
    return t, k, og


def check_pandas(res, time, key, bid, ask, kind, param):
    """The same windows in pandas: aggregate every (key, run, time) peer group, then groupby([key, run]).cumsum / cummin /
    cummax over the groups, joined back to the rows."""
    import pandas as pd
    df = pd.DataFrame({"k": key, "t": time, "bid": bid, "ask": ask, "spread": ask - bid}).sort_values(["k", "t"], kind="stable")
    if kind == "tumbling":
        df["run"] = df["t"] // param
    else:
        df["run"] = (df.groupby("k")["t"].diff() > param).astype(np.int64).groupby(df["k"]).cumsum()
    g = df.groupby(["k", "run", "t"]).agg(sb=("bid", "sum"), cnt=("bid", "size"), mx=("spread", "max"), sa=("ask", "sum"),
                                          mn=("bid", "min")).reset_index().sort_values(["k", "run", "t"])
    grp = g.groupby(["k", "run"])
    cum = pd.DataFrame({"k": g["k"], "run": g["run"], "t": g["t"], "n": grp["cnt"].cumsum(), "avg_bid": grp["sb"].cumsum() / grp["cnt"].cumsum(),
                        "max_spread": grp["mx"].cummax(), "sum_ask": grp["sa"].cumsum(), "min_bid": grp["mn"].cummin()})
    exp = df[["k", "run", "t"]].merge(cum, on=["k", "run", "t"], how="left").sort_values(["k", "t"], kind="stable")
    got = pd.DataFrame({"k": _keys(res["symbol"]), "t": _ints(res["time"]), **{c: res[c].to_numpy() for c in AGGD}})
    got = got.sort_values(["k", "t"], kind="stable")
    assert got["k"].tolist() == exp["k"].tolist() and got["t"].tolist() == exp["t"].tolist()
    assert got["n"].tolist() == exp["n"].astype(np.int64).tolist()
    for c in ("avg_bid", "max_spread", "sum_ask", "min_bid"):
        np.testing.assert_allclose(got[c].to_numpy(dtype=float), exp[c].to_numpy(dtype=float), rtol=RTOL, atol=1e-12, err_msg=c)


def check_completion(res, done, time, key, bid, ask, kind, param):
    """At the last row of every window the per-event row equals the window's OnCompletionTrigger row: COUNT / MIN / MAX bit for
    bit, SUM / AVG within twice the summation bound (w - 1) * 2^-53 * sum|v| (both are some order of the same sum)."""
    universe = np.concatenate([_keys(res["symbol"]), _keys(done["symbol"]), key])

    def runs(t, k):
        """(order by key and time, last row of each run in that order, each run's label: window start or first time)"""
        o = np.lexsort((t, k))
        t, k = t[o], k[o]
        brk = np.ones(len(t), bool)
        brk[1:] = (k[1:] != k[:-1]) | S.run_breaks(t[:-1], t[1:], kind, param)
        first = np.flatnonzero(brk)
        last = np.append(first[1:], len(t)) - 1
        return o, first, last, k[last], ((t[last] // np.int64(param)) * np.int64(param) if kind == "tumbling" else t[first])

    o, _, last, k_last, label = runs(_ints(res["time"]), _codes(_keys(res["symbol"]), universe))
    dk, dt = _codes(_keys(done["symbol"]), universe), _ints(done["time"])
    od = np.lexsort((dt, dk))
    assert np.array_equal(k_last, dk[od]) and np.array_equal(label, dt[od]), "windows differ"
    n = res["n"].to_numpy()[o][last]
    assert np.array_equal(n, done["n"].to_numpy()[od])
    oi, first_i, _, _, _ = runs(time, _codes(key, universe))
    for c, v in (("max_spread", None), ("min_bid", None), ("sum_ask", ask), ("avg_bid", bid)):
        a, b = res[c].to_numpy()[o][last], done[c].to_numpy()[od]
        if v is None:
            assert np.array_equal(a.view(np.int64), b.view(np.int64)), c
        else:
            s_abs = np.add.reduceat(np.abs(v[oi]), first_i) / (n if c == "avg_bid" else 1)
            assert np.all(np.abs(a - b) <= 2 * (n - 1) * U * s_abs * 1.0000001 + 2 * U * np.abs(a)), c


def _quotes(golden_dir):
    import os
    g = np.load(os.path.join(golden_dir, "asof_result2.npz"))
    syms = np.array([str(x) for x in g["symbols"]], dtype=object)
    time, sym, bid, ask = g["in_q_time"].astype(np.int64), g["in_q_symbol"], g["in_q_bid"], g["in_q_ask"]
    return time, syms[sym], bid.astype(np.float64), ask.astype(np.float64)


def case_events_reference_quotes(qc, golden_dir):
    """The reference's quote fixture (string symbols), tumbling 1000 and session 150, in one chunk and in chunks of 500 rows."""
    time, key, bid, ask = _quotes(golden_dir)
    table = pa.table({"time": time, "symbol": pa.array(list(key)), "bid": bid, "ask": ask})
    from quokka_b200.windowtypes import OnCompletionTrigger, OnEventTrigger
    for kind, param in (("tumbling", 1000), ("session", 150)):
        for chunk in (1 << 26, 500):
            res = _run(qc, table, _window(kind, param), OnEventTrigger(), chunk)
            check_events(res, time, key, bid, ask, kind, param)
            check_pandas(res, time, key, bid, ask, kind, param)
            check_completion(res, _run(qc, table, _window(kind, param), OnCompletionTrigger(), chunk), time, key, bid, ask, kind, param)


def case_events_timestamp_timedelta(qc):
    """A timestamp[us] time column with timedelta lengths: Window.ticks turns them into microseconds."""
    from quokka_b200.windowtypes import OnEventTrigger
    rng = np.random.default_rng(5)
    n = 3_000
    time = np.sort(rng.integers(0, 50_000_000, n)).astype(np.int64)
    time[100:140] = time[100]                                           # a tie group
    key = np.array(["AAA", "BB", "C", "DDDD"], dtype=object)[rng.integers(0, 4, n)]
    bid, ask = np.round(rng.uniform(10, 20, n), 2), np.round(rng.uniform(20, 30, n), 2)
    table = pa.table({"time": pa.array(time, type=pa.timestamp("us")), "symbol": pa.array(list(key)), "bid": bid, "ask": ask})
    for kind, td in (("tumbling", datetime.timedelta(seconds=2)), ("session", datetime.timedelta(milliseconds=40))):
        res = _run(qc, table, _window(kind, td), OnEventTrigger(), 700)
        assert pa.types.is_timestamp(res["time"].type)
        check_events(res, time, key, bid, ask, kind, int(td.total_seconds() * 10 ** 6))


def case_events_negative_times(qc):
    """Negative integer times (floor division puts -1 in [-size, 0)), integer keys, heavy ties, a key with a single row."""
    from quokka_b200.windowtypes import OnEventTrigger
    rng = np.random.default_rng(11)
    n = 2_500
    time = np.sort(rng.integers(-4_000, 1_000, n) // 7 * 7).astype(np.int64)
    key = rng.integers(0, 6, n).astype(np.int64)
    key[n // 2] = 99
    keyo = key.astype(object)
    bid, ask = rng.integers(-500, 500, n) / 8.0, rng.integers(0, 900, n) / 4.0
    table = pa.table({"time": time, "symbol": key, "bid": bid, "ask": ask})
    for kind, param in (("tumbling", 100), ("tumbling", 1), ("session", 0), ("session", 20)):
        res = _run(qc, table, _window(kind, param), OnEventTrigger(), 333)
        check_events(res, time, keyo, bid, ask, kind, param)


def case_events_after_sort(qc, golden_dir):
    """sort("time") then a per-event window gives what the same window gives on the sorted input."""
    from quokka_b200.windowtypes import OnEventTrigger
    time, key, bid, ask = _quotes(golden_dir)
    table = pa.table({"time": time, "symbol": pa.array(list(key)), "bid": bid, "ask": ask})
    shuffled = table.take(np.random.default_rng(3).permutation(table.num_rows))
    for kind, param in (("tumbling", 1000), ("session", 150)):
        res = qc.from_arrow(shuffled).sort("time").windowed_transform(_window(kind, param), OnEventTrigger()).collect()
        check_events(res, time, key, bid, ask, kind, param)


def case_events_hopping_raises(qc):
    """A hopping window (any that is not a TumblingWindow, whatever its hop) with OnEventTrigger raises, as in the reference."""
    from quokka_b200.windowtypes import HoppingWindow, OnEventTrigger
    table = pa.table({"time": np.arange(10, dtype=np.int64), "symbol": np.zeros(10, np.int64), "bid": np.ones(10), "ask": np.ones(10)})
    for hop in (1000, 3000):
        try:
            qc.from_arrow_sorted(table, "time").windowed_transform(HoppingWindow("time", "symbol", hop, 3000, AGGD), OnEventTrigger())
        except Exception as e:
            assert "OnEventTrigger" in str(e), e
        else:
            raise AssertionError("a hopping window with OnEventTrigger was accepted")


API_CASES = [case_events_reference_quotes, case_events_timestamp_timedelta, case_events_negative_times, case_events_after_sort,
             case_events_hopping_raises]
# the case list the gloo test and the in-process GPU runs share (tests/ranks.py run_cases names)
SUITE = ["window_events_cases:API_CASES"]
