"""OrderedStream.shift through the planner and the executors: the cases the CPU tests run on the numpy shims (1 rank and 2 gloo
ranks) and the GPU tests on the kernels (1 rank, and 2 NCCL ranks where there are two GPUs).  Every rank collects the whole
result.  Expected values come from tests/shift_cases.py, computed over the rows in the order collect() returns them -- the
stream order -- which is also checked against the input's order."""
import datetime

import numpy as np
import pyarrow as pa
import pytest

import shift_cases as SC


def _np(t: pa.Table, c: str):
    return t[c].to_numpy(zero_copy_only=False) if t[c].null_count == 0 else np.array(t[c].to_pylist(), dtype=object)


def _values(t: pa.Table, c: str):
    """(values with NULLs as 0, validity uint8) of a numeric column."""
    col = t[c]
    valid = np.array([v is not None for v in col.to_pylist()], np.uint8) if col.null_count else None
    return col.fill_null(0).to_numpy(zero_copy_only=False), valid


def _check(res: pa.Table, keys, n, cols, suffix, fill=None, src_table=None):
    """Columns c + suffix of `res` against the reference shift of `src_table`'s (default: res's) columns c, row for row."""
    src_table = res if src_table is None else src_table
    exp = SC.reference_shift(keys, n, {c: _values(src_table, c) for c in cols}, fill)
    for c in cols:
        got, gvalid = _values(res, c + suffix)
        ev, evalid = exp[c]
        gvalid = np.ones(len(got), np.uint8) if gvalid is None else gvalid
        assert np.array_equal(gvalid, evalid), (c, n)
        assert np.array_equal(got[evalid == 1], ev[evalid == 1]), (c, n)


def _codes(t: pa.Table, c: str):
    return np.unique(np.array(t[c].to_pylist(), dtype=object), return_inverse=True)[1].astype(np.int64)


def _quotes(n=3001, nsym=37, seed=0):
    rng = np.random.default_rng(seed)
    time = np.sort(rng.integers(0, n // 2, n)).astype(np.int64)
    sym = rng.integers(0, nsym, n)
    return pa.table({"time": time, "sym": pa.array([f"S{s:03d}" for s in sym]), "px": rng.standard_normal(n),
                     "sz": rng.integers(-100, 100, n).astype(np.int64), "q": rng.integers(0, 9, n).astype(np.int32),
                     "rowid": np.arange(n, dtype=np.int64)})


def _straddling():
    """Eleven rows in time order.  Key "a" has one row in each half (the halves are the ranks' shards on two ranks), so a shift
    by 3 reaches across both ranks for it; "b" sits across the boundary; "c" only in the second half."""
    return pa.table({"time": np.arange(11, dtype=np.int64),
                     "sym": pa.array(["b", "a", "b", "b", "b", "b", "a", "c", "b", "c", "a"]),
                     "px": np.arange(11, dtype=np.float64) * 1.5, "sz": np.arange(11, dtype=np.int64) - 5,
                     "q": np.arange(11, dtype=np.int32), "rowid": np.arange(11, dtype=np.int64)})


def case_shift_lag_lead(qc):
    """Lag and lead by key and over the whole stream, n in {0, +-1, +-3, +-rows, +-2^40}, whatever the batching; the stream
    order is the input's."""
    for tab in (_quotes(), _straddling()):
        for rows in (1 << 26, 700, 4):
            if rows == 4 and tab.num_rows > 100:
                continue
            qc.set_config("chunk_rows", rows)
            try:
                for by in ("sym", None):
                    for n in SC.n_cases(tab.num_rows):
                        res = qc.from_arrow_sorted(tab, "time").shift(n, by=by, columns=["px", "sz", "q"], suffix="_s").collect()
                        assert np.array_equal(_np(res, "rowid"), np.arange(tab.num_rows)), (by, n, rows)
                        _check(res, _codes(res, "sym") if by else None, n, ["px", "sz", "q"], "_s")
            finally:
                qc.set_config("chunk_rows", 1 << 26)


def case_shift_in_place(qc):
    """The reference's form: every column but `by` shifted in place, the schema unchanged, sorted_by cleared because the time
    column moved; a dict fill fills the columns it names and leaves NULLs in the others."""
    tab = _quotes(2000, 11, 3)
    s = qc.from_arrow_sorted(tab, "time").shift(2, "sym", {"px": 0.25, "sz": -1})
    assert s.sorted_by is None and s.schema == tab.column_names
    res = s.collect()
    assert res.column_names == tab.column_names
    keys = _codes(tab, "sym")
    _check(res, keys, 2, ["px", "sz"], "", {"px": 0.25, "sz": -1}, src_table=tab)
    _check(res, keys, 2, ["time", "q", "rowid"], "", None, src_table=tab)
    kept = qc.from_arrow_sorted(tab, "time").shift(1, "sym", columns=["px"])
    assert kept.sorted_by == "time"


def case_shift_fills(qc):
    """Fills converted to the column's type: a string joins the dictionary, dates, timestamps and booleans."""
    tab = pa.table({"time": np.arange(6, dtype=np.int64), "k": np.array([0, 1, 0, 1, 0, 2], np.int64),
                    "name": pa.array(["x", "y", "z", "x", "y", "z"]),
                    "d": pa.array([datetime.date(2020, 1, i + 1) for i in range(6)], pa.date32()),
                    "ts": pa.array([datetime.datetime(2021, 5, 1, 0, 0, i) for i in range(6)], pa.timestamp("us")),
                    "flag": pa.array([True, False, True, True, False, False])})
    fill = {"name": "none", "d": datetime.date(1999, 12, 31), "ts": datetime.datetime(2000, 1, 1, 12), "flag": True}
    res = qc.from_arrow_sorted(tab, "time").shift(1, by="k", fill_value=fill, columns=["name", "d", "ts", "flag"], suffix="_p").collect()
    assert res["name_p"].to_pylist() == ["none", "none", "x", "y", "z", "none"]
    assert res["d_p"].to_pylist() == [datetime.date(1999, 12, 31)] * 2 + [datetime.date(2020, 1, 1), datetime.date(2020, 1, 2),
                                                                          datetime.date(2020, 1, 3), datetime.date(1999, 12, 31)]
    assert res["ts_p"].to_pylist()[:3] == [datetime.datetime(2000, 1, 1, 12)] * 2 + [datetime.datetime(2021, 5, 1)]
    assert res["flag_p"].to_pylist() == [True, True, True, False, True, True]
    assert res["name"].to_pylist() == tab["name"].to_pylist()
    lead = qc.from_arrow_sorted(tab, "time").shift(-1, by="k", fill_value=7, columns=["ts"], suffix="_n").collect()
    assert [v.second if v.year == 2021 else None for v in lead["ts_n"].to_pylist()] == [2, 3, 4, None, None, None]


def case_shift_nulls_from_left_join(qc):
    """NULLs made by a left join upstream stay NULL when they move; rows without a source are NULL too."""
    n = 1500
    rng = np.random.default_rng(11)
    left = pa.table({"k": rng.integers(0, 40, n).astype(np.int64), "rowid": np.arange(n, dtype=np.int64)})
    right = pa.table({"k": np.arange(0, 40, 2, dtype=np.int64), "v": np.arange(20, dtype=np.float64) + 0.5})
    s = qc.from_arrow(left).join(qc.from_arrow(right), on="k", how="left").sort("rowid")
    res = s.shift(1, by=None, columns=["v"], suffix="_p").collect()
    assert np.array_equal(_np(res, "rowid"), np.arange(n))
    k = left["k"].to_numpy()
    v = [float(x // 2) + 0.5 if x % 2 == 0 else None for x in k]
    assert res["v"].to_pylist() == v
    assert res["v_p"].to_pylist() == [None] + v[:-1]


def case_sort_then_shift(qc):
    """A shuffled stream sorted by the engine, shifted per key and differenced: the reference's use of a lag."""
    tab = _quotes(4001, 29, 5)
    shuffled = tab.take(pa.array(np.random.default_rng(1).permutation(tab.num_rows)))
    s = qc.from_arrow(shuffled).sort(["time", "rowid"]).shift(1, by="sym", columns=["px"], suffix="_prev")
    assert s.sorted_by == "time"
    res = s.with_columns_sql("px - px_prev as d").collect()
    assert np.array_equal(_np(res, "rowid"), np.arange(tab.num_rows))
    _check(res, _codes(res, "sym"), 1, ["px"], "_prev")
    d = res["d"].to_pylist()
    prev = res["px_prev"].to_pylist()
    px = res["px"].to_pylist()
    assert all((a is None) == (p is None) and (a is None or a == x - p) for a, p, x in zip(d, prev, px))


def case_shift_then_asof(qc, golden_dir):
    """A shifted stream stays ordered and joins as-of: every matched quote carries its key's previous asize."""
    import os
    g = np.load(os.path.join(golden_dir, "asof1.npz"))
    syms = np.array([f"S{i:04d}" for i in range(int(max(g["t_sym"].max(), g["q_sym"].max())) + 1)], dtype=object)
    trades = pa.table({"time": g["t_time"], "symbol": pa.array(list(syms[g["t_sym"]])), "size": g["t_size"]})
    quotes = pa.table({"time": g["q_time"], "symbol": pa.array(list(syms[g["q_sym"]])), "asize": g["q_asize"],
                       "iq": np.arange(len(g["q_time"]), dtype=np.int64)})
    q = qc.from_arrow_sorted(quotes, "time").shift(1, by="symbol", fill_value=-1, columns=["asize"], suffix="_prev")
    res = qc.from_arrow_sorted(trades, "time").join_asof(q, on="time", by="symbol").collect()
    assert res.num_rows == len(g["t_time"])
    prev = SC.reference_shift(g["q_sym"].astype(np.int64), 1, {"a": (g["q_asize"], None)}, fill=-1)["a"][0]
    iq, ap = res["iq"].to_pylist(), res["asize_prev"].to_pylist()
    assert any(i is not None for i in iq)
    for i, a in zip(iq, ap):
        assert (a is None) if i is None else a == prev[i]


def case_shift_out_of_order(qc):
    """Rows of a key out of order in the sort column raise, also when each rank's piece is sorted and only the ranks' ranges
    are out of order (the second half holds the earlier times)."""
    n = 400
    t1 = np.arange(n, dtype=np.int64)
    t2 = np.concatenate([t1[n // 2:], t1[:n // 2]])
    for time in (t1[::-1].copy(), t2):
        tab = pa.table({"time": time, "k": np.arange(n, dtype=np.int64) % 3, "v": np.arange(n, dtype=np.float64)})
        with pytest.raises(Exception, match="not sorted by time"):
            qc.from_arrow_sorted(tab, "time").shift(1, by="k", columns=["v"]).collect()
    ok = pa.table({"time": t2, "k": np.arange(n, dtype=np.int64) % 3, "v": np.arange(n, dtype=np.float64)})
    qc.from_arrow_sorted(ok, "v").shift(1, by="k", columns=["time"], suffix="_p").collect()        # only the sort column is checked


def case_shift_errors(qc):
    from quokka_b200 import _lib as L
    tab = _quotes(50, 3, 1)
    s = qc.from_arrow_sorted(tab, "time")
    with pytest.raises(L.QkError, match="'sz'"):
        s.shift(1, "sym", fill_value=1.5, columns=["sz"]).collect()
    with pytest.raises(L.QkError, match="'q'"):
        s.shift(1, "sym", fill_value=1 << 40, columns=["q"]).collect()
    with pytest.raises(L.QkError, match="'sym'"):
        s.shift(1, None, fill_value=3, columns=["sym"]).collect()
    with pytest.raises(AssertionError):
        s.shift(1, "sym", columns=["sym", "px"])
    with pytest.raises(AssertionError):
        s.shift(1.0, "sym")
    with pytest.raises(AssertionError):
        s.shift(1, "nope")
    with pytest.raises(L.QkError, match="duplicated"):
        s.shift(1, "sym", columns=["px"], suffix="_x").shift(1, "sym", columns=["px"], suffix="_x")
    with pytest.raises(L.QkError, match="duplicated"):
        s.rename({"q": "px_p"}).shift(1, "sym", columns=["px"], suffix="_p")
    vec = pa.table({"time": np.arange(4, dtype=np.int64), "k": np.zeros(4, np.int64),
                    "v": pa.FixedSizeListArray.from_arrays(pa.array(np.arange(8, dtype=np.float32)), 2)})
    with pytest.raises(NotImplementedError, match="vector column"):
        qc.from_arrow_sorted(vec, "time").shift(1, "k")
    with pytest.raises(NotImplementedError, match="vector column"):
        qc.from_arrow_sorted(vec, "time").shift(1, "k", columns=["v"])
    res = qc.from_arrow_sorted(vec, "time").shift(1, "k", columns=["time"], suffix="_p").collect()      # a vector payload stays put
    assert res["v"].to_pylist()[3] == [6.0, 7.0] and res["time_p"].to_pylist() == [None, 0, 1, 2]
