"""DataStream.sort through the planner and the executors: the cases the CPU tests run on the numpy shims (1 rank and 2 gloo
ranks) and the GPU tests on the kernels (1 rank, and 2 NCCL ranks where there are two GPUs).  Every rank collects the whole
result, so every case checks the same thing on every rank.  Expected orders come from tests/sort_cases.py."""
import os

import numpy as np
import pyarrow as pa

import sort_cases as SC


def _world():
    from quokka_b200.columns import world_size
    return world_size()


def _np(t: pa.Table, c: str):
    col = t[c]
    if pa.types.is_string(col.type) or pa.types.is_large_string(col.type):
        return np.array(col.to_pylist(), dtype=object)
    return col.to_numpy(zero_copy_only=False) if col.null_count == 0 else np.array(col.to_pylist(), dtype=object)


def _mixed_table(n=5003, seed=3):
    rng = np.random.default_rng(seed)
    words = ["pear", "apple", "zebra", "Mango", "fig", "", "apple pie"]
    b = (rng.integers(0, 6, n) - 2).astype(np.float64)
    b[rng.random(n) < 0.05] = np.nan
    b[rng.random(n) < 0.05] = -0.0
    code = rng.integers(0, len(words), n)
    return {"a": rng.integers(-3, 3, n).astype(np.int64), "b": b, "code": code, "s": np.array(words, dtype=object)[code],
            "d": rng.integers(8000, 8100, n).astype(np.int32), "rowid": np.arange(n, dtype=np.int64)}, words


def _arrow(cols):
    return pa.table({c: (pa.array(list(v)) if v.dtype == object else v) for c, v in cols.items() if c != "code"})


def case_sort_collect(qc, chunk=700):
    """collect() of a sorted stream is in order, row for row: one and several columns, both directions, a string column by value,
    whatever the batching.  On one rank rows that tie keep their input order; across ranks they keep (source rank, arrival), so
    there the row id is made the last sort column."""
    cols, words = _mixed_table()
    tie = [] if _world() == 1 else ["rowid"]
    for by, desc in ((["a"], [False]), (["b"], [True]), (["s", "a"], [False, True]), (["d", "b", "s", "a"], [True, False, True, False])):
        for rows in (1 << 26, chunk):
            qc.set_config("chunk_rows", rows)
            try:
                res = qc.from_arrow(_arrow(cols)).sort(by + tie, desc + [False] * len(tie)).collect()
            finally:
                qc.set_config("chunk_rows", 1 << 26)
            assert res.column_names == [c for c in cols if c != "code"]
            keys = [cols["code"] if c == "s" else cols[c] for c in by + tie]
            perm = SC.reference_perm(keys, [None] * len(keys), desc + [False] * len(tie), [words if c == "s" else None for c in by + tie])
            assert np.array_equal(_np(res, "rowid"), cols["rowid"][perm]), (by, desc, rows)
            assert list(_np(res, "s")) == list(cols["s"][perm])


def case_sort_select_filter_keep_order(qc):
    """Row-wise operators above a sort keep its order, and the sort below a projection still gets its key columns."""
    cols, _ = _mixed_table(3001, 5)
    s = qc.from_arrow(_arrow(cols)).sort(["d", "rowid"], [True, False])
    res = s.filter_sql("a >= 0").select(["rowid"]).rename({"rowid": "r"}).collect()
    perm = SC.reference_perm([cols["d"], cols["rowid"]], [None, None], [True, False])
    assert np.array_equal(_np(res, "r"), cols["rowid"][perm][cols["a"][perm] >= 0])


def case_sort_nulls_from_left_join(qc):
    """NULLs made by a left join sort last in both directions and tie with each other."""
    n = 2000
    rng = np.random.default_rng(11)
    left = pa.table({"k": rng.integers(0, 50, n).astype(np.int64), "rowid": np.arange(n, dtype=np.int64)})
    right = pa.table({"k": np.arange(0, 50, 2, dtype=np.int64), "v": (np.arange(25) % 7).astype(np.float64)})
    k = left["k"].to_numpy()
    valid = (k % 2 == 0).astype(np.uint8)
    v = np.where(valid == 1, (k // 2) % 7, 0).astype(np.float64)
    for desc in (False, True):
        res = qc.from_arrow(left).join(qc.from_arrow(right), on="k", how="left").sort(["v", "rowid"], [desc, False]).collect()
        perm = SC.reference_perm([v, np.arange(n, dtype=np.int64)], [valid, None], [desc, False])
        assert np.array_equal(_np(res, "rowid"), perm.astype(np.int64)), desc
        assert res["v"].null_count == int((valid == 0).sum())
        assert res["v"].slice(res.num_rows - res["v"].null_count).null_count == res["v"].null_count       # all of them at the end


def _asof_tables(golden_dir, tag):
    g = np.load(os.path.join(golden_dir, f"asof{tag}.npz"))
    syms = np.array([f"S{i:04d}" for i in range(int(max(g["t_sym"].max(), g["q_sym"].max())) + 1)], dtype=object)
    trades = pa.table({"time": g["t_time"], "symbol": pa.array(list(syms[g["t_sym"]])), "size": g["t_size"]})
    quotes = pa.table({"time": g["q_time"], "symbol": pa.array(list(syms[g["q_sym"]])), "asize": g["q_asize"],
                       "iq": np.arange(len(g["q_time"]), dtype=np.int64)})
    return g, syms, trades, quotes


def _shuffled(t: pa.Table, seed: int) -> pa.Table:
    return t.take(pa.array(np.random.default_rng(seed).permutation(t.num_rows)))


def case_sort_then_asof(qc, golden_dir, tag="1"):
    """A shuffled, filtered, unsorted stream sorted by the engine joins as-of exactly like the pre-sorted input (the committed
    fixture's expected right rows).  Quotes of one time keep their file order through the second sort column."""
    g, syms, trades, quotes = _asof_tables(golden_dir, tag)
    t = qc.from_arrow(_shuffled(trades, 1)).filter_sql("size > -1000000").sort("time")
    q = qc.from_arrow(_shuffled(quotes, 2)).sort(["time", "iq"])
    assert t.sorted_by == "time"
    res = t.join_asof(q, on="time", by="symbol").collect()
    assert res.num_rows == len(g["t_time"])
    order = np.lexsort((_np(res, "size"), _np(res, "symbol"), _np(res, "time")))
    eorder = np.lexsort((g["t_size"], syms[g["t_sym"]], g["t_time"]))
    assert np.array_equal(res["iq"].fill_null(-1).to_numpy()[order], g["ridx"][eorder])
    if _world() > 1:
        asof = [x.obj for x in qc.last_graph.actors.values() if type(x.obj).__name__ == "SortedAsofExecutor"]
        assert asof and asof[0].time_ranges                                        # joined in place over the ranks' time ranges


def _frames_equal(a: pa.Table, b: pa.Table):
    assert a.column_names == b.column_names and a.num_rows == b.num_rows, (a.column_names, b.column_names, a.num_rows, b.num_rows)
    da, db = a.to_pandas(), b.to_pandas()
    cols = list(da.columns)
    da, db = da.sort_values(cols).reset_index(drop=True), db.sort_values(cols).reset_index(drop=True)
    for c in cols:
        x, y = da[c].to_numpy(), db[c].to_numpy()
        if x.dtype.kind == "f":
            np.testing.assert_allclose(x, y, rtol=1e-12, atol=1e-12, err_msg=c)
        else:
            assert list(x) == list(y), c


def case_sort_then_window(qc, golden_dir):
    from quokka_b200.windowtypes import OnEventTrigger, SlidingWindow
    _, _, _, quotes = _asof_tables(golden_dir, "1")
    quotes = quotes.set_column(2, "asize", quotes["asize"].cast(pa.float64()))
    w = SlidingWindow("time", "symbol", 2000, {"avg_a": "AVG(asize)", "n": "count(*)", "mx": "MAX(asize)"})
    exp = qc.from_arrow_sorted(quotes, "time").windowed_transform(w, OnEventTrigger()).collect()
    got = qc.from_arrow(_shuffled(quotes, 3)).sort("time").windowed_transform(w, OnEventTrigger()).collect()
    _frames_equal(got, exp)


def case_sort_then_pattern(qc, golden_dir):
    _, _, _, quotes = _asof_tables(golden_dir, "1")
    quotes = quotes.set_column(2, "asize", quotes["asize"].cast(pa.float64()))
    events = [("a", "asize > 3"), ("b", "b.asize < a.asize"), ("c", "c.asize > b.asize")]
    exp = qc.from_arrow_sorted(quotes, "time").pattern_recognize("time", events, 5000, "symbol").collect()
    got = qc.from_arrow(_shuffled(quotes, 4)).sort("time").pattern_recognize("time", events, 5000, "symbol").collect()
    assert exp.num_rows > 0
    _frames_equal(got, exp)


def case_sort_then_quantile_and_gram(qc):
    """A sorted stream feeding the quantile sketch and the Gram state gives the answers of the same programs without the sort:
    the sketch bit for bit, the Gram matrix within the summation bound of tests/gram_cases.py."""
    import gram_cases as GC
    rng = np.random.default_rng(29)
    n = 9_001
    cols = {"a": rng.normal(3e4, 5.0, n), "b": rng.integers(-1000, 1000, n),
            "c": rng.normal(-2.0, 1e-3, n).astype(np.float32)}
    names = list(cols)
    d = qc.from_arrow(pa.table(cols))
    qs = [0.0, 0.1, 0.5, 0.9, 1.0]
    assert d.sort("b").approximate_quantile(names, qs).collect().equals(d.approximate_quantile(names, qs).collect())
    g, bound = GC.gram_ref(np.stack([cols[c].astype(np.float64) for c in names], axis=1))
    for s in (d, d.sort("b", descending=True)):
        GC.assert_within(GC.table_matrix(s.gramian(names).collect(), names), g, bound, "gramian")


def case_sort_ranges(qc):
    """What the ranks hold after the sort: each is sorted, rank r's first-column values all precede rank r + 1's, no value is on
    two ranks -- also when a rank has no rows and when every row has the same value (one rank gets everything)."""
    from quokka_b200.columns import rank
    from quokka_b200.executors import SortExecutor
    n = 4001
    rng = np.random.default_rng(21)
    for name, k in (("random", rng.integers(0, 40, n).astype(np.int64)), ("all-equal", np.full(n, 7, np.int64)), ("tiny", np.array([5], np.int64))):
        tab = pa.table({"k": k, "rowid": np.arange(len(k), dtype=np.int64)})
        res = qc.from_arrow(tab).sort(["k", "rowid"]).collect()
        assert np.array_equal(_np(res, "rowid"), SC.reference_perm([k, np.arange(len(k))], [None, None], [False, False])), name
        ex = [a.instance for a in qc.last_graph.actors.values() if isinstance(a.instance, SortExecutor)][0]
        mine = ex.state["k"].data.cpu().numpy() if ex.state is not None else np.zeros(0, np.int64)
        assert np.all(mine[1:] >= mine[:-1])
        if _world() > 1:
            words = [len(mine), int(mine[0]) if len(mine) else 0, int(mine[-1]) if len(mine) else 0]
            rows = qc.last_graph.exchange.allgather_words(words)
            held = [r for r in rows if r[0]]
            assert sum(r[0] for r in rows) == len(k)
            assert all(a[2] < b[1] for a, b in zip(held, held[1:])), (name, rows)
            if name == "all-equal":
                assert len(held) == 1


def case_sort_errors(qc):
    import pytest
    cols, _ = _mixed_table(50, 1)
    s = qc.from_arrow(_arrow(cols))
    with pytest.raises(AssertionError):
        s.sort("nope")
    with pytest.raises(AssertionError):
        s.sort(["a", "b"], [True])
    with pytest.raises(AssertionError):
        s.sort("a", "yes")
    with pytest.raises(AssertionError):
        s.sort([])
    vec = pa.table({"x": np.arange(4, dtype=np.int64),
                    "v": pa.FixedSizeListArray.from_arrays(pa.array(np.arange(8, dtype=np.float32)), 2)})
    with pytest.raises(NotImplementedError, match="vector column"):
        qc.from_arrow(vec).sort("v")
    res = qc.from_arrow(vec).sort("x", True).collect()                         # a vector payload moves with its row
    assert res["x"].to_pylist() == [3, 2, 1, 0] and res["v"].to_pylist()[0] == [6.0, 7.0]
    d = s.sort("a", True)
    assert d.sorted_by is None
    from quokka_b200.windowtypes import OnEventTrigger, SlidingWindow
    with pytest.raises(AssertionError, match="sorted"):
        d.windowed_transform(SlidingWindow("a", "d", 5, {"n": "count(*)"}), OnEventTrigger())
