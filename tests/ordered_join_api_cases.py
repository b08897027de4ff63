"""DataStream.join(maintain_sort_order=...) through the planner and the executors: the cases the CPU tests run on the numpy shims
(1 rank and 2 gloo ranks) and the GPU tests on the kernels (1 rank, and 2 NCCL ranks where there are two GPUs).  Every case
compares collect() in exact row order with oracle.relops.join_indices applied to the collected inputs, under both plans: the
build side replicated (or one rank) and the build side hash-partitioned across ranks (`broadcast_rows` = 0)."""
import numpy as np
import pyarrow as pa

from oracle import relops as R
from quokka_b200.datastream import OrderedStream

PLANS = ({"broadcast_rows": 1 << 40, "broadcast_cost_based": False}, {"broadcast_rows": 0, "broadcast_cost_based": False})


def _plans(qc):
    """Yields once per plan with the context configured for it; restores the configuration afterwards."""
    saved = {k: qc.exec_config.get(k) for k in PLANS[0]}
    try:
        for plan in PLANS:
            qc.exec_config.update(plan)
            yield plan
    finally:
        for k, v in saved.items():
            if v is None:
                qc.exec_config.pop(k, None)
            else:
                qc.exec_config[k] = v


def _key_codes(a: pa.Array, b: pa.Array):
    """Both key columns as int64 codes that are equal exactly when the join matches: strings by value, fp64 by bit pattern
    with -0.0 folded into +0.0, integers as they are."""
    if pa.types.is_string(a.type) or pa.types.is_large_string(a.type):
        va, vb = a.to_pylist(), b.to_pylist()
        index = {v: i for i, v in enumerate(dict.fromkeys(va + vb))}
        return np.array([index[v] for v in va], np.int64), np.array([index[v] for v in vb], np.int64)
    x, y = a.to_numpy(zero_copy_only=False), b.to_numpy(zero_copy_only=False)
    if x.dtype.kind == "f":
        return (x + 0.0).view(np.int64), (y + 0.0).view(np.int64)
    return x.astype(np.int64), y.astype(np.int64)


def expected(lt: pa.Table, rt: pa.Table, left_on, right_on, how="inner", suffix="_2", keep="left") -> pa.Table:
    """The ordered join of two collected inputs: rows in `keep`'s order, matches in the other side's order."""
    lk, rk = _key_codes(lt[left_on].combine_chunks(), rt[right_on].combine_chunks())
    if keep == "left":
        li, ri = R.join_indices(lk, rk, how)
    else:
        ri, li = R.join_indices(rk, lk, how)
    out = {c: lt[c].take(pa.array(li)) for c in lt.column_names}
    if how in ("semi", "anti"):
        return pa.table(out)
    mask = pa.array(ri < 0)
    for c in rt.column_names:
        if c == right_on:
            continue
        col = rt[c].take(pa.array(np.maximum(ri, 0))) if rt.num_rows else pa.nulls(len(ri), rt[c].type)
        out[c + suffix if c in lt.column_names else c] = pa.compute.if_else(mask, pa.nulls(len(ri), col.type), col)
    return pa.table(out)


def same_rows(got: pa.Table, exp: pa.Table, what=""):
    assert got.column_names == exp.column_names, (what, got.column_names, exp.column_names)
    assert got.num_rows == exp.num_rows, (what, got.num_rows, exp.num_rows)
    for c in exp.column_names:
        assert got[c].to_pylist() == exp[c].to_pylist(), (what, c)


def _quotes(n=2400, nsym=40, seed=0):
    rng = np.random.default_rng(seed)
    return pa.table({"time": np.arange(n, dtype=np.int64) * 3 + rng.integers(0, 3, n), "symbol": rng.integers(0, nsym, n).astype(np.int64),
                     "px": rng.standard_normal(n), "rowid": np.arange(n, dtype=np.int64)})


def _symbols(nsym=40, seed=1, dup=3):
    """Symbols 0 .. nsym-1 with every third one missing and some repeated `dup` times (several matches per left row)."""
    rng = np.random.default_rng(seed)
    keys = [s for s in range(nsym) if s % 3 != 2 for _ in range(1 + (dup - 1) * (s % 4 == 0))]
    keys = rng.permutation(np.array(keys, np.int64))
    return pa.table({"symbol": keys, "sector": pa.array([f"S{k % 7}" for k in keys]), "weight": rng.integers(0, 100, len(keys)).astype(np.int32)})


def _check(qc, left, right, left_on, right_on, how, keep="left", suffix="_2", what=""):
    res = left.join(right, left_on=left_on, right_on=right_on, how=how, suffix=suffix, maintain_sort_order=keep)
    assert isinstance(res, OrderedStream)
    lt = left.collect()
    rt = right.collect() if not isinstance(right, pa.Table) else right
    got = res.collect()
    same_rows(got, expected(lt, rt, left_on, right_on, how, suffix, keep), what)
    ex = [a.obj for a in qc.last_graph.actors.values() if type(a.obj).__name__ == "OrderedJoinExecutor"]
    assert len(ex) == 1 and ex[0].streaming == (_world() == 1 or qc.exec_config["broadcast_rows"] > 0), what
    return res


def _world():
    from quokka_b200.runtime import world_size
    return world_size()


def case_inner_and_left(qc):
    q, s = _quotes(), _symbols()
    for _ in _plans(qc):
        for how in ("inner", "left"):
            for right in (s, qc.from_arrow(s)):
                res = _check(qc, qc.from_arrow_sorted(q, "time"), right, "symbol", "symbol", how, what=how)
                assert res.sorted_by == "time"


def case_semi_and_anti(qc):
    q, s = _quotes(1500, 30, 2), _symbols(30, 3)
    for _ in _plans(qc):
        for how in ("semi", "anti"):
            _check(qc, qc.from_arrow_sorted(q, "time"), qc.from_arrow(s), "symbol", "symbol", how, what=how)


def case_keep_right_order(qc):
    """maintain_sort_order="right": rows in the right stream's order, a right row's matches in the left's; sorted_by is the
    right's sort column under its output name, or the left key when it is the right key."""
    q = _quotes(1800, 25, 4).rename_columns(["time", "sym", "px", "rowid"])
    s = _symbols(25, 5)
    for _ in _plans(qc):
        res = _check(qc, qc.from_arrow(s), qc.from_arrow_sorted(q, "time"), "symbol", "sym", "inner", keep="right")
        assert res.sorted_by == "time"
        by_key = qc.from_arrow(s).join(qc.from_arrow_sorted(q, "sym"), left_on="symbol", right_on="sym", maintain_sort_order="right")
        assert by_key.sorted_by == "symbol"


def case_many_build_rows(qc):
    """One key with thousands of build rows (more than a thread orders in place) next to keys with a few."""
    rng = np.random.default_rng(6)
    q = pa.table({"time": np.arange(300, dtype=np.int64), "k": rng.integers(0, 4, 300).astype(np.int32)})
    b = np.concatenate([np.zeros(3000, np.int32), rng.integers(1, 3, 40).astype(np.int32)])
    s = pa.table({"k": rng.permutation(b), "v": np.arange(len(b), dtype=np.int64)})
    for _ in _plans(qc):
        for how in ("inner", "left"):
            _check(qc, qc.from_arrow_sorted(q, "time"), qc.from_arrow(s), "k", "k", how, what=how)


def case_string_and_fp64_keys(qc):
    """String keys whose dictionaries differ from batch to batch (and so from rank to rank), and fp64 keys with -0.0."""
    rng = np.random.default_rng(7)
    n = 900
    names = [f"N{i:02d}" for i in range(30)]
    q = pa.table({"time": np.arange(n, dtype=np.int64), "name": pa.array([names[i] for i in rng.integers(0, 30, n)]),
                  "f": rng.integers(-3, 4, n).astype(np.float64) * 0.5})
    s = pa.table({"name": pa.array([names[i] for i in rng.integers(5, 30, 60)]), "x": np.arange(60, dtype=np.int64)})
    fs = pa.table({"f": np.array([-0.0, 0.5, -1.5, 1.0, 0.5, 7.0]), "y": np.arange(6, dtype=np.int32)})
    saved = qc.exec_config["chunk_rows"]
    qc.set_config("chunk_rows", 97)
    try:
        for _ in _plans(qc):
            for how in ("inner", "left", "anti"):
                _check(qc, qc.from_arrow_sorted(q, "time"), qc.from_arrow(s), "name", "name", how, what=("str", how))
                _check(qc, qc.from_arrow_sorted(q, "time"), qc.from_arrow(fs), "f", "f", how, what=("f64", how))
    finally:
        qc.set_config("chunk_rows", saved)


def case_empty_sides(qc):
    """A rank with no left rows (one left row in all) and a rank with no build rows (one build row in all); an anti join
    against an empty build side passes the left side through."""
    q, s = _quotes(600, 10, 8), _symbols(10, 9)
    for _ in _plans(qc):
        for how in ("inner", "left", "semi", "anti"):
            _check(qc, qc.from_arrow_sorted(q.slice(0, 1), "time"), qc.from_arrow(s), "symbol", "symbol", how, what=("1 left", how))
            _check(qc, qc.from_arrow_sorted(q, "time"), qc.from_arrow(s.slice(0, 1)), "symbol", "symbol", how, what=("1 build", how))
        empty = qc.from_arrow(s).filter_sql("weight < 0")
        got = qc.from_arrow_sorted(q, "time").join(empty, on="symbol", how="anti", maintain_sort_order="left").collect()
        same_rows(got, q, "anti against an empty build")


def case_filter_after_join(qc):
    """Filters after the join, on a left column (pushed below it) and on a right column (kept above), keep the order."""
    q, s = _quotes(2000, 30, 10), _symbols(30, 11)
    for _ in _plans(qc):
        for how in ("inner", "left"):
            left = qc.from_arrow_sorted(q, "time")
            res = left.join(qc.from_arrow(s), on="symbol", how=how, maintain_sort_order="left")
            exp = expected(q, s, "symbol", "symbol", how)
            got = res.filter_sql("px > 0").collect()
            same_rows(got, exp.filter(pa.compute.greater(exp["px"], 0)), ("left filter", how))
            got = res.filter_sql("weight > 40").collect()
            same_rows(got, exp.filter(pa.compute.greater(exp["weight"], 40)), ("right filter", how))


def _frames_equal(a: pa.Table, b: pa.Table, what=""):
    assert a.column_names == b.column_names and a.num_rows == b.num_rows, (what, a.column_names, b.column_names)
    for c in a.column_names:
        x, y = a[c].to_pylist(), b[c].to_pylist()
        if a[c].type == pa.float64():
            np.testing.assert_allclose(np.array(x, dtype=float), np.array(y, dtype=float), rtol=1e-12, atol=1e-12, err_msg=f"{what} {c}")
        else:
            assert x == y, (what, c)


def case_join_then_ordered_ops(qc):
    """join(..., maintain_sort_order="left") feeds join_asof, shift and windowed_transform with no re-sort, and gives what
    the same program gives with the unordered join followed by sort().  One match per quote and distinct times, so the
    sort has no ties to break."""
    from quokka_b200.windowtypes import OnEventTrigger, SlidingWindow
    q = _quotes(2000, 30, 12)
    s = pa.table({"symbol": np.arange(30, dtype=np.int64)[::-1].copy(), "lot": (np.arange(30, dtype=np.int64) % 5 + 1) * 100})
    rng = np.random.default_rng(13)
    t = pa.table({"time": np.sort(rng.integers(0, 6000, 700)).astype(np.int64), "symbol": rng.integers(0, 30, 700).astype(np.int64),
                  "size": rng.integers(1, 50, 700).astype(np.int64)})
    w = SlidingWindow("time", "symbol", 300, {"avg_px": "AVG(px)", "n": "count(*)"})
    programs = {
        "asof": lambda x: qc.from_arrow_sorted(t, "time").join_asof(x, on="time", by="symbol"),
        "shift": lambda x: x.shift(1, by="symbol", columns=["px", "lot"], suffix="_prev"),
        "window": lambda x: x.windowed_transform(w, OnEventTrigger()),
    }
    for _ in _plans(qc):
        for name, prog in programs.items():
            kept = qc.from_arrow_sorted(q, "time").join(qc.from_arrow(s), on="symbol", maintain_sort_order="left")
            resorted = qc.from_arrow(q).join(qc.from_arrow(s), on="symbol").sort("time")
            got, exp = prog(kept).collect(), prog(resorted).collect()
            if name == "window":            # one row per input row and key, in no fixed order across keys
                key = ["symbol", "time"]
                got, exp = got.sort_by([(k, "ascending") for k in key]), exp.sort_by([(k, "ascending") for k in key])
            _frames_equal(got, exp, name)


API_CASES = [case_inner_and_left, case_semi_and_anti, case_keep_right_order, case_many_build_rows, case_string_and_fp64_keys,
             case_empty_sides, case_filter_after_join, case_join_then_ordered_ops]
