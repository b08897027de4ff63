"""Exact references for the nearest-neighbour kernels (qk_knn_topk / qk_knn_merge) and DataStream.vector_nn_join: numpy fp64.

The score of row x for the unit probe p (fp32, normalised in fp64 by the host) is s = (x . p) / ||x||, computed exactly enough in
fp64 to serve as s_fp64 of the error contract |s - s_fp64| <= (d + 8) 2^-21."""
from __future__ import annotations

import numpy as np
import pyarrow as pa


def bound(d: int) -> float:
    return (d + 8) * 2.0 ** -21


def normalise(P) -> np.ndarray:
    P = np.asarray(P, dtype=np.float64)
    return (P / np.linalg.norm(P, axis=1, keepdims=True)).astype(np.float32)


def exact_scores(X, phat) -> np.ndarray:
    """[n, q] fp64 scores; NaN where the row never matches (zero norm or a non-finite element)."""
    X = np.asarray(X, dtype=np.float64)
    with np.errstate(all="ignore"):
        norm = np.sqrt((X * X).sum(axis=1))
        s = (X @ np.asarray(phat, dtype=np.float64).T) / norm[:, None]
    bad = ~(np.isfinite(X).all(axis=1) & (norm > 0))
    s[bad] = np.nan
    return s


def exact_topk(X, phat, k):
    """(rows [q, k] int64 with -1 padding, scores [q, k] fp64) by fp64 score desc, ties by smaller row."""
    s = exact_scores(X, phat)
    n, q = s.shape
    rows = np.full((q, k), -1, np.int64)
    sc = np.full((q, k), -np.inf)
    for p in range(q):
        ok = np.nonzero(~np.isnan(s[:, p]))[0]
        order = ok[np.lexsort((ok, -s[ok, p]))][:k]
        rows[p, :len(order)] = order
        sc[p, :len(order)] = s[order, p]
    return rows, sc


def check_topk(X, phat, k, scores, rows):
    """Asserts the kernel's (scores, rows) meet the contract: every returned score within the bound of its exact score, the right
    number of rows per probe, best-first order, and the returned set equal to the exact top-k outside the tie band (entries whose
    exact score lies within 2 * bound of the k-th)."""
    scores, rows = np.asarray(scores, dtype=np.float64), np.asarray(rows)
    d = np.asarray(X).shape[1]
    b = bound(d)
    s = exact_scores(X, phat)
    er, es = exact_topk(X, phat, k)
    for p in range(len(phat)):
        nvalid = int((er[p] >= 0).sum())
        got = rows[p][rows[p] >= 0]
        assert len(got) == nvalid, f"probe {p}: {len(got)} rows, {nvalid} expected"
        assert (rows[p][nvalid:] == -1).all() and np.isneginf(scores[p][nvalid:]).all()
        if nvalid == 0:
            continue
        assert len(set(got.tolist())) == len(got), f"probe {p}: duplicate rows"
        gs = scores[p][:nvalid]
        assert np.all(np.abs(gs - s[got, p]) <= b), f"probe {p}: score error {np.max(np.abs(gs - s[got, p]))} > {b}"
        assert np.all((gs[:-1] > gs[1:]) | ((gs[:-1] == gs[1:]) & (got[:-1] < got[1:]))), f"probe {p}: not best-first"
        kth = es[p][nvalid - 1]
        sure = set(er[p][:nvalid][es[p][:nvalid] > kth + 2 * b].tolist())
        assert sure <= set(got.tolist()), f"probe {p}: missing rows {sorted(sure - set(got.tolist()))}"
        col = s[:, p]
        allowed = set(np.nonzero(col >= kth - 2 * b)[0].tolist())
        assert set(got.tolist()) <= allowed, f"probe {p}: rows outside the tie band {sorted(set(got.tolist()) - allowed)}"


# ------------------------------------------------------------------ generators
def signed_permutations(n, d, seed):
    """Rows that are signed permutations of one small-integer base vector (|v| <= 2047, and small enough that the squared norm
    stays below 2^24): every row has the same norm, computed exactly in fp32, and with the probes of `exact_probes` every dot
    product is exact, so the ranking is the exact integer-dot ranking and ties are real."""
    rng = np.random.default_rng(seed)
    amp = int(min(2047, np.sqrt(2.0 ** 24 / d)))
    base = rng.integers(-amp, amp + 1, size=d)
    base[0] = amp                                    # never the zero vector
    X = np.empty((n, d), np.float32)
    for i in range(n):
        X[i] = (base[rng.permutation(d)] * rng.choice([-1, 1], size=d)).astype(np.float32)
    return X


def exact_probes(q, d, seed):
    """Probes of 4 (d >= 4) or 1 entries +-1: their unit vectors hold +-0.5 / +-1, exact in fp32."""
    rng = np.random.default_rng(seed)
    P = np.zeros((q, d))
    m = 4 if d >= 4 else 1
    for p in range(q):
        P[p, rng.choice(d, m, replace=False)] = rng.choice([-1.0, 1.0], size=m)
    return P


def gaussian(n, d, seed, dtype=np.float32):
    return np.random.default_rng(seed).standard_normal((n, d)).astype(dtype)


def clustered(n, d, seed, clusters=8, spread=0.05, dtype=np.float32):
    rng = np.random.default_rng(seed)
    centres = rng.standard_normal((clusters, d))
    X = centres[rng.integers(0, clusters, size=n)] + spread * rng.standard_normal((n, d))
    return X.astype(dtype)


def vector_array(X, dtype=pa.float32()) -> pa.FixedSizeListArray:
    X = np.asarray(X)
    return pa.FixedSizeListArray.from_arrays(pa.array(X.reshape(-1), type=dtype), X.shape[1])


# ------------------------------------------------------------------ API cases
def api_stream(n=600, d=12, seed=5):
    """A stream table: id, a category, a price and a vector column; and its exact vectors."""
    rng = np.random.default_rng(seed)
    X = clustered(n, d, seed, clusters=5, spread=0.3)
    X[7] = 0.0                                       # a zero row: never a neighbour
    X[11, 3] = np.nan                                # a NaN row: never a neighbour
    tbl = pa.table({"id": pa.array(np.arange(n, dtype=np.int64)), "cat": pa.array(rng.integers(0, 4, n).astype(np.int32)),
                    "price": pa.array(rng.random(n)), "vec": vector_array(X)})
    return tbl, X


def api_probes(d=12, q=5, seed=9):
    rng = np.random.default_rng(seed)
    P = rng.standard_normal((q, d))
    return pa.table({"pid": pa.array(np.arange(q, dtype=np.int64) + 100), "vec": vector_array(P.astype(np.float32)),
                     "label": pa.array([f"p{i}" for i in range(q)])}), P.astype(np.float32)


def _raises(exc, fn, needle=None):
    try:
        fn()
    except exc as e:
        assert needle is None or needle in str(e), f"{needle!r} not in {e}"
        return
    raise AssertionError(f"{fn} did not raise {exc.__name__}")


def case_vector_roundtrip(qc):
    """fixed_size_list<f32> round-trips bit for bit (NaN payloads and -0 included); f16 stays f16; list<double> is rounded once to
    f32."""
    X = gaussian(37, 5, 1)
    X[3, 2], X[4, 0] = np.nan, -0.0
    t = pa.table({"i": pa.array(np.arange(37)), "v": vector_array(X)})
    out = qc.from_arrow(t).collect()
    assert out.schema.field("v").type == pa.list_(pa.float32(), 5)
    got = np.asarray(out["v"].combine_chunks().values.to_numpy(zero_copy_only=False)).reshape(37, 5)
    assert got.view(np.uint32).tolist() == X.view(np.uint32).tolist()
    H = X.astype(np.float16)
    out = qc.from_arrow(pa.table({"v": vector_array(H, pa.float16())})).collect()
    assert out.schema.field("v").type == pa.list_(pa.float16(), 5)
    assert out["v"].combine_chunks().values.to_numpy(zero_copy_only=False).view(np.uint16).tolist() == H.reshape(-1).view(np.uint16).tolist()
    D = np.random.default_rng(2).standard_normal((9, 3))
    out = qc.from_arrow(pa.table({"v": pa.array(D.tolist(), type=pa.list_(pa.float64()))})).collect()
    got = out["v"].combine_chunks().values.to_numpy(zero_copy_only=False).reshape(9, 3)
    assert got.dtype == np.float32 and (got == D.astype(np.float32)).all()
    import pandas as pd
    df = pd.DataFrame({"k": [1, 2], "v": [np.arange(4, dtype=np.float32), np.ones(4, dtype=np.float32)]})
    out = qc.from_pandas(df).collect()
    assert out["v"].combine_chunks().values.to_numpy(zero_copy_only=False).tolist() == [0, 1, 2, 3, 1, 1, 1, 1]


def case_vector_rejects(qc):
    from quokka_b200._lib import QkError
    bad = {"ragged": pa.array([[1.0, 2.0], [3.0]], type=pa.list_(pa.float32())),
           "null row": pa.array([[1.0, 2.0], None], type=pa.list_(pa.float32())),
           "null element": pa.array([[1.0, None], [3.0, 4.0]], type=pa.list_(pa.float32())),
           "integers": pa.array([[1, 2], [3, 4]], type=pa.list_(pa.int32())),
           "strings": pa.array([["a"], ["b"]], type=pa.list_(pa.string())),
           "too wide": vector_array(np.zeros((2, 4097), np.float32))}
    for what, arr in bad.items():
        _raises(QkError, lambda: qc.from_arrow(pa.table({"emb": arr})).collect(), "emb")


def case_vector_ops(qc):
    """select / drop / rename / filter on scalar columns / union / collect carry the vectors row for row."""
    tbl, X = api_stream(n=300, d=6)
    s = qc.from_arrow(tbl)
    f = s.filter("cat = 2 and price > 0.3").select(["id", "vec"]).rename({"vec": "e"})
    out = f.collect()
    keep = np.nonzero((tbl["cat"].to_numpy() == 2) & (tbl["price"].to_numpy() > 0.3))[0]
    ids = out["id"].to_numpy()
    assert sorted(ids.tolist()) == keep.tolist()
    got = out["e"].combine_chunks().values.to_numpy(zero_copy_only=False).reshape(-1, 6)
    assert got.view(np.uint32).tolist() == X[ids].view(np.uint32).tolist()
    out = s.drop(["price"]).filter(s["id"] < 10).collect()
    assert out.column_names == ["id", "cat", "vec"] and sorted(out["id"].to_numpy().tolist()) == list(range(10))
    u = s.filter("id < 5").union(s.filter("id >= 295")).collect()
    ids = u["id"].to_numpy()
    assert sorted(ids.tolist()) == list(range(5)) + list(range(295, 300))
    got = u["vec"].combine_chunks().values.to_numpy(zero_copy_only=False).reshape(-1, 6)
    assert got.view(np.uint32).tolist() == X[ids].view(np.uint32).tolist()


def case_vector_plan_errors(qc):
    """Every use that reads a vector column as a value or a key is refused while the plan is built, naming the column."""
    tbl, _ = api_stream(n=50, d=4)
    s = qc.from_arrow(tbl)
    other = qc.from_arrow(pa.table({"id": pa.array(np.arange(5, dtype=np.int64)), "w": pa.array(np.ones(5))}))
    for fn in (lambda: s.groupby("vec").agg({"price": "sum"}), lambda: s.join(other, left_on="vec", right_on="id"),
               lambda: s.join(other, on="id"), lambda: other.join(s, on="id"), lambda: s.filter("vec > 1"),
               lambda: s.with_columns({"z": s["vec"] + 1}), lambda: s.top_k(["vec"], 3), lambda: s.distinct(["vec"]),
               lambda: s.gramian(["vec"]), lambda: s.approximate_quantile(["vec"], 0.5)):
        _raises(NotImplementedError, fn, "'vec'")


def _join_arrays(out: pa.Table, vec_out="vec", score=None):
    ids = out["id"].to_numpy()
    vec = out[vec_out].combine_chunks().values.to_numpy(zero_copy_only=False).reshape(len(ids), -1)
    sc = out[score].to_numpy() if score else None
    return ids, vec, sc


def check_join(out: pa.Table, tbl, X, probes, P, k, score="score"):
    """vector_nn_join's output against the fp64 reference: columns, per-probe row counts and order, the probe columns, the score."""
    assert out.column_names == tbl.column_names + [c + "_probe" if c in tbl.column_names else c for c in probes.column_names] + [score]
    phat = normalise(P)
    er, es = exact_topk(X, phat, k)
    pids = out["pid"].to_numpy()
    q = len(P)
    nvalid = (er >= 0).sum(axis=1)
    expect_pid = np.repeat(probes["pid"].to_numpy(), nvalid)
    assert pids.tolist() == expect_pid.tolist(), "probes must come out in probe order with min(k, valid rows) rows each"
    ids, vec, sc = _join_arrays(out, score=score)
    assert vec.view(np.uint32).tolist() == X[ids].view(np.uint32).tolist()
    pv = out["vec_probe"].combine_chunks().values.to_numpy(zero_copy_only=False).reshape(len(ids), -1)
    pos = np.repeat(np.arange(q), nvalid)
    assert (pv == P[pos]).all()
    assert out["label"].to_pylist() == [f"p{i}" for i in pos]
    scores = np.full((q, k), -np.inf)
    rows = np.full((q, k), -1, np.int64)
    o = 0
    for p in range(q):
        scores[p, :nvalid[p]] = sc[o:o + nvalid[p]]
        rows[p, :nvalid[p]] = ids[o:o + nvalid[p]]
        o += nvalid[p]
    check_topk(X, phat, k, scores, rows)


def case_knn_api(qc, chunk_rows=97):
    tbl, X = api_stream()
    probes, P = api_probes()
    qc.set_config("chunk_rows", chunk_rows)                 # several batches: the per-rank merge runs
    s = qc.from_arrow(tbl)
    for k in (1, 4, 17):
        check_join(s.vector_nn_join(probes, vec_column="vec", k=k, score_column="score").collect(), tbl, X, probes, P, k)
    out = s.vector_nn_join(probes, vec_column="vec", k=3).collect()
    assert out.column_names == tbl.column_names + ["pid", "vec_probe", "label"]
    out = s.filter("cat = 1").vector_nn_join(probes.rename_columns(["pid", "q", "label"]), vec_column_left="vec",
                                             vec_column_right="q", k=2, suffix="_x").collect()
    keep = np.nonzero(tbl["cat"].to_numpy() == 1)[0]
    er, _ = exact_topk(X[keep], normalise(P), 2)
    assert out.column_names == tbl.column_names + ["pid", "q", "label"]
    assert len(out) == 2 * len(P) and set(out["id"].to_numpy().tolist()) <= set(keep.tolist())


def case_knn_fewer_rows(qc):
    """A stream with fewer valid rows than k: each probe gets what there is, best first; zero / NaN rows never match."""
    X = np.array([[1, 0, 0], [0, 0, 0], [0, 1, 0], [np.nan, 1, 1], [1, 1, 0]], np.float32)
    tbl = pa.table({"id": pa.array(np.arange(5, dtype=np.int64)), "vec": vector_array(X)})
    probes = pa.table({"pid": pa.array([0, 1]), "vec": vector_array(np.array([[1, 0, 0], [0, 0, 1]], np.float32))})
    out = qc.from_arrow(tbl).vector_nn_join(probes, vec_column="vec", k=8, score_column="s").collect()
    assert out["pid"].to_pylist() == [0, 0, 0, 1, 1, 1]
    assert out["id"].to_pylist() == [0, 4, 2, 0, 2, 4]          # probe 1 scores 0 for all three: ties by row
    assert out["s"].to_pylist()[3:] == [0.0, 0.0, 0.0]


def case_knn_args(qc):
    tbl, _ = api_stream(n=40, d=12)
    probes, P = api_probes()
    s = qc.from_arrow(tbl)
    _raises(NotImplementedError, lambda: s.vector_nn_join(probes, vec_column="vec", probe_side="left", tmp_directory="/tmp"))
    zero = pa.table({"vec": vector_array(np.vstack([P[:1], np.zeros((1, 12), np.float32)]))})
    _raises(ValueError, lambda: s.vector_nn_join(zero, vec_column="vec"), "zero norm")
    nan = P.copy()
    nan[1, 2] = np.nan
    _raises(ValueError, lambda: s.vector_nn_join(pa.table({"vec": vector_array(nan)}), vec_column="vec"), "non-finite")
    _raises(AssertionError, lambda: s.vector_nn_join(probes, vec_column="vec", k=0))
    _raises(ValueError, lambda: s.vector_nn_join(probes, vec_column="vec", k=257))
    _raises(AssertionError, lambda: s.vector_nn_join(probes, vec_column="vec", vec_column_left="vec"))
    _raises(AssertionError, lambda: s.vector_nn_join(probes, vec_column="nope"))
    _raises(AssertionError, lambda: s.vector_nn_join(probes, vec_column="vec", score_column="id"))
    import pandas as pd
    df = pd.DataFrame({"pid": [1], "vec": [P[0]]})
    out = s.vector_nn_join(df, vec_column="vec", k=2).collect()
    assert len(out) == 2 and out.column_names[-2:] == ["pid", "vec_probe"]


def case_vector_parquet(qc, tmp_dir):
    """read_parquet of a vector column through the host Arrow decode, over several row groups; the device decoder refuses it."""
    import os
    import pyarrow.parquet as pq
    from quokka_b200._lib import QkError
    X = gaussian(1000, 6, 21)
    path = os.path.join(str(tmp_dir), "vectors.parquet")
    pq.write_table(pa.table({"id": pa.array(np.arange(1000, dtype=np.int64)), "vec": vector_array(X)}), path, row_group_size=128)
    qc.set_config("device_parquet", False)
    out = qc.read_parquet(path).filter("id >= 300 and id < 700").collect()
    ids = out["id"].to_numpy()
    assert sorted(ids.tolist()) == list(range(300, 700))
    got = out["vec"].combine_chunks().values.to_numpy(zero_copy_only=False).reshape(-1, 6)
    assert got.view(np.uint32).tolist() == X[ids].view(np.uint32).tolist()
    qc.set_config("device_parquet", True)
    try:
        _raises(QkError, lambda: qc.read_parquet(path).collect(), "nested list")
    finally:
        qc.set_config("device_parquet", False)


def case_vector_empty_chunk(device):
    """An empty chunk of a variable-size list column does not know its row length; concatenating it with real rows works."""
    from quokka_b200.columns import DeviceTable, concat_tables
    empty = DeviceTable.from_arrow(pa.table({"v": pa.array([], type=pa.list_(pa.float32()))}), device)
    full = DeviceTable.from_arrow(pa.table({"v": pa.array([[1.0, 2.0, 3.0], [4.0, 5.0, 6.0]], type=pa.list_(pa.float32()))}), device)
    fixed_empty = DeviceTable.from_arrow(pa.table({"v": vector_array(np.zeros((0, 3), np.float32))}), device)
    assert tuple(fixed_empty["v"].data.shape) == (0, 3)
    t = concat_tables([empty, full, fixed_empty, full])
    assert tuple(t["v"].data.shape) == (4, 3)
    assert t.to_arrow()["v"].to_pylist() == [[1.0, 2.0, 3.0], [4.0, 5.0, 6.0]] * 2
