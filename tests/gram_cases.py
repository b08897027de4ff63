"""DataStream.gramian / covariance cases, written once and run against tests/cpu_shim.py + tests/gram_shim.py (tests/test_gram_cpu.py, also on two
gloo ranks) and against the real kernels (tests/test_gpu_gram.py), plus the reference computation they are checked with.

Reference: G_ref = (X - c)^T (X - c) with the shifted values rounded in fp64 first (as numpy's `x - demean`), then products and
sums in extended precision (np.longdouble: 64-bit significand).  Bound: a sum of n fp64 products in any order is within
n * 2^-53 * (|X - c|^T |X - c|) of the exact value; the reference's own error (one rounding of the result, plus 2^-64 per term)
is a small fraction of that (test_gram_cpu.py checks it against exact rational arithmetic)."""
from __future__ import annotations

import numpy as np
import pyarrow as pa

import api_cases as A
from oracle import tpch_gen as G

LINEITEM_COLS = ["l_quantity", "l_extendedprice", "l_discount", "l_tax"]       # apps/tpc-h/tpch.py:600-602


def gram_ref(x: np.ndarray, shift=None):
    """(G_ref, bound): x is n x k fp64 (NaN allowed), shift None or fp64[k]."""
    y = x if shift is None else x - np.asarray(shift, dtype=np.float64)
    yl = y.astype(np.longdouble)
    g = (yl.T @ yl).astype(np.float64)
    a = np.abs(y)
    bound = max(len(y), 1) * 2.0 ** -53 * (a.T @ a)
    return g, bound


def cov_ref(x: np.ndarray):
    """(covariance divided by n, bound) of the rows of x: the mean in extended precision, then gram_ref of the centred data.
    covariance() shifts each rank by one of its rows c and re-centres at the end, so its sums run over |x - c| <= |x - mu| + D
    (D = the largest deviation of a row from the mean): the bound is that of the sums over |x - mu| + D, three times over
    (G, the sums times the re-centring offset, and the rounding of the result)."""
    n = len(x)
    mu = (x.astype(np.longdouble).sum(axis=0) / n).astype(np.float64)
    g, _ = gram_ref(x, mu)
    a = np.abs(x - mu)
    a = a + a.max(axis=0)
    return g / n, 3 * 2.0 ** -53 * (a.T @ a) + 2.0 ** -52 * np.abs(g) / n


def assert_within(got, ref, bound, what=""):
    got = np.asarray(got, dtype=np.float64)
    nan = np.isnan(ref)
    assert np.array_equal(np.isnan(got), nan), f"{what}: NaN pattern differs"
    err = np.abs(got - ref)[~nan]
    lim = bound[~nan]
    assert np.all(err <= lim), f"{what}: max excess {np.max(err - lim)} (max err {np.max(err)})"


def table_matrix(t: pa.Table, columns) -> np.ndarray:
    assert t.column_names == list(columns)
    assert t.num_rows == len(columns)
    return np.stack([t[c].to_numpy(zero_copy_only=False).astype(np.float64) for c in columns], axis=1)


def _x(tbl: pa.Table, columns) -> np.ndarray:
    return np.stack([tbl[c].to_numpy(zero_copy_only=False).astype(np.float64) for c in columns], axis=1)


def case_gram_lineitem(qc):
    """tpch.py:600-602: lineitem.gramian(...) -- and the same with demean, and covariance -- against the reference."""
    li = A.tables()[0]
    x = _x(li, LINEITEM_COLS)
    d = qc.from_arrow(li)
    g, b = gram_ref(x)
    assert_within(table_matrix(d.gramian(LINEITEM_COLS).collect(), LINEITEM_COLS), g, b, "gramian")
    mean = x.mean(axis=0)
    g, b = gram_ref(x, mean)
    assert_within(table_matrix(d.gramian(LINEITEM_COLS, demean=mean).collect(), LINEITEM_COLS), g, b, "gramian demean")
    c, b = cov_ref(x)
    cov = table_matrix(d.covariance(LINEITEM_COLS), LINEITEM_COLS)
    assert_within(cov, c, b, "covariance")
    np.testing.assert_allclose(cov, np.cov(x, rowvar=False, bias=True), rtol=1e-9, atol=0)


def case_gram_filtered_ints(qc):
    """A filter in front of the gramian (the existing edge applies it); integer and float columns mixed."""
    li = A.tables()[0]
    cols = ["l_orderkey", "l_quantity", "l_extendedprice", "l_linenumber"]
    d = qc.from_arrow(li).filter_sql("l_discount >= 0.05 and l_quantity < 30")
    keep = (li["l_discount"].to_numpy() >= 0.05) & (li["l_quantity"].to_numpy() < 30)
    x = _x(li, cols)[keep]
    g, b = gram_ref(x)
    assert_within(table_matrix(d.gramian(cols).collect(), cols), g, b, "filtered gramian")
    c, b = cov_ref(x)
    assert_within(table_matrix(d.covariance(cols), cols), c, b, "filtered covariance")


def case_gram_ragged_batches(qc):
    """from_device in batches of 997 rows: the state accumulates over batches of every size."""
    from quokka_b200.columns import DeviceTable
    rng = np.random.default_rng(7)
    n = 10_007
    cols = {"a": rng.normal(1e3, 1.0, n), "b": rng.integers(-50, 50, n).astype(np.int32),
            "c": rng.normal(0, 1e-3, n).astype(np.float32), "d": rng.integers(0, 1 << 40, n).astype(np.int64)}
    names = list(cols)
    d = qc.from_device(DeviceTable.from_numpy(cols), batch_rows=997)
    x = np.stack([cols[c].astype(np.float64) for c in names], axis=1)
    g, b = gram_ref(x)
    assert_within(table_matrix(d.gramian(names).collect(), names), g, b, "ragged gramian")
    shift = np.array([1e3, 0.5, 0.0, 2.0 ** 39])
    g, b = gram_ref(x, shift)
    assert_within(table_matrix(d.gramian(names, demean=shift).collect(), names), g, b, "ragged gramian demean")
    c, b = cov_ref(x)
    assert_within(table_matrix(d.covariance(names), names), c, b, "ragged covariance")


def case_gram_left_join_nulls(qc):
    """The right side of a left join carries NULLs: they count as NaN (Polars to_numpy), so every entry that touches that
    column is NaN and the others are exact."""
    n = 3000
    rng = np.random.default_rng(3)
    left = pa.table({"k": np.arange(n, dtype=np.int64), "x": rng.normal(5, 2, n)})
    rk = np.arange(0, n, 3, dtype=np.int64)
    right = pa.table({"k": rk, "y": rng.normal(-1, 1, len(rk))})
    j = qc.from_arrow(left).join(qc.from_arrow(right), on="k", how="left")
    yfull = np.full(n, np.nan)
    yfull[rk] = right["y"].to_numpy()
    x = np.stack([left["x"].to_numpy(), yfull], axis=1)
    with np.errstate(invalid="ignore"):
        g, b = gram_ref(x)
    got = table_matrix(j.gramian(["x", "y"]).collect(), ["x", "y"])
    assert_within(got, g, np.nan_to_num(b), "gramian with nulls")
    assert np.isfinite(got[0, 0]) and np.isnan(got[0, 1]) and np.isnan(got[1, 1])
    cov = table_matrix(j.covariance(["x", "y"]), ["x", "y"])
    assert np.isfinite(cov[0, 0]) and np.isnan(cov[0, 1]) and np.isnan(cov[1, 0]) and np.isnan(cov[1, 1])


def case_gram_empty(qc):
    """No row reaches the gramian: k x k zeros; the covariance of nothing is NaN."""
    li = A.tables()[0]
    d = qc.from_arrow(li).filter_sql("l_quantity < 0")
    g = table_matrix(d.gramian(LINEITEM_COLS).collect(), LINEITEM_COLS)
    assert np.array_equal(g, np.zeros((4, 4)))
    c = table_matrix(d.covariance(LINEITEM_COLS), LINEITEM_COLS)
    assert np.all(np.isnan(c))


def case_gram_rejects_strings_and_dates(qc):
    import pytest
    li = A.tables()[0]
    d = qc.from_arrow(li)
    with pytest.raises(Exception, match="string column"):
        d.gramian(["l_quantity", "l_returnflag"]).collect()
    with pytest.raises(Exception, match="not a number"):
        d.covariance(["l_shipdate", "l_quantity"])
