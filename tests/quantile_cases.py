"""DataStream.approximate_quantile / approximate_median cases, written once and run against tests/cpu_shim.py +
tests/quantile_shim.py (tests/test_quantile_cpu.py, also on two gloo ranks) and against the real kernels
(tests/test_gpu_quantile.py), plus the two references they are checked with:

- `quantile_nearest`: the exact target, Polars' quantile(q) with interpolation "nearest" (the reference's materialised
  branch, pyquokka/datastream.py:1024): NULLs dropped, values sorted ascending with NaN last, element
  round-half-away((n - 1) q) (Rust's f64::round; numpy's method="nearest" rounds half to even and is not this rule).
- `sketch_entries` / `sketch_quantiles`: the device sketch restated in numpy -- per (column, image >> 42) bucket the count,
  the min and the max image; the answer is the min at the bucket's first rank, the max at its last, else the bucket's middle
  image clamped to [min, max].  Results must equal it bit for bit and meet the guarantee (`check_guarantee`) against the
  exact target."""
from __future__ import annotations

import numpy as np
import pyarrow as pa

import api_cases as A
import gram_cases as GC

SHIFT = 42
SIGN = np.uint64(1 << 63)
CANON_NAN = np.uint64(0x7FF8000000000000)
QUANT_COLS = ["l_quantity", "l_extendedprice", "l_discount", "l_tax"]
EXACT_COLS = ["l_quantity", "l_discount", "l_tax"]          # every bucket holds one distinct value


def round_half_away(v: float) -> int:
    f = np.floor(v)
    return int(f) + int(v - f >= 0.5)


def quantile_nearest(x: np.ndarray, q: float):
    """Polars' quantile(q, interpolation="nearest") of the non-NULL values x (fp64): None when x is empty."""
    x = np.asarray(x, dtype=np.float64)
    if len(x) == 0:
        return None
    return float(np.sort(x)[round_half_away((len(x) - 1) * float(q))])          # np.sort puts NaN last


def images(x: np.ndarray) -> np.ndarray:
    """Order-preserving uint64 image of every value widened to fp64 (NaN first made the canonical quiet NaN)."""
    d = np.asarray(x).astype(np.float64)
    b = d.view(np.uint64).copy()
    b[np.isnan(d)] = CANON_NAN
    return np.where((b >> np.uint64(63)) == 1, ~b, b | SIGN)


def value_of(img: int) -> float:
    img = np.uint64(img)
    b = img ^ SIGN if img >> np.uint64(63) else ~img
    return float(np.array([b], dtype=np.uint64).view(np.float64)[0])


def sketch_entries(columns, masks=None):
    """(key, count, min image, max image) uint64 arrays sorted by key, key = column << 22 | image >> 42."""
    ks, ims = [], []
    for c, x in enumerate(columns):
        x = np.asarray(x)
        if masks is not None and masks[c] is not None:
            x = x[np.asarray(masks[c]).astype(bool)]
        img = images(x)
        ks.append((np.uint64(c) << np.uint64(22)) | (img >> np.uint64(SHIFT)))
        ims.append(img)
    key, img = np.concatenate(ks), np.concatenate(ims)
    if len(key) == 0:
        e = np.zeros(0, dtype=np.uint64)
        return e, e.copy(), e.copy(), e.copy()
    order = np.lexsort((img, key))
    key, img = key[order], img[order]
    first = np.concatenate([[0], np.flatnonzero(np.diff(key)) + 1])
    last = np.concatenate([first[1:] - 1, [len(key) - 1]])
    return key[first], (last - first + 1).astype(np.uint64), img[first], img[last]


def sketch_quantiles(entries, k, qs):
    """(fp64 [len(qs), k], bool valid [len(qs), k]) answered from sketch entries, one bucket at a time."""
    key, cnt, mn, mx = (np.asarray(e, dtype=np.uint64) for e in entries)
    order = np.argsort(key, kind="stable")
    key, cnt, mn, mx = key[order], cnt[order], mn[order], mx[order]
    out = np.full((len(qs), k), np.nan)
    valid = np.zeros((len(qs), k), dtype=bool)
    for c in range(k):
        sel = (key >> np.uint64(22)) == c
        kc, cc, lo_img, hi_img = key[sel], cnt[sel].astype(np.int64), mn[sel], mx[sel]
        n = int(cc.sum())
        if n == 0:
            continue
        cum = np.cumsum(cc)
        for i, q in enumerate(qs):
            r = round_half_away((n - 1) * float(q))
            b = int(np.searchsorted(cum, r, side="right"))
            first, last = int(cum[b] - cc[b]), int(cum[b] - 1)
            bucket = int(kc[b]) & ((1 << 22) - 1)
            mid = (bucket << SHIFT) | (1 << (SHIFT - 1))
            a, z = int(lo_img[b]), int(hi_img[b])
            img = a if r == first else z if r == last else min(max(mid, a), z)
            out[i, c] = value_of(img)
            valid[i, c] = True
    return out, valid


def check_guarantee(got: float, x: np.ndarray, q: float, what=""):
    """The documented guarantee of approximate_quantile against the exact target of the non-NULL values x."""
    x = np.asarray(x, dtype=np.float64)
    t = quantile_nearest(x, q)
    if np.isnan(t):
        assert np.isnan(got), f"{what}: target NaN, got {got}"
        return
    tb = int(images(np.array([t]))[0]) >> SHIFT
    same = x[(images(x) >> np.uint64(SHIFT)) == tb]
    if len(np.unique(same)) == 1 or q in (0, 1) or q == 0.0 or q == 1.0:
        assert got == t, f"{what}: q={q} must be exact: got {got!r}, target {t!r}"
    elif abs(t) >= 2.0 ** -1022:
        assert abs(got - t) <= 2.0 ** -11 * abs(t), f"{what}: q={q}: got {got!r}, target {t!r}"
    else:
        assert abs(got - t) <= 2.0 ** (41 - 1074), f"{what}: q={q}: subnormal got {got!r}, target {t!r}"


def table_values(t: pa.Table, columns, nq):
    """(fp64 [nq, k] with NaN for NULL, valid [nq, k]) of a result table, after checking its shape and types."""
    assert t.column_names == list(columns)
    assert t.num_rows == nq
    vals = np.full((nq, len(columns)), np.nan)
    valid = np.zeros((nq, len(columns)), dtype=bool)
    for j, c in enumerate(columns):
        col = t[c].combine_chunks()
        assert pa.types.is_float64(col.type), f"{c}: {col.type}"
        valid[:, j] = col.is_valid().to_numpy(zero_copy_only=False)
        vals[:, j] = col.fill_null(np.nan).to_numpy(zero_copy_only=False)
    return vals, valid


def assert_matches(t: pa.Table, columns, qs, xs, masks=None, what=""):
    """Result table == numpy sketch bit for bit (and NULL where a column has no rows), and the guarantee holds."""
    got, gvalid = table_values(t, columns, len(qs))
    ref, rvalid = sketch_quantiles(sketch_entries(xs, masks), len(columns), qs)
    assert np.array_equal(gvalid, rvalid), f"{what}: NULL pattern {gvalid} != {rvalid}"
    assert np.array_equal(got[rvalid].view(np.uint64), ref[rvalid].view(np.uint64)), f"{what}: {got} != sketch {ref}"
    for j, x in enumerate(xs):
        x = np.asarray(x)
        if masks is not None and masks[j] is not None:
            x = x[np.asarray(masks[j]).astype(bool)]
        for i, q in enumerate(qs):
            if len(x):
                check_guarantee(got[i, j], x, q, f"{what} {columns[j]}")
    return got, gvalid


def _cols(tbl, columns):
    return [tbl[c].to_numpy(zero_copy_only=False) for c in columns]


def case_quantile_lineitem(qc):
    """lineitem columns at several quantile lists; l_quantity / l_discount / l_tax are exact."""
    li = A.tables()[0]
    d = qc.from_arrow(li)
    xs = _cols(li, QUANT_COLS)
    for qs in ([0.1, 0.5, 0.9], [0.0, 1.0], [0.25], [0.999, 0.001, 0.5, 0.5], [0, 1]):
        got, _ = assert_matches(d.approximate_quantile(QUANT_COLS, qs).collect(), QUANT_COLS, qs, xs, what=f"lineitem {qs}")
        for j, c in enumerate(QUANT_COLS):
            if c in EXACT_COLS:
                assert [quantile_nearest(xs[j], q) for q in qs] == list(got[:, j]), c


def case_quantile_tpch_606(qc):
    """apps/tpc-h/tpch.py:606 verbatim, and approximate_median."""
    lineitem = qc.from_arrow(A.tables()[0])
    t = lineitem.approximate_quantile(["l_tax"], 0.9).collect()
    x = A.tables()[0]["l_tax"].to_numpy()
    assert_matches(t, ["l_tax"], [0.9], [x], what="tpch.py:606")
    assert t["l_tax"][0].as_py() == quantile_nearest(x, 0.9)
    m = lineitem.approximate_median(["l_tax", "l_quantity"]).collect()
    assert_matches(m, ["l_tax", "l_quantity"], [0.5], _cols(A.tables()[0], ["l_tax", "l_quantity"]), what="median")


def special_columns(n, seed):
    """Columns of every supported dtype with NaN / +-0 / +-inf / subnormals / negatives mixed in."""
    rng = np.random.default_rng(seed)
    f64 = rng.lognormal(0, 8, n) * rng.choice([-1.0, 1.0], n)
    special = np.array([np.nan, -np.nan, 0.0, -0.0, np.inf, -np.inf, 5e-324, -5e-324, 2.0 ** -1030, 1.0, -1.0])
    k = min(n, n // 7 + 1)
    f64[rng.integers(0, n, k)] = special[rng.integers(0, len(special), k)]
    f32 = (rng.normal(0, 100, n)).astype(np.float32)
    f32[rng.integers(0, n, k)] = special[rng.integers(0, len(special), k)].astype(np.float32)
    i64 = rng.integers(-(1 << 62), 1 << 62, n)
    i64[rng.integers(0, n, k)] = rng.integers(-3000, 3000, k)
    i32 = rng.integers(-2_000_000_000, 2_000_000_000, n).astype(np.int32)
    u8 = rng.integers(0, 256, n).astype(np.uint8)
    return {"f64": f64, "f32": f32, "i64": i64, "i32": i32, "u8": u8}


def case_quantile_ragged_batches(qc):
    """from_device in batches of 997 rows gives bit-identical answers to one batch, on every dtype and special value."""
    from quokka_b200.columns import DeviceTable
    cols = special_columns(10_007, 7)
    names = list(cols)
    qs = [0.0, 0.01, 0.3, 0.5, 0.77, 0.99, 1.0]
    whole = qc.from_device(DeviceTable.from_numpy(cols)).approximate_quantile(names, qs).collect()
    ragged = qc.from_device(DeviceTable.from_numpy(cols), batch_rows=997).approximate_quantile(names, qs).collect()
    a, _ = assert_matches(whole, names, qs, [cols[c] for c in names], what="whole")
    b, _ = assert_matches(ragged, names, qs, [cols[c] for c in names], what="ragged")
    assert np.array_equal(a.view(np.uint64), b.view(np.uint64))


def case_quantile_left_join_nulls(qc):
    """The right side of a left join carries NULLs: they are skipped.  A column whose every row is NULL gives NULL."""
    n = 3000
    rng = np.random.default_rng(3)
    left = pa.table({"k": np.arange(n, dtype=np.int64), "x": rng.normal(5, 2, n)})
    rk = np.arange(0, n, 3, dtype=np.int64)
    right = pa.table({"k": rk, "y": rng.normal(-1, 1, len(rk))})
    j = qc.from_arrow(left).join(qc.from_arrow(right), on="k", how="left")
    yfull = np.zeros(n)
    yfull[rk] = right["y"].to_numpy()
    ymask = np.zeros(n, dtype=bool)
    ymask[rk] = True
    qs = [0.1, 0.5, 1.0]
    assert_matches(j.approximate_quantile(["x", "y"], qs).collect(), ["x", "y"], qs, [left["x"].to_numpy(), yfull],
                   [None, ymask], what="left join")
    none = pa.table({"k": np.arange(n, n + 10, dtype=np.int64), "z": np.ones(10)})
    jz = qc.from_arrow(left).join(qc.from_arrow(none), on="k", how="left")
    got, valid = table_values(jz.approximate_quantile(["x", "z"], qs).collect(), ["x", "z"], len(qs))
    assert valid[:, 0].all() and not valid[:, 1].any()


def case_quantile_empty(qc):
    """No row reaches the sketch: one NULL row per quantile."""
    li = A.tables()[0]
    d = qc.from_arrow(li).filter_sql("l_quantity < 0")
    got, valid = table_values(d.approximate_quantile(QUANT_COLS, [0.1, 0.9]).collect(), QUANT_COLS, 2)
    assert not valid.any()
    _, valid = table_values(d.approximate_median(["l_tax"]).collect(), ["l_tax"], 1)
    assert not valid.any()


def case_quantile_rejects(qc):
    """String and date columns raise; bad quantiles / sample_factor are refused as in the reference."""
    import pytest
    li = A.tables()[0]
    d = qc.from_arrow(li)
    with pytest.raises(Exception, match="string column"):
        d.approximate_quantile(["l_quantity", "l_returnflag"], 0.5).collect()
    with pytest.raises(Exception, match="not a number"):
        d.approximate_median(["l_shipdate"]).collect()
    for bad in (1.5, -0.1, [0.5, 2.0], "0.5", (0.1, 0.9), []):
        with pytest.raises(AssertionError):
            d.approximate_quantile(["l_tax"], bad)
    for sf in (0, -1, 1.5):
        with pytest.raises(AssertionError):
            d.approximate_quantile(["l_tax"], 0.5, sample_factor=sf)
    t = d.approximate_quantile(["l_tax"], 0.5, sample_factor=0.25).collect()     # accepted; every row is counted
    assert t["l_tax"][0].as_py() == quantile_nearest(li["l_tax"].to_numpy(), 0.5)


def case_quantile_winsorised_covariance(qc):
    """blog/approxquant.md, apps/andy.py: clip every column to its [0.1, 0.9] quantiles, then covariance()."""
    li = A.tables()[0]
    d = qc.from_arrow(li)
    z = d.approximate_quantile(QUANT_COLS, [0.1, 0.9]).collect()
    xs = _cols(li, QUANT_COLS)
    assert_matches(z, QUANT_COLS, [0.1, 0.9], xs, what="winsorising quantiles")
    bounds = {c: tuple(z[c].to_pylist()) for c in QUANT_COLS}
    cov = GC.table_matrix(d.clip(bounds).covariance(QUANT_COLS), QUANT_COLS)
    x = np.stack([np.clip(xs[j].astype(np.float64), *bounds[c]) for j, c in enumerate(QUANT_COLS)], axis=1)
    c, b = GC.cov_ref(x)
    GC.assert_within(cov, c, b, "winsorised covariance")
