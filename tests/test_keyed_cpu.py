"""The keyed-kernel references (tests/keyed_cases.py) on the CPU: each reference against a brute-force Python loop, the CPU
shim's HashAggState / JoinTable / topk_candidates against the references, executors.sort_table and top_k_table through the
shim on both sides of the 4 096-row host switch, and a grouped MIN / MAX over NaN data through the DataStream API."""
import math

import numpy as np
import pyarrow as pa
import pytest
import torch

import cpu_shim
import keyed_cases as K
from quokka_b200 import _lib as L

EDGE_F = [0.0, -0.0, K.NAN_POS, K.NAN_NEG, K.NAN_PAYLOAD, np.inf, -np.inf, 1.5, -1.5, 2.0]
EDGE_I64 = [K.I64_MIN, K.I64_MAX, K.I64_MIN + 1, K.I64_MAX - 1, -1, 0, 1, 7]


def _col(rng, dt, n):
    if dt == "f64":
        return np.array(EDGE_F)[rng.integers(0, len(EDGE_F), n)]
    if dt == "f32":
        with np.errstate(invalid="ignore"):
            return np.array(EDGE_F)[rng.integers(0, len(EDGE_F), n)].astype(np.float32)
    if dt == "i64":
        return np.array(EDGE_I64, np.int64)[rng.integers(0, len(EDGE_I64), n)]
    if dt == "i32":
        return np.array([K.I32_MIN, K.I32_MAX, -1, 0, 5], np.int32)[rng.integers(0, 5, n)]
    if dt == "u8":
        return rng.choice(np.array([0, 1, 255], np.uint8), n)
    return rng.integers(0, 2, n).astype(np.bool_)


# ------------------------------------------------------------------ references against brute force
def test_row_key_states_the_rules():
    asc = sorted([K.NAN_NEG, np.inf, -0.0, 0.0, -np.inf, K.NAN_POS, 1.0], key=lambda x: K.row_key(x, False))
    assert [repr(x) for x in asc[:2]] == ["-inf", "-0.0"] and asc[3:5] == [1.0, np.inf] and all(map(math.isnan, asc[5:]))
    desc = sorted([1.0, K.NAN_NEG, -np.inf, np.inf], key=lambda x: K.row_key(x, True))
    assert math.isnan(desc[0]) and desc[1:] == [np.inf, 1.0, -np.inf]
    assert sorted([K.I64_MIN, K.I64_MAX, 0], key=lambda x: K.row_key(x, True)) == [K.I64_MAX, 0, K.I64_MIN]
    assert K.row_key(5, True, False) > K.row_key(K.NAN_POS, True) and K.row_key(5, False, False) > K.row_key(K.NAN_POS, False)
    assert K.row_key(-0.0, False) == K.row_key(0.0, False)


@pytest.mark.parametrize("seed", range(12))
def test_ref_order_equals_python_sort(seed):
    rng = np.random.default_rng(seed)
    dts = ["f64", "f32", "i64", "i32", "u8", "bool"]
    ncol = 1 + seed % 4
    n = int(rng.integers(1, 300))
    cols = [_col(rng, dts[(seed + j) % len(dts)], n) for j in range(ncol)]
    desc = [bool(b) for b in rng.integers(0, 2, ncol)]
    valids = [None if rng.random() < 0.5 else (rng.random(n) > 0.2).astype(np.uint8) for _ in range(ncol)]
    assert np.array_equal(K.ref_order(cols, desc, valids), np.array(K.python_order(cols, desc, valids)))


@pytest.mark.parametrize("dt", ["f64", "f32", "i64", "i32", "u8", "bool"])
@pytest.mark.parametrize("desc", [False, True])
def test_ref_candidates_equal_brute_force(dt, desc):
    rng = np.random.default_rng(len(dt) * 2 + desc)
    v = _col(rng, dt, 200)
    for k in (1, 2, 37, 199, 200, 201):
        keys = [K.row_key(x.item(), desc) for x in v]
        kth = sorted(keys)[min(k, len(v)) - 1]
        assert K.ref_candidates(v, k, desc).tolist() == [i for i, x in enumerate(keys) if x <= kth], k


def test_ref_groupby_equals_python_loop():
    rng = np.random.default_rng(5)
    n = 3000
    keys = [K.int_keys(rng, np.int64, n, 7), K.int_keys(rng, np.int32, n, 5), K.int_keys(rng, np.uint8, n, 3)]
    v = K.float_values(rng, n, "normal", specials=True)
    ops = ["sum", "min", "max"]
    ref = K.ref_groupby(keys, [v, v, v], ops)
    groups = {}
    for i in range(n):
        groups.setdefault(tuple(int(k[i]) for k in keys), []).append(float(v[i]))
    assert [tuple(int(k[g]) for k in ref["keys"]) for g in range(len(ref["cnt"]))] == sorted(groups)
    for g, key in enumerate(sorted(groups)):
        xs = groups[key]
        fin = [x for x in xs if not math.isnan(x)]
        assert ref["cnt"][g] == len(xs)
        assert ref["vals"][1][g] == min(fin, default=math.inf) and ref["vals"][2][g] == max(fin, default=-math.inf)
        s = ref["vals"][0][g]
        if any(math.isnan(x) for x in xs) or (math.inf in xs and -math.inf in xs):
            assert math.isnan(s)
        elif math.inf in xs or -math.inf in xs:
            assert s == (math.inf if math.inf in xs else -math.inf)
    fin = np.isfinite(v)
    ref2 = K.ref_groupby([keys[0][fin]], [v[fin]], ["sum"])
    for g, key in enumerate(ref2["keys"][0]):
        assert ref2["vals"][0][g] == math.fsum(v[fin][keys[0][fin] == key])


@pytest.mark.parametrize("how", ["inner", "left", "semi", "anti"])
@pytest.mark.parametrize("dts", [("i64", "i64"), ("i32", "i64"), ("u8", "i32"), ("i64", "u8"), ("f64", "f64")])
def test_ref_join_equals_nested_loops(how, dts):
    rng = np.random.default_rng(len(how) + 10 * len(dts[0]))
    pool = {"i64": np.array([K.I64_MIN, K.I64_MAX, -1, 0, 200, 255, -(1 << 40)], np.int64),
            "i32": np.array([K.I32_MIN, -1, 0, 200, 255], np.int32), "u8": np.array([0, 200, 255], np.uint8),
            "f64": np.array([0.0, -0.0, np.inf, -np.inf, K.NAN_POS, 1.5], np.float64)}
    probe = rng.choice(pool[dts[0]], 60)
    build = rng.choice(pool[dts[1]], 40)
    build = build[K.join_key(build) != K.I64_MIN]
    pi, bi = K.ref_join(probe, build, how)
    bp, bb = K.brute_join(probe, build, how)
    assert np.array_equal(pi, bp) and (bi is None and bb is None or np.array_equal(bi, bb))
    with pytest.raises(ValueError):
        K.ref_join(probe, np.array([K.I64_MIN], np.int64), how)


# ------------------------------------------------------------------ the shim against the references
@pytest.mark.parametrize("layout", [("u8",), ("bool",), ("i32",), ("i64",), ("u8", "i64"), ("i32", "i32", "i32", "i32")])
def test_cpu_shim_hash_aggregate_matches_reference(layout):
    rng = np.random.default_rng(len(layout))
    n = 5000
    keys = [K.int_keys(rng, K.KEY_DTYPES[d], n, 40) for d in layout]
    v = K.float_values(rng, n, "dyadic", specials=True)
    st = cpu_shim.HashAggState([torch.from_numpy(k).dtype for k in keys], [L.AGG_SUM, L.AGG_MIN, L.AGG_MAX], 2 * n, "cpu")
    for lo in range(0, n, 1700):
        st.update([torch.from_numpy(k[lo:lo + 1700]) for k in keys], [torch.from_numpy(v[lo:lo + 1700])] * 3)
    ok, ov, oc = st.finalize()
    K.check_groupby([o.numpy() for o in ok], [o.numpy() for o in ov], oc.numpy(),
                    K.ref_groupby(keys, [v] * 3, ["sum", "min", "max"]), ["sum", "min", "max"], exact=True)
    with pytest.raises(L.QkError):
        st.finalize(max_groups=1)


def test_cpu_shim_hash_aggregate_min_max_skip_nan():
    """atomic_minmax in csrc/hashagg.cu (`!(v < cur)`) never stores a NaN; the shim used to let np.minimum.at through it."""
    k = np.array([0, 0, 0, 1, 1, 2], np.int64)
    v = np.array([K.NAN_POS, 3.0, -2.0, K.NAN_NEG, K.NAN_POS, 4.0])
    st = cpu_shim.HashAggState([torch.int64], [L.AGG_MIN, L.AGG_MAX], 16, "cpu")
    st.update([torch.from_numpy(k)], [torch.from_numpy(v)] * 2)
    _, ov, oc = st.finalize()
    assert ov[0].tolist() == [-2.0, math.inf, 4.0] and ov[1].tolist() == [3.0, -math.inf, 4.0] and oc.tolist() == [3, 2, 1]


@pytest.mark.parametrize("dt", ["f64", "f32", "i64", "i32", "u8", "bool"])
def test_cpu_shim_topk_candidates_match_reference(dt):
    rng = np.random.default_rng(len(dt))
    v = _col(rng, dt, 5000)
    for desc in (False, True):
        for k in (1, 10, 4999, 5000, 5001):
            got = cpu_shim.topk_candidates(torch.from_numpy(v), k, desc).numpy()
            assert got.tolist() == K.ref_candidates(v, k, desc).tolist(), (dt, desc, k)


@pytest.mark.parametrize("how", ["inner", "left", "semi", "anti"])
def test_cpu_shim_join_matches_reference(how):
    rng = np.random.default_rng(3)
    probe = K.int_keys(rng, np.int32, 3000, 300)
    build = K.int_keys(rng, np.int64, 2000, 300, edges=False)
    t = cpu_shim.JoinTable(len(build), "cpu")
    t.build(torch.from_numpy(build[:700]))
    t.build(torch.from_numpy(build[700:]))
    pi, bi = t.probe(torch.from_numpy(probe), {"inner": L.JOIN_INNER, "left": L.JOIN_LEFT, "semi": L.JOIN_SEMI, "anti": L.JOIN_ANTI}[how])
    rp, rb = K.ref_join(probe, build, how)
    assert np.array_equal(pi.numpy(), rp) and (bi is None or np.array_equal(bi.numpy(), rb))


# ------------------------------------------------------------------ sort_table / top_k_table through the shim
@pytest.fixture
def shim(monkeypatch):
    cpu_shim.install(monkeypatch)
    from quokka_b200 import executors
    return executors


def _table(cols, valids):
    from quokka_b200.columns import DeviceColumn, DeviceTable
    n = len(cols[0])
    d = {f"c{j}": DeviceColumn(torch.from_numpy(np.ascontiguousarray(c)), valid=None if m is None else torch.from_numpy(m))
         for j, (c, m) in enumerate(zip(cols, valids))}
    d["id"] = DeviceColumn(torch.arange(n, dtype=torch.int64))
    return DeviceTable(d)


def _run(X, cols, desc, valids, k, fn):
    t = _table(cols, valids)
    by = [f"c{j}" for j in range(len(cols))]
    out = X.top_k_table(t, by, desc, k) if fn == "top_k" else X.sort_table(t, by, desc, k)
    ids = out["id"].data.numpy()
    K.check_topk(ids, cols, desc, valids, k, tag=(fn, desc, k))
    for j, c in enumerate(cols):                                         # the values and masks travel with their rows
        assert np.array_equal(out[f"c{j}"].data.numpy(), c[ids], equal_nan=c.dtype.kind == "f")
        if valids[j] is not None:
            assert np.array_equal(out[f"c{j}"].valid.numpy(), valids[j][ids])
    return ids


@pytest.mark.parametrize("n", [4096, 4097, 20_000])
@pytest.mark.parametrize("case", range(8))
def test_top_k_table_orders_like_the_reference(shim, n, case):
    """Both sides of the 4 096-row switch: INT64_MIN / MAX, NaN of both signs, ±0 ties on the primary column decided by the
    second one, NULL primary and secondary columns, mixed ASC / DESC over 2-4 columns."""
    rng = np.random.default_rng(case * 101 + n)
    dts = [["i64", "f64"], ["f64", "i32"], ["f32", "u8", "i64"], ["i64", "i64"], ["u8", "bool", "f64", "i32"],
           ["f64", "f64"], ["i32", "f32", "i64"], ["bool", "i64"]][case]
    cols = [_col(rng, d, n) for d in dts]
    valids = [None] * len(cols)
    if case in (1, 3, 5, 6):
        valids[0] = (rng.random(n) > 0.3).astype(np.uint8)
    if case in (2, 5, 7):
        valids[1] = (rng.random(n) > 0.5).astype(np.uint8)
    for desc0 in (False, True):
        desc = [desc0] + [bool(b) for b in rng.integers(0, 2, len(cols) - 1)]
        for k in (1, 10, 3000, n - 1, n, n + 1):
            _run(shim, cols, desc, valids, k, "top_k")


def test_top_k_table_int64_min_desc(shim):
    """`-v` wrapped for INT64_MIN, which then sorted first in DESC order."""
    v = np.array([5, K.I64_MIN, K.I64_MAX, -3, K.I64_MIN + 1], np.int64)
    ids = _run(shim, [v], [True], [None], 5, "top_k")
    assert v[ids].tolist() == [K.I64_MAX, 5, -3, K.I64_MIN + 1, K.I64_MIN]
    assert v[_run(shim, [v], [False], [None], 2, "sort")].tolist() == [K.I64_MIN, K.I64_MIN + 1]


def test_sort_table_nulls_last_both_directions(shim):
    """A left join's unmatched row carries the gather placeholder 0 under valid == 0: it must not rank as 0."""
    v = np.array([3.0, 0.0, -1.0, 0.0, 7.0])
    m = np.array([1, 0, 1, 1, 0], np.uint8)
    for desc, want in ((False, [2, 3, 0]), (True, [0, 3, 2])):
        ids = _run(shim, [v], [desc], [m], 5, "sort")
        assert ids[:3].tolist() == want and sorted(ids[3:].tolist()) == [1, 4]


def test_sort_table_nan_and_signed_zero(shim):
    v = np.array([K.NAN_NEG, 1.0, -0.0, 0.0, K.NAN_POS, -np.inf])
    s = np.array([0, 0, 2, 1, 1, 0], np.int64)
    asc = _run(shim, [v, s], [False, False], [None, None], 6, "sort")
    assert asc.tolist()[:4] == [5, 3, 2, 1] and sorted(asc[4:].tolist()) == [0, 4]
    desc = _run(shim, [v, s], [True, True], [None, None], 6, "sort")
    assert sorted(desc[:2].tolist()) == [0, 4] and desc.tolist()[2:] == [1, 2, 3, 5]


def test_top_k_same_answer_on_both_sides_of_the_switch(shim):
    """The host path (<= 4 096 rows) and the select path (> 4 096) give the same keys for the same rows: the extra row is a
    NULL primary, which comes after all of them."""
    rng = np.random.default_rng(9)
    n = 4096
    cols = [_col(rng, "f64", n), _col(rng, "i64", n)]
    for desc in ([True, False], [False, True]):
        small = _run(shim, cols, desc, [None, None], 50, "top_k")
        big_cols = [np.append(c, c[:1]) for c in cols]
        big = _run(shim, big_cols, desc, [np.append(np.ones(n, np.uint8), 0), None], 50, "top_k")
        keys = np.stack(K.order_keys(cols, desc), 1)
        assert np.array_equal(keys[small], keys[big])


# ------------------------------------------------------------------ the DataStream API on the shim
@pytest.fixture
def qc(monkeypatch):
    cpu_shim.install(monkeypatch)
    from quokka_b200.df import QuokkaContext
    return QuokkaContext()


def test_grouped_min_max_over_nan_through_the_api(qc):
    """groupby(int key).agg(min, max, count) with NaN values: the hash aggregate skips NaN; an all-NaN group gives the
    identities.  Before, the shim propagated NaN here while the kernel did not."""
    rng = np.random.default_rng(11)
    n = 6000
    k = K.int_keys(rng, np.int64, n, 60)
    x = K.float_values(rng, n, "dyadic", specials=True)
    x[k == k[0]] = K.NAN_NEG                                             # one group of NaN only
    got = qc.from_arrow(pa.table({"k": k, "x": x})).groupby("k").agg_sql("min(x) as mn, max(x) as mx, count(*) as c") \
        .collect().to_pandas().sort_values("k")
    ref = K.ref_groupby([k], [x, x], ["min", "max"])
    assert np.array_equal(got["k"].to_numpy(), ref["keys"][0])
    assert np.array_equal(got["c"].to_numpy(np.int64), ref["cnt"])
    assert np.array_equal(got["mn"].to_numpy(), ref["vals"][0]) and np.array_equal(got["mx"].to_numpy(), ref["vals"][1])
    g0 = int(np.searchsorted(ref["keys"][0], k[0]))
    assert ref["vals"][0][g0] == math.inf and ref["vals"][1][g0] == -math.inf
