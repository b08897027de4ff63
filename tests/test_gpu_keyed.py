"""The keyed kernels against exact references (tests/keyed_cases.py): K2 hash aggregate (csrc/hashagg.cu) with the executors
that grow it, K4 / K5 hash join (csrc/join.cu) with gather, K8 top-k select (csrc/topk.cu) with executors.top_k_table.
Integer work is bit-exact; MIN / MAX bit-exact; SUM bit-exact on dyadic data.  No case provokes a fault: the overflow cases
use the kernels' bounded probes and the flags they return."""
import zlib

import numpy as np
import pytest
import torch

import keyed_cases as K

pytestmark = pytest.mark.gpu

OPS = ["sum", "min", "max"]


def _seed(*a) -> int:
    return zlib.crc32(repr(a).encode())


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    return t.cpu().numpy()


@pytest.fixture(scope="module")
def qb():
    from quokka_b200 import _lib, edge, executors, expr, ops
    from quokka_b200.columns import DeviceColumn, DeviceTable
    _lib.lib()
    return type("QB", (), dict(L=_lib, ops=ops, X=executors, edge=edge, E=expr, DC=DeviceColumn, DT=DeviceTable))


# ------------------------------------------------------------------ K2 hash aggregate
def _codes(qb, ops):
    return [{"sum": qb.L.AGG_SUM, "min": qb.L.AGG_MIN, "max": qb.L.AGG_MAX}[o] for o in ops]


def _hash_agg(qb, keys, vals, capacity, batch=None, ops=OPS, max_groups=None):
    st = qb.ops.HashAggState([dev(k[:0]).dtype for k in keys], _codes(qb, ops), capacity, "cuda")
    n = len(keys[0])
    batch = batch or max(n, 1)
    for lo in range(0, n, batch):
        st.update([dev(k[lo:lo + batch]) for k in keys], [dev(v[lo:lo + batch]) for v in vals])
    ok, ov, oc = st.finalize(max_groups)
    return [host(o) for o in ok], [host(o) for o in ov], host(oc)


def _check_agg(qb, keys, v, capacity, batch=None, tag=""):
    ok, ov, oc = _hash_agg(qb, keys, [v] * 3, capacity, batch)
    K.check_groupby(ok, ov, oc, K.ref_groupby(keys, [v] * 3, OPS), OPS, exact=True, tag=tag)


LAYOUTS = [("u8",), ("bool",), ("i32",), ("i64",), ("u8", "i64"), ("i64", "i64"), ("i32", "i32", "i32", "i32"),
           ("u8", "u8", "i32", "i64")]


@pytest.mark.parametrize("mode", ["one", "many", "hot"])
@pytest.mark.parametrize("layout", LAYOUTS)
def test_hash_aggregate_layouts(qb, layout, mode):
    """Every key layout (one word, two words, 128 bits over four int32) with a single group, ~n groups, and one hot key that
    holds half the rows (contention on the count / SUM atomics and the MIN / MAX CAS loop); NaN of both signs, ±inf, ±0."""
    rng = np.random.default_rng(_seed(layout, mode))
    n = 100_003
    card = {"one": 1, "many": n, "hot": 5000}[mode]
    keys = [K.int_keys(rng, K.KEY_DTYPES[d], n, card, edges=mode != "one") for d in layout]
    if mode == "hot":
        hot = rng.random(n) < 0.5
        for k in keys:
            k[hot] = k[0]
    v = K.float_values(rng, n, "dyadic", specials=True)
    _check_agg(qb, keys, v, 2 * n, batch=30_001, tag=(layout, mode))


def test_hash_aggregate_all_rows_distinct_with_int64_extremes(qb):
    rng = np.random.default_rng(1)
    n = 300_000
    k = np.unique(rng.integers(K.I64_MIN + 1, K.I64_MAX, n + 1000, dtype=np.int64))[:n - 4]
    k = rng.permutation(np.concatenate([[K.I64_MIN, K.I64_MAX, -1, 0], k[(k != -1) & (k != 0)]]))
    v = K.float_values(rng, n, "normal", specials=True)
    _check_agg(qb, [k.astype(np.int64)], v, 2 * n)


def test_hash_aggregate_negative_int32_packed_next_to_other_fields(qb):
    """An int32 key is stored zero-extended inside its word: a negative one must not spill into the field above it."""
    rng = np.random.default_rng(2)
    n = 50_000
    a = rng.integers(-3, 3, n).astype(np.int32)                    # many -1 / -2 / -3: sign-extended they cover bits 32..63
    b = rng.integers(K.I32_MIN, K.I32_MIN + 4, n).astype(np.int32)
    c = rng.integers(-5, 5, n).astype(np.int32)
    d = rng.integers(0, 3, n).astype(np.uint8)
    v = K.float_values(rng, n)
    _check_agg(qb, [a, b], v, 2 * n, tag="i32,i32")
    _check_agg(qb, [a, d, c, d], v, 2 * n, tag="i32,u8,i32,u8")
    _check_agg(qb, [d, a, b, c], v, 2 * n, tag="u8,i32,i32,i32")


@pytest.mark.parametrize("layout", ["i64,i64", "i32x4"])
def test_hash_aggregate_keys_differing_only_in_word_1(qb, layout):
    """Keys equal in the first packed word: groups = capacity / 2 of them, so probe chains cross each other's slots."""
    rng = np.random.default_rng(3)
    cap, m = 1 << 14, 1 << 13
    w1 = rng.permutation(m).astype(np.int64) * 104729 - 7
    idx = rng.integers(0, m, 4 * m)
    if layout == "i64,i64":
        keys = [np.full(4 * m, -1, np.int64), w1[idx]]
    else:
        keys = [np.full(4 * m, -1, np.int32), np.full(4 * m, 5, np.int32), (w1[idx] & 0x7fff).astype(np.int32) - 9,
                (w1[idx] >> 15).astype(np.int32)]
    v = K.float_values(rng, 4 * m, specials=True)
    _check_agg(qb, keys, v, cap, batch=7777, tag=layout)


@pytest.mark.parametrize("fill", ["half", "full"])
def test_hash_aggregate_table_load(qb, fill):
    rng = np.random.default_rng(4)
    cap = 4096
    g = cap // 2 if fill == "half" else cap
    k = np.repeat(rng.permutation(np.arange(g, dtype=np.int64) * 65_537 - 1_000_000), 3)
    k = k[rng.permutation(len(k))]
    v = K.float_values(rng, len(k), specials=True)
    _check_agg(qb, [k], v, cap, batch=5000, tag=fill)


def test_hash_aggregate_overflow_raises(qb):
    """capacity + 1 distinct keys: the bounded probe of the last one finds no slot, the overflow flag is raised and
    finalize reports it instead of returning a short result."""
    cap = 4096
    k = np.arange(cap + 1, dtype=np.int64) * 3
    with pytest.raises(qb.L.QkError, match="overflowed"):
        _hash_agg(qb, [k], [np.ones(len(k))], cap, ops=["sum"])


def test_hash_aggregate_rejects_keys_over_128_bits(qb):
    for dts in ([torch.int64, torch.int64, torch.uint8], [torch.int32, torch.int64, torch.int64]):
        with pytest.raises(qb.L.QkError):
            qb.ops.HashAggState(dts, [qb.L.AGG_SUM], 1024, "cuda")


def test_hash_aggregate_column_counts_must_match_the_state(qb):
    st = qb.ops.HashAggState([torch.int64], [qb.L.AGG_SUM, qb.L.AGG_MIN], 64, "cuda")
    k, v = dev(np.arange(8, dtype=np.int64)), dev(np.ones(8))
    for keys, vals in (([k], [v]), ([k, k], [v, v]), ([], [v, v])):
        with pytest.raises(qb.L.QkError, match="columns for a state"):
            st.update(keys, vals)


def test_hash_aggregate_finalize_too_small_raises(qb):
    k = np.arange(100, dtype=np.int64)
    with pytest.raises(qb.L.QkError, match="sized for"):
        _hash_agg(qb, [k], [np.ones(100)], 1024, ops=["sum"], max_groups=99)
    ok, _, oc = _hash_agg(qb, [k], [np.ones(100)], 1024, ops=["sum"], max_groups=100)
    assert sorted(ok[0].tolist()) == k.tolist() and (oc == 1).all()


def test_hash_aggregate_empty_and_single_row(qb):
    _check_agg(qb, [np.zeros(0, np.int64)], np.zeros(0), 16)
    _check_agg(qb, [np.array([K.I64_MIN])], np.array([K.NAN_NEG]), 16)


def test_sql_agg_executor_grow(qb, monkeypatch): K.case_sql_agg_executor_grow(qb.X, monkeypatch)


def test_distinct_executor_grow(qb, monkeypatch): K.case_distinct_executor_grow(qb.X, monkeypatch)


def test_dense_and_hash_paths_agree(qb, monkeypatch):
    """The same MIN / MAX / COUNT grouping on a dictionary column, once through the dense kernel and once through the hash
    aggregate: the same groups, counts and values (NaN skipped by both; a ±0 pair may resolve either way in either)."""
    rng = np.random.default_rng(7)
    n = 200_003
    names = [f"g{i:02d}" for i in range(40)]
    codes = rng.integers(0, 40, n).astype(np.uint8)
    x = K.float_values(rng, n, "normal", specials=True)
    x[codes == 3] = K.NAN_NEG
    t = qb.DT({"k": qb.DC(dev(codes), names), "x": qb.DC(dev(x))})
    agg = qb.edge.PartialAgg(["k"], [("min", qb.E.col("x"), "mn"), ("max", qb.E.col("x"), "mx"), ("count", None, "c")])
    runs = []
    for force_hash in (False, True):
        if force_hash:
            monkeypatch.setattr(qb.edge, "dense_agg_fits", lambda *a: False)
            monkeypatch.setattr(qb.edge, "world_size", lambda: 2)
        out = agg(t).to_numpy()
        runs.append((agg.last_path, out))
    assert runs[0][0] != "hash" and runs[1][0] == "hash", [r[0] for r in runs]
    ref = K.ref_groupby([codes], [x, x], ["min", "max"])
    for path, out in runs:
        o = np.argsort(out["k"])
        assert np.array_equal(out["k"][o], ref["keys"][0]) and np.array_equal(out["c"][o], ref["cnt"]), path
        assert np.array_equal(out["mn"][o], ref["vals"][0]) and np.array_equal(out["mx"][o], ref["vals"][1]), path


# ------------------------------------------------------------------ K4 / K5 join
HOWS = ["inner", "left", "semi", "anti"]
_RANGE = {"u8": (0, 255), "i32": (K.I32_MIN, K.I32_MAX), "i64": (K.I64_MIN + 1, K.I64_MAX)}
_NP = {"u8": np.uint8, "i32": np.int32, "i64": np.int64}


def _join_keys(rng, pdt, bdt, n_probe, n_build):
    """Keys that overlap across the two widths: 70 % from a pool both dtypes hold, the rest from each side's own range
    (negatives and the extremes included)."""
    lo = max(_RANGE[pdt][0], _RANGE[bdt][0])
    hi = min(_RANGE[pdt][1], _RANGE[bdt][1])
    common = np.unique(rng.integers(lo, hi, 400, dtype=np.int64, endpoint=True))

    def side(dt, n):
        own = rng.integers(*_RANGE[dt], n, dtype=np.int64, endpoint=True)
        own[:4] = [_RANGE[dt][0], _RANGE[dt][1], 0, _RANGE[dt][0] + 1][:min(n, 4)]
        return np.where(rng.random(n) < 0.7, common[rng.integers(0, len(common), n)], own).astype(_NP[dt])
    return side(pdt, n_probe), side(bdt, n_build)


def _probe(qb, probe, build_parts, how, capacity_rows=None):
    t = qb.ops.JoinTable(capacity_rows if capacity_rows is not None else sum(len(b) for b in build_parts), "cuda")
    for b in build_parts:
        t.build(dev(b))
    code = {"inner": qb.L.JOIN_INNER, "left": qb.L.JOIN_LEFT, "semi": qb.L.JOIN_SEMI, "anti": qb.L.JOIN_ANTI}[how]
    pi, bi = t.probe(dev(probe), code)
    t.check_flags()
    return host(pi).astype(np.int64), None if bi is None else host(bi).astype(np.int64)


def _check_join(got, ref, tag=""):
    (pi, bi), (rp, rb) = got, ref
    if rb is None:
        assert bi is None and np.array_equal(np.sort(pi), rp), tag
        return
    o = np.lexsort((bi, pi))
    assert len(pi) == len(rp), (tag, len(pi), len(rp))
    assert np.array_equal(pi[o], rp) and np.array_equal(bi[o], rb), tag


@pytest.mark.parametrize("how", HOWS)
@pytest.mark.parametrize("pdt,bdt", [("u8", "u8"), ("i32", "i32"), ("i64", "i64"), ("u8", "i32"), ("i32", "u8"), ("i32", "i64"),
                                     ("i64", "i32"), ("u8", "i64"), ("i64", "u8")])
def test_join_key_dtypes(qb, pdt, bdt, how):
    """Key widths on each side, mixed pairs, negatives and extremes; the build fed in batches (row_base); probe sizes that
    are not multiples of 32.  The (probe, build) pairs are compared bit-exact."""
    rng = np.random.default_rng(_seed(pdt, bdt, how))
    for n_probe, n_build in ((1, 1), (31, 40), (33, 1000), (10_007, 3001)):
        probe, build = _join_keys(rng, pdt, bdt, n_probe, n_build)
        if pdt == "i64" and n_probe > 4:
            probe[3] = K.I64_MIN                                   # matches nothing: emitted by left / anti joins only
        cuts = [0, n_build // 3, n_build // 3 + 1, n_build]
        got = _probe(qb, probe, [build[a:b] for a, b in zip(cuts[:-1], cuts[1:])], how)
        _check_join(got, K.ref_join(probe, build, how), tag=(pdt, bdt, how, n_probe))


def test_join_int64_min_probe_key(qb):
    probe = np.array([K.I64_MIN, 5, K.I64_MIN, K.I64_MAX], np.int64)
    build = np.array([5, K.I64_MAX, 5], np.int64)
    for how in HOWS:
        _check_join(_probe(qb, probe, [build], how), K.ref_join(probe, build, how), tag=how)
    assert _probe(qb, probe, [build], "anti")[0].tolist() == [0, 2]


def test_join_int64_min_build_key_raises(qb):
    t = qb.ops.JoinTable(4, "cuda")
    t.build(dev(np.array([1, K.I64_MIN, 3], np.int64)))
    with pytest.raises(qb.L.QkError, match="reserved"):
        t.check_flags()


@pytest.mark.parametrize("how", HOWS)
def test_join_float_keys(qb, how):
    """fp64 keys through executors._float_key: -0.0 matches +0.0, ±inf match themselves, a NaN matches the identical NaN."""
    rng = np.random.default_rng(8)
    pool = np.array([0.0, -0.0, np.inf, -np.inf, K.NAN_POS, 1.5, -1.5, 1e300, 5e-324, 0.1])
    probe = pool[rng.integers(0, len(pool), 5003)]
    build = np.concatenate([pool[[0, 2, 3, 4, 5, 9]], pool[rng.integers(0, len(pool), 700)]])
    t = qb.ops.JoinTable(len(build), "cuda")
    t.build(qb.X._float_key(dev(build)))
    code = {"inner": qb.L.JOIN_INNER, "left": qb.L.JOIN_LEFT, "semi": qb.L.JOIN_SEMI, "anti": qb.L.JOIN_ANTI}[how]
    pi, bi = t.probe(qb.X._float_key(dev(probe)), code)
    got = (host(pi).astype(np.int64), None if bi is None else host(bi).astype(np.int64))
    _check_join(got, K.ref_join(probe, build, how), tag=how)


@pytest.mark.parametrize("how", ["inner", "left"])
def test_join_heavy_duplication_takes_the_retry(qb, how):
    """One key 4 096 times on the build side and 2 048 times on the probe side: 8 M pairs overflow the first output buffer
    (sized for the probe rows), and the probe runs again at the exact size."""
    rng = np.random.default_rng(9)
    build = np.concatenate([np.full(4096, 42, np.int64), rng.integers(-1000, 1000, 3000)])[rng.permutation(7096)]
    probe = np.concatenate([np.full(2048, 42, np.int64), rng.integers(-1000, 1000, 2001)])[rng.permutation(4049)]
    got = _probe(qb, probe, [build[:3000], build[3000:]], how)
    assert len(got[0]) > 8_000_000
    _check_join(got, K.ref_join(probe, build, how), tag=how)


@pytest.mark.parametrize("how", HOWS)
def test_join_empty_sides(qb, how):
    keys = np.array([1, 2, 3], np.int64)
    empty = np.zeros(0, np.int64)
    _check_join(_probe(qb, keys, [], how, capacity_rows=0), K.ref_join(keys, empty, how), tag="no build")
    _check_join(_probe(qb, keys, [empty], how), K.ref_join(keys, empty, how), tag="empty build")
    _check_join(_probe(qb, empty, [keys], how), K.ref_join(empty, keys, how), tag="empty probe")


def test_gather_every_dtype(qb):
    rng = np.random.default_rng(10)
    n = 1000
    srcs = [rng.integers(0, 256, n).astype(np.uint8), rng.integers(0, 2, n).astype(np.bool_),
            rng.integers(K.I32_MIN, K.I32_MAX, n).astype(np.int32), rng.integers(K.I64_MIN, K.I64_MAX, n, dtype=np.int64),
            rng.normal(size=n).astype(np.float32), K.float_values(rng, n, "normal", specials=True)]
    idx = rng.integers(-1, n, 4099).astype(np.int32)
    idx[:3] = [-1, n - 1, 0]
    outs = qb.ops.gather([dev(s) for s in srcs], dev(idx))
    for s, o in zip(srcs, outs):
        want = np.where(idx >= 0, s[np.maximum(idx, 0)], np.zeros(1, s.dtype))
        assert host(o).dtype == s.dtype
        assert np.array_equal(host(o).view(np.uint8), want.view(np.uint8)), s.dtype      # bit-exact, NaN payloads included


# ------------------------------------------------------------------ K8 top-k
DTYPES = {"u8": np.uint8, "bool": np.bool_, "i32": np.int32, "i64": np.int64, "f32": np.float32, "f64": np.float64}


def _cands(qb, v, k, desc):
    return np.sort(host(qb.ops.topk_candidates(dev(v), k, desc)).astype(np.int64))


@pytest.mark.parametrize("desc", [False, True])
@pytest.mark.parametrize("n", [4096, 4097, 100_003])
@pytest.mark.parametrize("dt", list(DTYPES))
def test_topk_candidates_match_reference(qb, dt, n, desc):
    """The candidates are exactly the rows at least as good as the k-th best: ties at the cut, ±0 and NaN of both signs at
    and next to the cut, ±inf, the integer extremes."""
    rng = np.random.default_rng(_seed(dt, n, desc))
    for card in (50, n):
        v = K.order_column(rng, DTYPES[dt], n, card)
        for k in (1, 7, n // 2, n - 1, n, n + 1):
            assert np.array_equal(_cands(qb, v, k, desc), K.ref_candidates(v, k, desc)), (dt, n, desc, card, k)


@pytest.mark.parametrize("dt", ["f64", "i64", "f32", "i32"])
def test_topk_candidates_10m(qb, dt):
    rng = np.random.default_rng(11)
    n = 10_000_000
    v = K.order_column(rng, DTYPES[dt], n, 1_000_000)
    for desc, k in ((True, 1000), (False, 1), (True, n - 1)):
        assert np.array_equal(_cands(qb, v, k, desc), K.ref_candidates(v, k, desc)), (dt, desc, k)


def test_topk_candidates_edges_at_the_cut(qb):
    n = 5000
    rng = np.random.default_rng(12)
    signed_zero = np.where(rng.random(n) < 0.5, -0.0, 0.0)              # all equal: -0.0 = +0.0
    for v in (np.full(n, 3.0), signed_zero, signed_zero.astype(np.float32), np.full(n, K.I64_MIN, np.int64),
              np.full(n, K.NAN_NEG), np.full(n, 255, np.uint8)):
        for desc in (False, True):
            for k in (1, n - 1):
                assert np.array_equal(_cands(qb, v, k, desc), np.arange(n)), (v.dtype, desc, k)
    # the k-th best is 0, with -0.0 and +0.0 rows on both sides of the cut
    v = np.concatenate([np.arange(1, 11, dtype=np.float64), np.full(20, -0.0), np.full(20, 0.0), -np.arange(1, 4951.0)])
    v = v[rng.permutation(n)]
    assert len(_cands(qb, v, 15, True)) == 50
    assert np.array_equal(_cands(qb, v, 15, True), K.ref_candidates(v, 15, True))
    # two NaN rows: first in DESC order, last in ASC order, whatever their sign
    for nan in (K.NAN_POS, K.NAN_NEG, K.NAN_PAYLOAD):
        w = rng.normal(size=n)
        w[[17, 4000]] = [nan, K.NAN_NEG]
        assert set(_cands(qb, w, 2, True).tolist()) == {17, 4000}
        assert not {17, 4000} & set(_cands(qb, w, 10, False).tolist())
        assert np.array_equal(_cands(qb, w, 10, True), K.ref_candidates(w, 10, True))
        f = w.astype(np.float32)
        f[17] = K.F32_NAN_NEG
        assert not {17, 4000} & set(_cands(qb, f, 10, False).tolist())


def _table(qb, cols, valids):
    d = {f"c{j}": qb.DC(dev(c), valid=None if m is None else dev(m)) for j, (c, m) in enumerate(zip(cols, valids))}
    d["id"] = qb.DC(torch.arange(len(cols[0]), dtype=torch.int64, device="cuda"))
    return qb.DT(d)


def _top_k(qb, cols, desc, valids, k):
    out = qb.X.top_k_table(_table(qb, cols, valids), [f"c{j}" for j in range(len(cols))], desc, k)
    ids = host(out["id"].data)
    K.check_topk(ids, cols, desc, valids, k, tag=(desc, k, len(cols[0])))
    for j, c in enumerate(cols):
        assert np.array_equal(host(out[f"c{j}"].data).view(np.uint8), c[ids].view(np.uint8))
    return ids


@pytest.mark.parametrize("nulls", [False, True])
@pytest.mark.parametrize("n", [4096, 4097, 200_003])
@pytest.mark.parametrize("dt", list(DTYPES))
def test_top_k_table_matches_reference(qb, dt, n, nulls):
    """top_k_table: the select on the primary column, then the host ordering on all columns, against the reference key
    sequence; the secondary column decides ties on the primary (±0 and NaN ties included); NULL primaries come last."""
    rng = np.random.default_rng(_seed(dt, n, nulls))
    cols = [K.order_column(rng, DTYPES[dt], n, 40), K.order_column(rng, np.float64, n, 30), K.order_column(rng, np.int64, n, n)]
    valids = [(rng.random(n) > 0.4).astype(np.uint8) if nulls else None, None, None]
    for desc in ([True, False, True], [False, True, False], [True, True, True]):
        for k in (1, 100, n - 1, n, n + 1):
            _top_k(qb, cols, desc, valids, k)


def test_top_k_table_signed_zero_cut_decided_by_second_column(qb):
    """top_k(["x", "y"], k, [DESC, ASC]) where the k-th x is 0: rows with x = -0.0 are candidates and y decides among them."""
    rng = np.random.default_rng(13)
    n = 6000
    x = np.concatenate([np.arange(1, 6, dtype=np.float64), np.full(50, -0.0), np.full(50, 0.0), -np.arange(1, n - 104.0)])
    y = rng.permutation(n).astype(np.int64)
    y[5:55] = np.arange(50)                                             # the best y of the zero rows are all on -0.0 rows
    y[55:105] = 1000 + np.arange(50)
    o = rng.permutation(n)
    x, y = x[o], y[o]
    ids = _top_k(qb, [x, y], [True, False], [None, None], 30)
    assert sorted(y[ids][5:].tolist()) == list(range(25))


def test_top_k_table_nan_and_nulls(qb):
    rng = np.random.default_rng(14)
    n = 5000
    x = rng.normal(size=n)
    x[[3, 4000]] = [K.NAN_POS, K.NAN_NEG]
    ids = _top_k(qb, [x], [True], [None], 10)                           # NaN first in DESC
    assert sorted(ids[:2].tolist()) == [3, 4000]
    ids = _top_k(qb, [x], [False], [None], n)                           # NaN last in ASC
    assert sorted(ids[-2:].tolist()) == [3, 4000]
    m = np.ones(n, np.uint8)
    m[rng.permutation(n)[:4990]] = 0
    xz = np.where(m == 1, x, 0.0)                                       # a left join's unmatched rows: value 0, valid 0
    ids = _top_k(qb, [xz, rng.permutation(n).astype(np.int64)], [True, False], [m, None], 20)
    assert (m[ids[:10]] == 1).all() and (m[ids[10:]] == 0).all()


def test_top_k_same_answer_on_both_sides_of_the_switch(qb):
    """The same rows through the host ordering (4 096 rows) and through the select (4 097 rows, the extra one a NULL
    primary that comes last) give the same key sequence."""
    rng = np.random.default_rng(15)
    n = 4096
    for dt in DTYPES:
        cols = [K.order_column(rng, DTYPES[dt], n, 30), K.order_column(rng, np.float64, n, 20)]
        for desc in ([True, False], [False, True]):
            for k in (1, 64, 4096):
                small = _top_k(qb, cols, desc, [None, None], k)
                big = _top_k(qb, [np.append(c, c[:1]) for c in cols], desc, [np.append(np.ones(n, np.uint8), 0), None], k)
                keys = np.stack(K.order_keys(cols, desc), 1)
                assert np.array_equal(keys[small], keys[big]), (dt, desc, k)
