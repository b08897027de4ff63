"""Exact references and seeded generators for the keyed kernels: the hash aggregate (csrc/hashagg.cu), the hash join
(csrc/join.cu) and the top-k select (csrc/topk.cu) with the host ordering after it (executors.sort_table / top_k_table).
numpy only: no torch, no quokka_b200 import, so the CPU suite can check these references against brute-force loops.  The two
executor cases at the end take the executors module from their caller, which runs them on the device or on the CPU shim.

Ordering (DESIGN.md section 2, DuckDB's ORDER BY):
  numbers compare by value and -0.0 = +0.0; every NaN, whichever sign, is greater than +inf (last ASC, first DESC);
  NULL comes after everything in both directions (NULLS LAST); integers are exact over their full range.

Group-by: exact keys and counts; MIN / MAX skip NaN, so a group of NaN values keeps the identity (+inf for MIN, -inf for
MAX); SUM exact on dyadic data and within n_g * 2^-53 * sum|x| of the exact sum otherwise.

Join: integer keys compare by value whatever their width (uint8 zero-extends, int32 sign-extends); fp64 keys compare by bit
pattern after -0.0 is folded into +0.0 (executors._float_key), so a NaN matches the identical NaN and nothing else;
INT64_MIN is reserved (the empty-slot marker): a probe key INT64_MIN matches nothing, a build key INT64_MIN is an error."""
from __future__ import annotations

import math

import numpy as np

I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
I32_MIN, I32_MAX = -(1 << 31), (1 << 31) - 1
NAN_POS = np.array([0x7FF8000000000000], np.uint64).view(np.float64)[0]
NAN_NEG = np.array([0xFFF8000000000000], np.uint64).view(np.float64)[0]      # x86's default NaN (e.g. inf - inf)
NAN_PAYLOAD = np.array([0x7FF0000000000001], np.uint64).view(np.float64)[0]
F32_NAN_NEG = np.array([0xFFC00000], np.uint32).view(np.float32)[0]


# ------------------------------------------------------------------ ordering
def row_key(x, desc: bool, valid: bool = True) -> tuple:
    """The sort key of one value, as a tuple that Python compares in ascending order: the rules above, one value at a
    time.  Integers are Python ints (exact); floats are Python floats (-0.0 == 0.0)."""
    if not valid:
        return (1, 0, 0)
    if isinstance(x, (float, np.floating)) and math.isnan(x):
        return (0, 0, 0) if desc else (0, 1, 0)
    v = int(x) if isinstance(x, (int, np.integer, bool, np.bool_)) else float(x)
    return (0, 1, -v) if desc else (0, 0, v)


def python_order(cols: list, desc: list, valids: list | None = None) -> list:
    """Row indices in ORDER BY order by Python's stable sort over row_key tuples (the spec, O(n log n) in Python)."""
    valids = valids or [None] * len(cols)
    n = len(cols[0])

    def key(i):
        return tuple(row_key(c[i].item() if hasattr(c[i], "item") else c[i], d, True if m is None else bool(m[i]))
                     for c, d, m in zip(cols, desc, valids))
    return sorted(range(n), key=key)


def rank_key(v: np.ndarray, desc: bool, valid: np.ndarray | None = None) -> list:
    """Vectorised form of row_key for one column: [null flag, dense rank] with ascending order = ORDER BY order.  The rank
    comes from np.unique, which compares values (exact for integers, -0.0 == +0.0, NaNs collapsed and last)."""
    u, inv = np.unique(v, return_inverse=True, equal_nan=True) if v.dtype.kind == "f" else np.unique(v, return_inverse=True)
    r = inv.reshape(-1).astype(np.int64)
    if desc:
        r = -r
    null = np.zeros(len(v), np.int64) if valid is None else (np.asarray(valid) == 0).astype(np.int64)
    return [null, np.where(null != 0, 0, r)]


def order_keys(cols: list, desc: list, valids: list | None = None) -> list:
    valids = valids or [None] * len(cols)
    out = []
    for c, d, m in zip(cols, desc, valids):
        out += rank_key(c, d, m)
    return out


def ref_order(cols: list, desc: list, valids: list | None = None, k: int | None = None) -> np.ndarray:
    keys = order_keys(cols, desc, valids)
    o = np.lexsort(keys[::-1]) if len(cols[0]) else np.zeros(0, np.int64)
    return o if k is None else o[:k]


def ref_candidates(v: np.ndarray, k: int, desc: bool) -> np.ndarray:
    """Every row whose primary key is at least as good as the k-th best (all rows when n <= k), ascending row ids."""
    if len(v) <= k:
        return np.arange(len(v))
    r = rank_key(v, desc)[1]
    kth = np.sort(r)[k - 1]
    return np.nonzero(r <= kth)[0]


def check_topk(got_ids: np.ndarray, cols: list, desc: list, valids: list | None, k: int, tag=""):
    """`got_ids` (row ids carried through the ordering as a payload column) against the reference: the same sequence of
    sort keys as the first k reference rows, and distinct rows.  Rows that tie on every sort column may come in any
    order; distinct ids with equal keys cover exactly that freedom (a tie group before the last one is then the whole group)."""
    keys = np.stack(order_keys(cols, desc, valids), 1) if len(cols[0]) else np.zeros((0, 2 * len(cols)), np.int64)
    ref = ref_order(cols, desc, valids, k)
    got_ids = np.asarray(got_ids, np.int64)
    assert len(got_ids) == len(ref), (tag, len(got_ids), len(ref))
    assert len(np.unique(got_ids)) == len(got_ids), (tag, "a row came twice")
    bad = np.nonzero((keys[got_ids] != keys[ref]).any(1))[0]
    assert len(bad) == 0, (tag, "first wrong position", int(bad[0]), got_ids[bad[0]], ref[bad[0]])


# ------------------------------------------------------------------ group-by
def exact_sums(gid: np.ndarray, v: np.ndarray, ng: int) -> np.ndarray:
    """Correctly rounded per-group sums (math.fsum) of finite values."""
    out = np.zeros(ng)
    if len(v) == 0:
        return out
    order = np.argsort(gid, kind="stable")
    bounds = np.searchsorted(gid[order], np.arange(ng + 1))
    sv = v[order]
    for g in range(ng):
        out[g] = math.fsum(sv[bounds[g]:bounds[g + 1]])
    return out


def ref_groupby(keys: list, vals: list, ops: list) -> dict:
    """keys: integer arrays; vals[j] with ops[j] in sum|min|max.  Returns {"keys": [unique arrays, lexicographic order],
    "cnt", "vals": [per aggregate], "abs": [sum |x| per SUM aggregate]} -- the rules in the module docstring."""
    n = len(keys[0])
    if n == 0:
        return {"keys": [k[:0] for k in keys], "cnt": np.zeros(0, np.int64), "vals": [np.zeros(0) for _ in vals],
                "abs": [np.zeros(0) for _ in vals]}
    wide = [k.astype(np.int64) for k in keys]                 # uint8 / bool / int32 / int64 all fit int64 exactly
    order = np.lexsort(wide[::-1])
    new = np.zeros(n, bool)
    new[0] = True
    for k in wide:
        new[1:] |= k[order][1:] != k[order][:-1]
    gid = np.empty(n, np.int64)
    gid[order] = np.cumsum(new) - 1
    ng = int(new.sum())
    out = {"keys": [k[order][new] for k in keys], "cnt": np.bincount(gid, minlength=ng).astype(np.int64), "vals": [], "abs": []}
    for v, op in zip(vals, ops):
        if op == "sum":
            out["vals"].append(exact_sums(gid, v, ng) if np.isfinite(v).all() else np.bincount(gid, weights=v, minlength=ng))
            out["abs"].append(np.bincount(gid, weights=np.abs(v), minlength=ng))
        else:
            acc = np.full(ng, np.inf if op == "min" else -np.inf)
            (np.fmin if op == "min" else np.fmax).at(acc, gid, v)
            out["vals"].append(acc)
            out["abs"].append(np.zeros(ng))
    return out


def check_groupby(got_keys: list, got_vals: list, got_cnt: np.ndarray, ref: dict, ops: list, exact: bool, tag=""):
    """Kernel output (any row order) against ref_groupby: keys and counts bit-exact, MIN / MAX bit-exact (a -0.0 / +0.0
    pair may come either way round: both are the minimum), SUM bit-exact on dyadic data, else within n_g * 2^-53 * sum|x|."""
    wide = [np.asarray(k).astype(np.int64) for k in got_keys]
    order = np.lexsort(wide[::-1]) if len(wide[0]) else np.zeros(0, np.int64)
    assert len(order) == len(ref["cnt"]), (tag, "groups", len(order), len(ref["cnt"]))
    for a, b in zip(got_keys, ref["keys"]):
        assert np.array_equal(np.asarray(a)[order].astype(np.int64), b.astype(np.int64)), (tag, "keys")
    assert np.array_equal(np.asarray(got_cnt)[order], ref["cnt"]), (tag, "counts")
    for j, (g, r, op) in enumerate(zip(got_vals, ref["vals"], ops)):
        g = np.asarray(g)[order]
        if op == "sum" and not exact:
            tol = ref["cnt"] * 2.0 ** -53 * ref["abs"][j]
            fin = np.isfinite(r)
            assert np.array_equal(g[~fin], r[~fin], equal_nan=True), (tag, j, "non-finite sums")
            assert (np.abs(g[fin] - r[fin]) <= tol[fin]).all(), (tag, j, np.max(np.abs(g[fin] - r[fin]) - tol[fin]))
        else:
            assert np.array_equal(g, r, equal_nan=True), (tag, op, j, np.nonzero(~((g == r) | (np.isnan(g) & np.isnan(r))))[0][:5])


# ------------------------------------------------------------------ join
def float_key(a: np.ndarray) -> np.ndarray:
    """executors._float_key in numpy: -0.0 folded into +0.0, then the bits."""
    with np.errstate(invalid="ignore"):                  # a signalling NaN stays a NaN
        return (a.astype(np.float64) + 0.0).view(np.int64)


def join_key(a: np.ndarray) -> np.ndarray:
    return float_key(a) if a.dtype.kind == "f" else a.astype(np.int64)


def ref_join(probe: np.ndarray, build: np.ndarray, how: str):
    """(probe_idx, build_idx | None) in probe-row order, build rows ascending among equal keys; build_idx -1 for an
    unmatched row of a left join.  Keys of any integer width on either side, or fp64 on both."""
    pk, bk = join_key(probe), join_key(build)
    if (bk == I64_MIN).any():
        raise ValueError("INT64_MIN is reserved as a build key")
    order = np.argsort(bk, kind="stable")
    sk = bk[order]
    lo, hi = np.searchsorted(sk, pk, "left"), np.searchsorted(sk, pk, "right")
    cnt = hi - lo
    if how == "semi":
        return np.nonzero(cnt > 0)[0], None
    if how == "anti":
        return np.nonzero(cnt == 0)[0], None
    emit = np.maximum(cnt, 1) if how == "left" else cnt
    total = int(emit.sum())
    pi = np.repeat(np.arange(len(pk)), emit)
    within = np.arange(total) - np.repeat(np.cumsum(emit) - emit, emit)
    bi = np.full(total, -1, np.int64)
    m = np.repeat(cnt > 0, emit)
    bi[m] = order[(np.repeat(lo, emit) + within)[m]]
    return pi, bi


def brute_join(probe, build, how):
    """Nested loops over Python values (floats through float_key): the same result as ref_join, slowly."""
    pk, bk = [int(x) for x in join_key(probe)], [int(x) for x in join_key(build)]
    pi, bi = [], []
    for i, a in enumerate(pk):
        hits = [j for j, b in enumerate(bk) if a == b]
        if how == "semi" and hits or how == "anti" and not hits:
            pi.append(i)
        elif how in ("inner", "left"):
            for j in hits or ([-1] if how == "left" else []):
                pi.append(i)
                bi.append(j)
    return np.array(pi, np.int64), (np.array(bi, np.int64) if how in ("inner", "left") else None)


# ------------------------------------------------------------------ generators
KEY_DTYPES = {"u8": np.uint8, "bool": np.bool_, "i32": np.int32, "i64": np.int64}


def int_keys(rng, dt, n: int, card: int, edges: bool = True) -> np.ndarray:
    """n keys of dtype `dt` drawn from `card` distinct values spread over the dtype's range (negatives included); with
    `edges` the extremes of the type are among the values."""
    dt = np.dtype(dt)
    if dt == np.bool_:
        return rng.integers(0, 2, n).astype(np.bool_)
    if dt == np.uint8:
        pool = rng.permutation(256)[:max(1, min(card, 256))]
        if edges and len(pool) > 2:
            pool[:2] = [0, 255]
        return pool[rng.integers(0, len(pool), n)].astype(np.uint8)
    info = np.iinfo(dt)
    pool = np.unique(rng.integers(info.min, info.max, max(1, card), dtype=np.int64, endpoint=True))
    if edges and len(pool) > 4:
        pool[:4] = [info.min, info.max, -1, 0]
        pool = np.unique(pool)
    return pool[rng.integers(0, len(pool), n)].astype(dt)


def float_values(rng, n: int, kind: str = "dyadic", specials: bool = False) -> np.ndarray:
    """fp64 aggregate inputs: `dyadic` k / 8 with |k| < 2^20 (every partial sum exact), `normal` N(0, 1e4); with
    `specials` about 1 % each of NaN (both signs), +inf, -inf, +0.0, -0.0."""
    v = rng.integers(-(1 << 20), 1 << 20, n) / 8.0 if kind == "dyadic" else rng.normal(size=n) * 1e4
    if specials and n:
        pick = rng.integers(0, 100, n)
        for code, x in enumerate([NAN_POS, NAN_NEG, np.inf, -np.inf, 0.0, -0.0]):
            v[pick == code] = x
    return v


def order_column(rng, dt, n: int, card: int, specials: bool = True) -> np.ndarray:
    """A top-k primary column of `card` distinct values with the edges of its type: ±0 and NaN of both signs, ±inf and
    the integer extremes."""
    dt = np.dtype(dt)
    if dt.kind == "f":
        pool = np.round(rng.normal(size=max(1, card)) * 100, 1)
        if specials and len(pool) > 8:
            pool[:8] = [0.0, -0.0, NAN_POS, NAN_NEG, np.inf, -np.inf, NAN_PAYLOAD, 1.5]
        v = pool[rng.integers(0, len(pool), n)]
        return v.astype(dt) if dt == np.float32 else v
    return int_keys(rng, dt, n, card, edges=specials)


# ------------------------------------------------------------------ the executors that grow the hash aggregate
# (the executors module comes from the caller: on the device, or on the CPU shim)
def count_grows(X, monkeypatch) -> list:
    """Records the incoming row count of every re-insertion into a larger table, whichever executor asks for it."""
    grows = []
    real = X._GrowingHashAgg._grow
    monkeypatch.setattr(X._GrowingHashAgg, "_grow", lambda self, inc: (grows.append(inc), real(self, inc))[1])
    return grows


def case_sql_agg_executor_grow(X, monkeypatch):
    """SQLAggExecutor re-inserts its groups into a larger table when a batch would push the load past 1/2; batches of rising
    cardinality grow it several times.  SUM / MIN / MAX of the re-inserted partials equal one aggregate over all rows."""
    import pyarrow as pa
    rng = np.random.default_rng(5)
    grows = count_grows(X, monkeypatch)
    ex = X.SQLAggExecutor(["k"], None, "SUM(v) AS s, MIN(v) AS mn, MAX(v) AS mx")
    parts = []
    for n, card in zip([1000, 40_000, 100_000, 400_000, 20_000], [300, 20_000, 80_000, 400_000, 500_000]):
        parts.append((rng.integers(-card, card, n).astype(np.int64) * 31, float_values(rng, n, "dyadic", specials=True)))
    for k, v in parts:
        ex.execute([pa.table({"k": k, "v": v})], 0, 0)
    out = ex.done(0).to_numpy()
    assert len(grows) >= 2, grows
    k = np.concatenate([p[0] for p in parts])
    v = np.concatenate([p[1] for p in parts])
    ref = ref_groupby([k], [v] * 3, ["sum", "min", "max"])
    o = np.argsort(out["k"])
    assert np.array_equal(out["k"][o], ref["keys"][0])
    for name, r in zip(("s", "mn", "mx"), ref["vals"]):
        assert np.array_equal(out[name][o], r, equal_nan=True), name


def case_distinct_executor_grow(X, monkeypatch):
    import pyarrow as pa
    rng = np.random.default_rng(6)
    grows = count_grows(X, monkeypatch)
    ex = X.DistinctExecutor(["a", "b"])
    seen = []
    for n, card in zip([2000, 60_000, 200_000, 300_000], [100, 30_000, 150_000, 600_000]):
        a = rng.integers(-card, card, n).astype(np.int64)
        b = rng.integers(-3, 3, n).astype(np.int32)
        seen.append((a, b))
        ex.execute([pa.table({"a": a, "b": b})], 0, 0)
    assert ex._ha.state.capacity > (1 << 16) and len(grows) >= 2, grows      # the table grew
    out = ex.done(0).to_numpy()
    a = np.concatenate([s[0] for s in seen])
    b = np.concatenate([s[1] for s in seen])
    ref = ref_groupby([a, b], [], [])
    o = np.lexsort((out["b"], out["a"]))
    assert np.array_equal(out["a"][o], ref["keys"][0]) and np.array_equal(out["b"][o], ref["keys"][1])
