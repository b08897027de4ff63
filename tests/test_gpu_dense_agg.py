"""Every device path of qk_scan_filter_agg_dense (csrc/scan.cu) against the exact reference of tests/dense_agg_cases.py:
the typed plans q1 / rev1 / mul1 (TMA kernel, variant 3, in each shape of its fallback chain), the runtime-described plan
(variant 7) in each of its six (threads x rows) shapes with its typed tile walk (config ends in "t") and its generic per-row walk, and
the postfix interpreter (variant 1).  After every call the test asserts which kernel, shape and walk ran.

On dyadic data every path matches the reference bit for bit, SUMs included; on TPC-H data SUMs are within
n_g * 2^-53 * sum|x| of the exact sum.  MIN / MAX follow `agg_combine` (fmin / fmax): a NaN value is skipped, a group
without rows keeps the identity (+inf for MIN, -inf for MAX), ±0 compare equal.

QK_DENSE_AGG_REPORT=<path> writes the distinct (last_variant, last_variant_config) pairs the module reached."""
import functools
import os
import re

import numpy as np
import pytest
import torch

import dense_agg_cases as D

pytestmark = pytest.mark.gpu

REACHED = set()
CFG = re.compile(r"nt(\d+)v(\d+)s3c(\d+)(t?)x(\d+)$")


@pytest.fixture(scope="module")
def qk():
    from quokka_b200 import _lib, ops
    _lib.lib()
    yield ops
    path = os.environ.get("QK_DENSE_AGG_REPORT")
    if path:
        with open(path, "w") as f:
            f.write("\n".join(f"{v}\t{c}" for v, c in sorted(REACHED)) + "\n")


@functools.lru_cache(maxsize=3)
def data(n, seed, mode="dyadic"):
    d = D.make_data(n, seed, mode)
    return d, {k: torch.from_numpy(v).cuda() for k, v in d.items()}


def run(qk, plan, d, dd, variant, state=None):
    """one update() of a fresh (or the given) state; returns (state, last_variant, last_variant_config)"""
    names, pred, gslots, progs = D.compile_plan(plan, d)
    st = state or qk.DenseAggState(plan.cards, plan.agg_ops, "cuda")
    st.update([dd[c] for c in names], pred, gslots, progs, variant=variant)
    v, cfg = qk.last_variant(), qk.last_variant_config()
    REACHED.add((v, cfg))
    return st, v, cfg


def host(st):
    return st.acc.cpu().numpy(), st.cnt.cpu().numpy()


def run_and_check(qk, plan, d, dd, variant, exact, tag=""):
    n = len(next(iter(d.values())))
    before = (qk.last_variant(), qk.last_variant_config())
    st, v, cfg = run(qk, plan, d, dd, variant)
    acc, cnt = host(st)
    if n == 0:                             # no rows: nothing is launched, the state stays zero
        assert (v, cfg) == before and not acc.any() and not cnt.any()
        return v, cfg
    D.check(plan, acc, cnt, D.reference(plan, d), exact, tag=f"{tag} variant {variant} n {n} ({v} {cfg})")
    return v, cfg


def assert_dyn(v, cfg, shape=None, fast=None, ncols=None):
    assert v == "fused_tma:dyn", (v, cfg)
    m = CFG.match(cfg)
    assert m, cfg
    if shape is not None:
        assert (int(m[1]), int(m[2])) == shape, (cfg, shape)
    if fast is not None:
        assert (m[4] == "t") == fast, (cfg, fast)
    if ncols is not None:
        assert int(m[3]) == ncols, (cfg, ncols)
    return m


# ------------------------------------------------------------------ the runtime-described plan: six shapes x two walks x sizes
def shape_plan(fast, mode="dyadic"):
    """4 terms (int32 range, fp64 compare, code set, column pair), two keys (one int32 or int64), a shared product prefix,
    a MIN and a CASE-gated SUM.  Fits every shape: 8 columns, 8 or 6 groups, 4 aggregates."""
    key2 = ("k32", 4) if fast else ("k64", 3)
    a = [D.f_col("fa"), D.f_kminus(0.5, "fb")]
    dy = mode == "dyadic"
    terms = [D.irange("i32a", "<", 600 if dy else D.G.DAY_1995_06_17), D.fcmp("fb", ">=", -12.0 if dy else 0.02),
             D.inset("u8", [1, 3, 5, 64, 70, 200]).negate(), D.colcol("i32a", "!=", "i32b")]
    return D.Plan(terms, [("k8b", 2), key2],
                  [D.Agg("sum", a), D.Agg("sum", a + [D.f_kplus(1.0, "fc")]), D.Agg("min", a),
                   D.Agg("sum", [D.f_col("fa")], D.inset("u8", [0, 2, 4, 6, 8]))])


def sizes(tile):
    return [0, 1, tile - 1, tile, tile + 1, 37 * tile + 5, 3_000_017]


@pytest.mark.parametrize("fast", [True, False], ids=["typed_walk", "row_walk"])
@pytest.mark.parametrize("shape", D.DYN_SHAPES, ids=[f"{a}x{b}" for a, b in D.DYN_SHAPES])
def test_dyn_shapes_and_sizes(qk, monkeypatch, shape, fast):
    """Each pinned shape at n = 0, 1, TILE-1, TILE, TILE+1, fewer full tiles than CTAs, and 3 000 017 rows (many tiles per
    CTA and a ragged tail for CTA 0); variant 7 and the interpreter, both bit-exact on dyadic data."""
    monkeypatch.setenv("QK_DYN_SHAPE", f"{shape[0]}x{shape[1]}")
    plan = shape_plan(fast)
    for n in sizes(shape[0] * shape[1]):
        d, dd = data(n, n + 11)
        v, cfg = run_and_check(qk, plan, d, dd, 7, True, f"shape {shape}")
        if n:
            assert_dyn(v, cfg, shape, fast, len(plan.columns))
        v, cfg = run_and_check(qk, plan, d, dd, 1, True)
        if n:
            assert (v, cfg) == ("generic", "nt256")


@pytest.mark.parametrize("fast", [True, False], ids=["typed_walk", "row_walk"])
def test_dyn_tpch_data(qk, fast):
    """The same plan on TPC-H measures: SUMs within n_g * 2^-53 * sum|x|, counts and MIN exact."""
    plan = shape_plan(fast, "tpch")
    for n in (100_003, 3_000_017):
        d, dd = data(n, 5, "tpch")
        assert_dyn(*run_and_check(qk, plan, d, dd, 7, False), fast=fast)
        assert run_and_check(qk, plan, d, dd, 1, False)[0] == "generic"


# ------------------------------------------------------------------ typed plans
def typed_plan(name, mode, pred_hi=500):
    k = (0.5, 1.5, 2.0) if mode == "dyadic" else (1.0, 1.0, 1.0)
    hi = pred_hi if mode == "dyadic" else D.G.DAY_1998_09_02
    pred = [D.irange("i32a", "<=", hi)]
    if name == "q1":
        aggs = [[D.f_col("fd")], [D.f_col("fa")], [D.f_col("fa"), D.f_kminus(k[0], "fb")],
                [D.f_col("fa"), D.f_kminus(k[1], "fb"), D.f_kplus(k[2], "fc")], [D.f_col("fb")]]
        return D.Plan(pred, [("k8a", 3), ("k8b", 2)], [D.Agg("sum", a) for a in aggs])
    if name == "rev1":
        return D.Plan(pred, [("k8a", 3)], [D.Agg("sum", [D.f_col("fa"), D.f_kminus(k[0], "fb")])])
    return D.Plan(pred, [("k8a", 3)], [D.Agg("sum", [D.f_col("fa"), D.f_col("fb")])])


TYPED_CFG = {0: "nt256v4s3", 3: "nt256v4s3"}


@pytest.mark.parametrize("mode", ["dyadic", "tpch"])
@pytest.mark.parametrize("variant", [0, 3])
@pytest.mark.parametrize("name", ["q1", "rev1", "mul1"])
def test_typed_plans(qk, name, variant, mode):
    plan = typed_plan(name, mode)
    for n in (0, 1, 511, 512, 513, 1023, 1024, 1025, 60 * 1024 + 3, 3_000_017):
        if mode == "tpch" and n not in (0, 1, 1025, 60 * 1024 + 3, 3_000_017):
            continue
        d, dd = data(n, n + 3, mode)
        v, cfg = run_and_check(qk, plan, d, dd, variant, mode == "dyadic", name)
        if n:
            assert (v, cfg) == ("fused_tma:" + name, TYPED_CFG[variant])


def test_int32_bound_beyond_int32_is_clamped(qk):
    """`i32a < 2^32 + 5` holds for every int32: the typed plans and the typed tile walk compare in 32 bits, so int_range
    (csrc/common.cuh) must clamp the bound to INT32_MAX, not truncate it."""
    d, dd = data(50_003, 9)
    for k in ((1 << 32) + 5, -(1 << 32) + 5, D.I32_MAX + 1, D.I32_MIN):
        for cmp in D.CMPS:
            plan = typed_plan("mul1", "dyadic")
            plan.terms = [D.irange("i32a", cmp, k)]
            for variant in (3, 1):
                run_and_check(qk, plan, d, dd, variant, True, f"i32a {cmp} {k}")
            plan.aggs.append(D.Agg("min", [D.f_kplus(20.0, "fa")]))           # not a typed plan: the dyn plan, typed walk
            assert_dyn(*run_and_check(qk, plan, d, dd, 7, True, f"i32a {cmp} {k}"), fast=True)


# 256 threads x V rows x 3 stages of Q1's 38 B rows plus 256 lane-private copies of 5 SUMs and a count per group must fit
# 227 KB (csrc/scan.cu launch_tma)
Q1_ROW_BYTES, Q1_GROUP_BYTES = 38, 5 * 8 + 4


def typed_q1_max_groups(v):
    return (D.SMEM_CAP - 3 * Q1_ROW_BYTES * 256 * v) // (Q1_GROUP_BYTES * 256)


@pytest.mark.parametrize("v", [4, 2, 1])
def test_typed_q1_largest_grouping_per_shape(qk, v):
    """The typed Q1 plan at the largest group count each shape of its fallback chain (256 threads x 4, 2, 1 rows) holds
    runs in that shape; one group more takes the next shape, and after the last one the runtime-described plan."""
    ng = typed_q1_max_groups(v)
    assert ng == {4: 10, 2: 15, 1: 18}[v]
    n = 60_011
    rng = np.random.default_rng(100 + v)
    for groups, want in ((ng, ("fused_tma:q1", f"nt256v{v}s3")),
                         (ng + 1, ("fused_tma:q1", f"nt256v{v // 2}s3") if v > 1 else ("fused_tma:dyn", None))):
        cards = next(((groups // p, p) for p in (3, 2) if groups % p == 0), (groups, 1))
        d = {"i32a": rng.integers(-1000, 1000, n).astype(np.int32),
             "q0": rng.integers(0, cards[0], n).astype(np.uint8), "q1": rng.integers(0, cards[1], n).astype(np.uint8)}
        for c in ("fa", "fb", "fc", "fd"):
            d[c] = D.dyadic(rng, n)
        dd = {k: torch.from_numpy(x).cuda() for k, x in d.items()}
        plan = typed_plan("q1", "dyadic")
        plan.keys = [("q0", cards[0]), ("q1", cards[1])]
        v_, cfg = run_and_check(qk, plan, d, dd, 0, True, f"ng {groups}")
        assert v_ == want[0] and (want[1] is None or cfg == want[1]), (groups, v_, cfg)


# ------------------------------------------------------------------ targeted edges of the grammar, both walks
EDGE_N = 10_007


@functools.lru_cache(maxsize=1)
def edge_data():
    """make_data plus `fe`: fp64 with the constant 0.5 and its nextafter neighbours, ±0, NaN, ±inf and ±5e-324 in 30 % of
    the rows; `fp`: strictly positive dyadic values"""
    d = dict(D.make_data(EDGE_N, 77))
    rng = np.random.default_rng(78)
    special = np.array([0.5, np.nextafter(0.5, 1), np.nextafter(0.5, 0), 0.0, -0.0, np.nan, np.inf, -np.inf, 5e-324, -5e-324])
    fe = D.dyadic(rng, EDGE_N)
    at = rng.random(EDGE_N) < 0.3
    fe[at] = special[rng.integers(0, len(special), int(at.sum()))]
    d["fe"] = fe
    d["fp"] = np.abs(D.dyadic(rng, EDGE_N)) + 1.0
    return d, {k: torch.from_numpy(v).cuda() for k, v in d.items()}


def edge_terms(fast):
    t = [D.fcmp("fe", op, c) for op in D.CMPS for c in (0.5, 0.0, -0.0, np.inf, -np.inf, 5e-324, -5e-324)]
    t += [D.irange("i32a", op, k) for op in D.CMPS for k in (D.I32_MIN - 5, D.I32_MAX + 5, (1 << 32) + 5, -(1 << 32) - 5, 7)]
    t += [D.irange("i64a", op, k) for op in D.CMPS for k in (D.I64_MIN, D.I64_MAX, D.I64_MIN + 1, D.I64_MAX - 1)]
    t += [D.between("i32a", 9, 3), D.between("i64a", 9, 3), D.between("i32a", -5, 5)]
    t += [D.inset("u8", [1, 3, 5]), D.inset("u8", [0, 7, 63]), D.inset("u8", [2, 64]), D.inset("u8", list(range(0, 200, 3)))]
    t += [D.colcol("i32a", op, "i32b") for op in D.CMPS] + [D.colcol("i64a", op, "i64b") for op in D.CMPS]
    if not fast:
        t += [D.inset("c32", [1, 3, 5]), D.inset("c32", [0, 7, 63]), D.inset("c32", [2, 64]), D.irange("u8", "<", 300),
              D.irange("u8", ">", -3), D.fcmp("g32", "<", 0.5), D.fcmp("g32", ">=", -0.0)]
        t += [D.colcol("i32b", op, "i64b") for op in D.CMPS]
    return t + [x.negate() for x in t]


def edge_aggs():
    return [D.Agg("sum", [D.f_col("fa")]), D.Agg("min", [D.f_kplus(20.0, "fa")]), D.Agg("max", [D.f_kminus(-20.0, "fb")])]


@pytest.mark.parametrize("fast", [True, False], ids=["typed_walk", "row_walk"])
def test_dyn_term_edges(qk, fast):
    """One term per plan: open and closed fp bounds at exactly a data value and its nextafter neighbours, ±0 / NaN / ±inf
    data, ±inf constants, the subnormal nextafter(0), int32 columns against constants beyond ±2^31, int64 columns at their
    extremes, empty BETWEENs, sets of 6, 64 and 65 bits with codes beyond the set (uint8 codes up to 255, int32 codes
    -5..79), column pairs, and NOT of each.  MIN of positive and MAX of negative values: a wrong fold with the
    zero-initialised state shows."""
    d, dd = edge_data()
    key = ("k32", 4) if fast else ("k64", 3)
    for t in edge_terms(fast):
        plan = D.Plan([t], [("k8a", 3), key], edge_aggs())
        assert_dyn(*run_and_check(qk, plan, d, dd, 7, True, t.sql), fast=fast)
        assert run_and_check(qk, plan, d, dd, 1, True, t.sql)[0] == "generic"
        gated = D.Plan([], [key], [D.Agg("sum", [D.f_col("fb")], t)])                # the same term as a CASE gate
        assert_dyn(*run_and_check(qk, gated, d, dd, 7, True, "gate " + t.sql), fast=fast)
        assert run_and_check(qk, gated, d, dd, 1, True, "gate " + t.sql)[0] == "generic"


def edge_agg_plans(fast):
    key = ("k32", 4) if fast else ("k64", 3)
    ab = [D.f_col("fa"), D.f_col("fb")]
    abk = [D.f_col("fa"), D.f_kminus(0.5, "fb")]
    abk2 = [D.f_col("fa"), D.f_kminus(1.5, "fb"), D.f_col("fc")]
    plans = {
        "affine": [D.Agg("sum", [D.f_const(2.0)]), D.Agg("sum", [D.f_neg("fa")]), D.Agg("sum", [D.f_kminus(0.75, "fa")]),
                   D.Agg("sum", [D.f_minusk("fa", 0.75)]), D.Agg("sum", [D.f_kplus(-1.25, "fa")]), D.Agg("min", [D.f_neg("fa")]),
                   D.Agg("max", [D.f_minusk("fa", 3.0)]), D.Agg("max", [D.f_const(-2.0), D.f_col("fa")])],
        "prefix": [D.Agg("sum", ab), D.Agg("sum", ab + [D.f_col("fc")]), D.Agg("sum", ab + [D.f_col("fc")], D.irange("i32a", ">", 0)),
                   D.Agg("min", ab + [D.f_col("fc")]), D.Agg("sum", abk), D.Agg("sum", abk2), D.Agg("sum", ab + [D.f_col("fc")]),
                   D.Agg("sum", ab)],
        "prefix_same_cols_other_k": [D.Agg("sum", abk), D.Agg("sum", abk2), D.Agg("max", [D.f_col("fa"), D.f_kminus(0.5, "fb")]),
                                     D.Agg("min", [D.f_col("fa"), D.f_kplus(0.5, "fb"), D.f_col("fc")])],
    }
    out = [D.Plan([D.fcmp("fa", "<", 10.0)], [key], a) for a in plans.values()]
    out.append(D.Plan([D.irange("i32a", ">", -500)], [("k8a", 3), key], []))                       # COUNT only
    out.append(D.Plan([D.irange("i32a", ">", -500)], [("k8a", 5), key], edge_aggs()))             # groups 3, 4 of k8a: no rows
    return out


@pytest.mark.parametrize("fast", [True, False], ids=["typed_walk", "row_walk"])
def test_dyn_aggregate_edges(qk, fast):
    """sum(2), -x, k - x, x - k, k + x; product chains a*b, a*b*c shared with the previous aggregate, behind a CASE gate
    and behind a MIN; a*(k-b) followed by a*(k'-b)*c (same columns, other constant: no sharing); COUNT only; groups
    without rows (cardinalities beyond the codes present)."""
    d, dd = edge_data()
    for plan in edge_agg_plans(fast):
        assert_dyn(*run_and_check(qk, plan, d, dd, 7, True), fast=fast)
        assert run_and_check(qk, plan, d, dd, 1, True)[0] == "generic"
        assert run_and_check(qk, plan, d, dd, 0, True)[0] == "fused_tma:dyn"


@pytest.mark.parametrize("fast", [True, False], ids=["typed_walk", "row_walk"])
def test_min_max_signed_zero_nan_inf(qk, fast):
    """MIN / MAX over ±0, NaN and ±inf on every device path that takes them: fmin / fmax skip NaN (a group of NaN rows
    keeps the identity); zeros compare equal whatever their sign."""
    d, dd = edge_data()
    key = ("k32", 4) if fast else ("k64", 3)
    plan = D.Plan([], [("k8a", 3), key], [D.Agg("min", [D.f_col("fe")]), D.Agg("max", [D.f_col("fe")]),
                                          D.Agg("min", [D.f_neg("fe")]), D.Agg("max", [D.f_col("fe"), D.f_col("fe")])])
    plan_nan = D.Plan([D.fcmp("fe", "!=", 0.5)], [("k8a", 3), key], plan.aggs)
    for p in (plan, plan_nan):
        assert_dyn(*run_and_check(qk, p, d, dd, 7, True), fast=fast)
        assert run_and_check(qk, p, d, dd, 1, True)[0] == "generic"
    allnan = {k: v[:4096].copy() for k, v in d.items()}
    allnan["fe"][allnan["k8a"] == 1] = np.nan
    dn = {k: torch.from_numpy(v).cuda() for k, v in allnan.items()}
    for variant in (7, 1):
        run_and_check(qk, plan, allnan, dn, variant, True, "all-NaN group")


# ------------------------------------------------------------------ limits of the dynamic plan
def test_dyn_term_and_column_limits(qk):
    """6 terms and 10 staged columns run in the dynamic plan; a 7th term or an 11th column leaves it (the interpreter
    takes the call) and the result stays right."""
    d, dd = edge_data()
    six = [D.irange("i32a", ">", -900), D.fcmp("fa", "<", 15.0), D.inset("u8", [1, 2, 3, 100, 200]).negate(),
           D.colcol("i32a", "!=", "i32b"), D.irange("i64a", "<", 900), D.fcmp("fb", ">", -15.0)]
    keys = [("k8a", 3), ("k32", 4)]
    aggs = [D.Agg("sum", [D.f_col("fc")]), D.Agg("min", [D.f_col("fd")])]
    p10 = D.Plan(six, keys, aggs)                                      # i32a fa u8 i32b i64a fb k8a k32 fc fd
    assert len(p10.columns) == 10
    assert_dyn(*run_and_check(qk, p10, d, dd, 0, True, "6 terms 10 cols"), fast=True, ncols=10)
    p7 = D.Plan(six + [D.fcmp("fc", "!=", 0.25)], keys, aggs)
    assert run_and_check(qk, p7, d, dd, 0, True, "7 terms")[0] == "generic"
    with pytest.raises(Exception, match="no fused plan"):
        run(qk, p7, d, dd, 7)
    p11 = D.Plan(six, keys, aggs + [D.Agg("max", [D.f_col("fp")])])
    assert len(p11.columns) == 11
    assert run_and_check(qk, p11, d, dd, 0, True, "11 cols")[0] == "generic"
    with pytest.raises(Exception, match="no fused plan"):
        run(qk, p11, d, dd, 7)


def _four_cards(ng):
    """ng as a product of four key cardinalities (prime factors spread over the keys, 1 where they run out)"""
    f, p, m = [], 2, ng
    while m > 1:
        while m % p == 0:
            f.append(p)
            m //= p
        p += 1
    cards = [1, 1, 1, 1]
    for x in sorted(f, reverse=True):
        cards[int(np.argmin(cards))] *= x
    return cards


@pytest.mark.parametrize("shape", D.DYN_SHAPES, ids=[f"{a}x{b}" for a, b in D.DYN_SHAPES])
def test_dyn_largest_grouping_per_shape(qk, monkeypatch, shape):
    """Four int32 keys whose product is the largest group count the pinned shape accepts run in that shape; one group
    more does not fit it and falls through to the shape launch_dyn picks, to the interpreter, or to the
    `exceed the shared-memory dense path` error when nothing holds it."""
    monkeypatch.setenv("QK_DYN_SHAPE", f"{shape[0]}x{shape[1]}")
    n = 60_011
    rng = np.random.default_rng(shape[0] * 10 + shape[1])
    row_bytes = 4 * 4 + 8
    for ng in (D.dyn_max_groups(row_bytes, 1, *shape), D.dyn_max_groups(row_bytes, 1, *shape) + 1):
        cards = _four_cards(ng)
        d = {f"q{i}": rng.integers(0, c, n).astype(np.int32) for i, c in enumerate(cards)}
        d["fa"] = D.dyadic(rng, n)
        dd = {k: torch.from_numpy(v).cuda() for k, v in d.items()}
        plan = D.Plan([], [(f"q{i}", c) for i, c in enumerate(cards)], [D.Agg("sum", [D.f_col("fa")])])
        if ng == D.dyn_max_groups(row_bytes, 1, *shape):
            assert_dyn(*run_and_check(qk, plan, d, dd, 0, True, f"ng {ng}"), shape=shape, fast=True)
            continue
        pick = D.dyn_pick(row_bytes, ng, 1)
        if pick is None and not qk.dense_agg_fits(ng, 1):
            with pytest.raises(Exception, match="exceed the shared-memory dense path"):
                run(qk, plan, d, dd, 0)
            continue
        v, cfg = run_and_check(qk, plan, d, dd, 0, True, f"ng {ng}")
        if pick is None:
            assert v == "generic", (v, cfg)
        else:
            assert pick != shape
            assert_dyn(v, cfg, shape=pick, fast=True)


# ------------------------------------------------------------------ state across calls, determinism, misaligned views
def test_state_across_variants_and_determinism(qk):
    """Three update() calls into one DenseAggState through variants 7, 1 and 0; the first batch holds only the groups of
    k8a = 0, so MIN / MAX of the others start in the second.  Running the same calls again gives bit-equal acc / cnt."""
    d, dd = data(300_007, 21)
    plan = D.Plan([D.fcmp("fa", ">", -14.0)], [("k8a", 3), ("k8b", 2)],
                  [D.Agg("min", [D.f_kplus(20.0, "fb")]), D.Agg("max", [D.f_kminus(-20.0, "fc")]), D.Agg("sum", [D.f_col("fa"), D.f_col("fb")]),
                   D.Agg("max", [D.f_col("fd")])])
    batches = [d["k8a"] == 0, (d["k8a"] != 0) & (np.arange(len(d["fa"])) % 2 == 0), (d["k8a"] != 0) & (np.arange(len(d["fa"])) % 2 == 1)]
    states = []
    for _ in range(2):
        st = None
        for sel, variant, want in zip(batches, (7, 1, 0), ("fused_tma:dyn", "generic", "fused_tma:dyn")):
            bd = {k: np.ascontiguousarray(v[sel]) for k, v in d.items()}
            st, v, _ = run(qk, plan, bd, {k: torch.from_numpy(x).cuda() for k, x in bd.items()}, variant, st)
            assert v == want
        acc, cnt = host(st)
        D.check(plan, acc, cnt, D.reference(plan, d), True, "batches")
        states.append(st)
    assert torch.equal(states[0].acc, states[1].acc) and torch.equal(states[0].cnt, states[1].cnt)


@pytest.mark.parametrize("offset", range(1, 16))
def test_misaligned_views_decline_to_the_interpreter(qk, offset):
    """Column views that start `offset` rows into their buffers (the uint8 columns `offset` bytes off a 16-byte boundary):
    the TMA and vector-load paths need 16-byte aligned bases, so the default dispatch takes the interpreter and a forced
    fused variant is refused; the results stay right."""
    n = 20_011
    d, dd = data(n + 16, 31)
    dv = {k: v[offset:offset + n] for k, v in d.items()}
    ddv = {k: v[offset:offset + n] for k, v in dd.items()}
    for plan in (typed_plan("q1", "dyadic"), shape_plan(True)):
        assert run_and_check(qk, plan, dv, ddv, 0, True, f"offset {offset}")[0] == "generic"
        for variant in (3, 7):
            with pytest.raises(Exception, match="no fused plan"):
                run(qk, plan, dv, ddv, variant)


# ------------------------------------------------------------------ random differential
@pytest.mark.parametrize("seed", range(300))
def test_random_plans_dyn_vs_interpreter(qk, seed):
    """A generated plan (dense_agg_cases.random_plan, its own seed) over 100 003 rows, on variant 7 and on the interpreter,
    both against the reference: bit for bit on dyadic data (two seeds in three), within the error bound on TPC-H data."""
    mode = "tpch" if seed % 3 == 0 else "dyadic"
    fast = seed % 2 == 1
    d, dd = data(100_003, 0 if mode == "dyadic" else 1, mode)
    plan = D.random_plan(np.random.default_rng(seed), d, fast=fast)
    v, cfg = run_and_check(qk, plan, d, dd, 7, mode == "dyadic", f"seed {seed}")
    m = assert_dyn(v, cfg, ncols=len(plan.columns))
    if fast:
        assert m[4] == "t", cfg
    assert run_and_check(qk, plan, d, dd, 1, mode == "dyadic", f"seed {seed}")[0] == "generic"


# ------------------------------------------------------------------ one large run on the default path
def test_forty_million_rows_default_path(qk):
    """40 000 003 rows through the default dispatch: the typed Q1 plan, then a plan only the dynamic plan takes, whose grid
    of up to six CTAs per SM folds hundreds of partial states (MAX_PART_BLOCKS = 1024)."""
    n = 40_000_003
    rng = np.random.default_rng(40)
    d = {"i32a": rng.integers(-1000, 1000, n).astype(np.int32), "k8a": rng.integers(0, 3, n).astype(np.uint8),
         "k8b": rng.integers(0, 2, n).astype(np.uint8)}
    for c in ("fa", "fb", "fc", "fd"):
        d[c] = D.dyadic(rng, n)
    dd = {k: torch.from_numpy(v).cuda() for k, v in d.items()}
    q1 = typed_plan("q1", "dyadic")
    assert run_and_check(qk, q1, d, dd, 0, True, "40M")[0] == "fused_tma:q1"
    dyn = D.Plan(q1.terms + [D.fcmp("fa", "!=", 1.0)], q1.keys, q1.aggs[:3] + [D.Agg("min", [D.f_kplus(20.0, "fd")])])
    assert_dyn(*run_and_check(qk, dyn, d, dd, 0, True, "40M"), fast=True)
    del dd
    torch.cuda.empty_cache()


# ------------------------------------------------------------------ routing of dictionary groupings
@pytest.fixture
def qc():
    from quokka_b200.df import QuokkaContext
    return QuokkaContext()


@pytest.mark.parametrize("pred", D.ROUTING_PREDS)
@pytest.mark.parametrize("nsum", D.ROUTING_AGGS)
@pytest.mark.parametrize("n_groups", D.ROUTING_GROUPS)
def test_dictionary_groupby_routing(qk, qc, monkeypatch, n_groups, nsum, pred):
    """groupby(<dictionary column>) of 66, 67, 150 and 1 024 values against pandas: a dense kernel at or below
    ops.dense_agg_fits, the per-row path above it (it raised QK_ERR_UNSUPPORTED before when the call reached the
    interpreter)."""
    paths = D.routing_case(qc, monkeypatch, n_groups, nsum, pred)
    for p in paths:
        if qk.dense_agg_fits(n_groups, nsum):
            assert p in ("fused_tma:dyn", "generic"), paths
        else:
            assert p == "rows", paths
