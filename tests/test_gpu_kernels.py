"""Parity of every libqk.so kernel against the oracle, through the C-ABI (quokka_b200.ops -> ctypes).
Bar: bit-exact for integer / byte / index work; fp64 aggregates within 1e-9 relative (north_star)."""
import os

import numpy as np
import pytest
import torch

from oracle import queries as Q
from oracle import relops as R
from oracle import tpch_gen as G

pytestmark = pytest.mark.gpu

RTOL = 1e-9      # north_star: fp64 aggregates within 1e-9 relative


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    return t.cpu().numpy()


@pytest.fixture(scope="module")
def qb():
    from quokka_b200 import _lib, expr, ops, synth
    _lib.lib()
    return type("QB", (), dict(L=_lib, E=expr, ops=ops, synth=synth))


# ------------------------------------------------------------------ synthetic generator
def test_synth_matches_numpy_generator(qb):
    sf = 0.01
    li = G.gen_lineitem(sf)
    for name, v in li.items():
        got = host(qb.synth.column(name, sf))
        assert got.dtype == v.dtype, name
        assert np.array_equal(got, v), name
    for name, v in {**G.gen_orders(sf), **G.gen_customer(sf), **G.gen_supplier(sf)}.items():
        assert np.array_equal(host(qb.synth.column(name, sf)), v), name
    # any row range, far into an SF-100 table
    lo, hi = 599_000_000, 599_000_000 + 5000
    ref = G.gen_lineitem(100, lo, hi, ["l_extendedprice", "l_shipdate", "l_returnflag", "l_orderkey"])
    for name, v in ref.items():
        assert np.array_equal(host(qb.synth.column(name, 100, lo, hi)), v), name
    for tid in (G.T_TRADES, G.T_QUOTES):
        ref = G.gen_ticks(tid, 20000, 100)
        got = qb.synth.ticks(tid, 20000, 100)
        for name, v in ref.items():
            assert np.array_equal(host(got[name]), v), (tid, name)


# ------------------------------------------------------------------ K1 scan / filter / project
def _schema(qb, cols, dicts=None):
    sch = {}
    for i, (name, t) in enumerate(cols.items()):
        sch[name] = qb.E.ColumnInfo(i, qb.ops.qk_dtype(t), (dicts or {}).get(name))
    return sch


@pytest.mark.parametrize("n", [0, 1, 31, 1000, 2049, 100_003])
@pytest.mark.parametrize("stable", [False, True])
def test_scan_filter_project(qb, n, stable):
    li = G.gen_lineitem(1, 0, n, ["l_orderkey", "l_shipdate", "l_extendedprice", "l_discount", "l_returnflag"])
    d = {k: dev(v) for k, v in li.items()}
    sch = _schema(qb, d)
    pred = qb.E.compile_expr(qb.E.parse("l_shipdate > date '1995-03-15' and l_discount >= 0.05"), sch)
    projs = [qb.E.compile_expr(qb.E.parse(s), sch) for s in
             ("l_orderkey", "l_extendedprice * (1 - l_discount)", "l_returnflag", "l_shipdate")]
    outs, m = qb.ops.scan_filter_project(list(d.values()), pred, projs, stable=stable)
    mask = (li["l_shipdate"] > G.DAY_1995_03_15) & (li["l_discount"] >= 0.05)
    assert m == int(mask.sum())
    exp = [li["l_orderkey"][mask], (li["l_extendedprice"] * (1 - li["l_discount"]))[mask], li["l_returnflag"][mask],
           li["l_shipdate"][mask]]
    got = [host(o) for o in outs]
    assert got[0].dtype == np.int64 and got[1].dtype == np.float64 and got[2].dtype == np.uint8 and got[3].dtype == np.int32
    if stable:
        for g, e in zip(got, exp):
            assert np.array_equal(g, e)          # bit-exact, including the fp64 expression (no FMA contraction)
    else:
        # unordered compaction: same multiset of rows
        order_g = np.lexsort((got[1], got[0]))
        order_e = np.lexsort((exp[1], exp[0]))
        for g, e in zip(got, exp):
            assert np.array_equal(g[order_g], e[order_e])


def test_scan_predicate_forms(qb):
    n = 50_000
    li = G.gen_lineitem(1, 0, n, ["l_suppkey", "l_partkey", "l_quantity", "l_discount", "l_shipdate", "l_returnflag"])
    d = {k: dev(v) for k, v in li.items()}
    sch = _schema(qb, d, {"l_returnflag": G.RETURNFLAG_DICT})
    cases = {
        "l_suppkey = l_partkey or l_quantity < 3": (li["l_suppkey"] == li["l_partkey"]) | (li["l_quantity"] < 3),
        "l_returnflag = 'R' and not l_quantity > 25": (li["l_returnflag"] == 2) & ~(li["l_quantity"] > 25),
        "l_returnflag != 'N'": li["l_returnflag"] != 1,
        "l_returnflag = 'ZZZ'": np.zeros(n, bool),
        "l_discount between 0.06 - 0.01 and 0.06 + 0.01 and l_quantity < 24": (li["l_discount"] >= 0.06 - 0.01) & (li["l_discount"] <= 0.06 + 0.01) & (li["l_quantity"] < 24),
        "l_suppkey in (1, 2, 3, 5000)": np.isin(li["l_suppkey"], [1, 2, 3, 5000]),
        "l_shipdate >= date '1994-01-01' and l_shipdate < date '1994-01-01' + interval '1' year": (li["l_shipdate"] >= G.DAY_1994_01_01) & (li["l_shipdate"] < G.DAY_1995_01_01),
        "l_quantity * 2 + 1 > l_discount * 100": li["l_quantity"] * 2 + 1 > li["l_discount"] * 100,
    }
    for sql, mask in cases.items():
        pred = qb.E.compile_expr(qb.E.parse(sql), sch)
        outs, m = qb.ops.scan_filter_project(list(d.values()), pred, [qb.E.compile_expr(qb.E.parse("l_partkey"), sch)], stable=True)
        assert m == int(mask.sum()), sql
        assert np.array_equal(host(outs[0]), li["l_partkey"][mask]), sql


def test_set_membership_and_select_ops(qb):
    """QK_OP_IN_SET (inline 64-bit bitmap and device bitmap) and QK_OP_SELECT against numpy: LIKE / IN over a 150-value
    dictionary (TPC-H p_type) is ONE node (pyquokka/sql_utils.py:131-149), CASE evaluates its condition once
    (sql_utils.py:161-168) and an unselected NaN / inf arm does not leak."""
    rng = np.random.default_rng(7)
    n = 200_003
    types = [f"{a} {b} {c}" for a in ("STANDARD", "SMALL", "MEDIUM", "LARGE", "ECONOMY", "PROMO")
             for b in ("ANODIZED", "BURNISHED", "PLATED", "POLISHED", "BRUSHED") for c in ("TIN", "NICKEL", "BRASS", "STEEL", "COPPER")]
    big = [f"v{i:05d}" for i in range(3000)]
    h = {"p_type": rng.integers(0, 150, n).astype(np.uint8), "big": rng.integers(0, 3000, n).astype(np.int32),
         "k": rng.integers(-3, 70, n).astype(np.int64), "x": rng.random(n) * 100, "y": rng.random(n).round(2)}
    d = {k: dev(v) for k, v in h.items()}
    sch = _schema(qb, d, {"p_type": types, "big": big})
    promo = np.array([t.startswith("PROMO") for t in types])
    brass = np.array([t.endswith("BRASS") for t in types])
    big7 = np.array([v.endswith("7") for v in big])
    with np.errstate(all="ignore"):
        cases = {
            "p_type like 'PROMO%'": promo[h["p_type"]],
            "p_type not like '%BRASS' and x < 50": ~brass[h["p_type"]] & (h["x"] < 50),
            "p_type in ('PROMO PLATED TIN', 'SMALL BRUSHED STEEL', 'nope')": np.isin(h["p_type"], [types.index("PROMO PLATED TIN"), types.index("SMALL BRUSHED STEEL")]),
            "big like '%7'": big7[h["big"]],                                    # 300 of 3000 codes: device bitmap
            "k in (0, 3, 63, 64, 69)": np.isin(h["k"], [0, 3, 63, 64, 69]),         # spans > 64 bits: device bitmap
            "k in (1, 2, 63)": np.isin(h["k"], [1, 2, 63]),                        # inline bitmap, negative codes present
            "k in (-1, 5)": np.isin(h["k"], [-1, 5]),                              # OR-chain of exact compares
        }
        vals = {
            "case when p_type like 'PROMO%' then x * (1 - y) else 0 end": np.where(promo[h["p_type"]], h["x"] * (1 - h["y"]), 0.0),
            "case when y > 0 then x / y else -1 end": np.where(h["y"] > 0, h["x"] / np.where(h["y"] > 0, h["y"], 1.0), -1.0),
            "case when k < 0 then 1 when k < 10 then 2 else 3 end": np.where(h["k"] < 0, 1.0, np.where(h["k"] < 10, 2.0, 3.0)),
        }
    ident = qb.E.compile_expr(qb.E.parse("k"), sch)
    for sql, mask in cases.items():
        pred = qb.E.compile_expr(qb.E.parse(sql), sch)
        assert len(pred) <= 6, sql
        outs, m = qb.ops.scan_filter_project(list(d.values()), pred, [ident], stable=True)
        assert m == int(mask.sum()), sql
        assert np.array_equal(host(outs[0]), h["k"][mask]), sql
    for sql, exp in vals.items():
        outs, m = qb.ops.scan_filter_project(list(d.values()), None, [qb.E.compile_expr(qb.E.parse(sql), sch)], stable=True)
        assert m == n and np.array_equal(host(outs[0]), exp), sql              # bit-exact: same fp64 operations, no FMA
    # the same programs inside the dense aggregate (Q14's promo_revenue shape), generic interpreter
    st = qb.ops.DenseAggState([], [qb.L.AGG_SUM, qb.L.AGG_SUM], d["x"].device)
    progs = [qb.E.compile_expr(qb.E.parse(e), sch) for e in ("case when p_type like 'PROMO%' then x * (1 - y) else 0 end", "x * (1 - y)")]
    st.update(list(d.values()), qb.E.compile_expr(qb.E.parse("big like '%7'"), sch), [], progs)
    m = big7[h["big"]]
    rev = h["x"] * (1 - h["y"])
    assert np.allclose(host(st.acc)[0], [rev[m & promo[h["p_type"]]].sum(), rev[m].sum()], rtol=RTOL)
    assert int(host(st.cnt)[0]) == int(m.sum())


# ------------------------------------------------------------------ K1+K2 dense aggregate (Q1)
Q1_COLS = ["l_shipdate", "l_returnflag", "l_linestatus", "l_quantity", "l_extendedprice", "l_discount", "l_tax"]
Q1_AGGS = ["l_quantity", "l_extendedprice", "l_extendedprice * (1 - l_discount)",
           "l_extendedprice * (1 - l_discount) * (1 + l_tax)", "l_discount"]


def run_q1_dense(qb, d, variant, pred_sql="l_shipdate <= date '1998-12-01' - interval '90' day", aggs=Q1_AGGS, ops=None):
    sch = _schema(qb, d)
    pred = qb.E.compile_expr(qb.E.parse(pred_sql), sch) if pred_sql else None
    progs = [qb.E.compile_expr(qb.E.parse(a), sch) for a in aggs]
    st = qb.ops.DenseAggState([3, 2], ops or [qb.L.AGG_SUM] * len(aggs), "cuda")
    st.update(list(d.values()), pred, [sch["l_returnflag"].slot, sch["l_linestatus"].slot], progs, variant=variant)
    return st


def check_q1(st, li):
    exp = Q.q1(li)
    acc, cnt = host(st.acc), host(st.cnt)
    gid = exp["l_returnflag"].astype(int) * 2 + exp["l_linestatus"].astype(int)
    assert np.array_equal(cnt[gid], exp["count_order"])                       # bit-exact counts
    assert cnt.sum() == exp["count_order"].sum()                              # no rows in other groups
    for j, name in enumerate(["sum_qty", "sum_base_price", "sum_disc_price", "sum_charge"]):
        np.testing.assert_allclose(acc[gid, j], exp[name], rtol=RTOL, atol=0)
    np.testing.assert_allclose(acc[gid, 4] / cnt[gid], exp["avg_disc"], rtol=RTOL, atol=0)
    np.testing.assert_allclose(acc[gid, 0] / cnt[gid], exp["avg_qty"], rtol=RTOL, atol=0)


@pytest.mark.parametrize("variant,name", [(1, "generic"), (3, "fused_tma:q1"), (7, "fused_tma:dyn"), (0, "fused_tma:q1")])
@pytest.mark.parametrize("n", [1, 1023, 1024, 1025, 4099, 300_007])
def test_q1_dense_agg_variants(qb, variant, name, n):
    li = G.gen_lineitem(1, 5_000_000, 5_000_000 + n, Q1_COLS)
    d = {k: dev(li[k]) for k in Q1_COLS}
    st = run_q1_dense(qb, d, variant)
    assert qb.ops.last_variant() == name
    check_q1(st, li)


def test_q1_typed_plan_accumulates_over_batches_and_is_deterministic(qb):
    n = 500_000
    li = G.gen_lineitem(1, 0, n, Q1_COLS)
    d = {k: dev(li[k]) for k in Q1_COLS}
    whole = run_q1_dense(qb, d, 3)
    again = run_q1_dense(qb, d, 3)
    assert torch.equal(whole.acc, again.acc) and torch.equal(whole.cnt, again.cnt)     # fixed reduction order
    sch = _schema(qb, d)
    pred = qb.E.compile_expr(qb.E.parse("l_shipdate <= date '1998-09-02'"), sch)
    progs = [qb.E.compile_expr(qb.E.parse(a), sch) for a in Q1_AGGS]
    st = qb.ops.DenseAggState([3, 2], [qb.L.AGG_SUM] * 5, "cuda")
    for lo in range(0, n, 123_457):                      # ragged batches; misaligned slices take the generic kernel
        part = [t[lo:lo + 123_457] for t in d.values()]
        st.update(part, pred, [1, 2], progs)
    check_q1(st, li)
    np.testing.assert_allclose(host(st.acc), host(whole.acc), rtol=1e-12)


def test_dense_agg_min_max_and_rev1_typed_and_dyn(qb):
    n = 200_000
    li = G.gen_lineitem(1, 0, n, Q1_COLS)
    d = {k: dev(li[k]) for k in Q1_COLS}
    st = run_q1_dense(qb, d, 0, aggs=["l_extendedprice", "l_extendedprice", "l_quantity + l_tax"],
                      ops=[qb.L.AGG_MIN, qb.L.AGG_MAX, qb.L.AGG_SUM])
    assert qb.ops.last_variant() == "generic"
    m = li["l_shipdate"] <= G.DAY_1998_09_02
    keys = {"a": li["l_returnflag"][m], "b": li["l_linestatus"][m]}
    exp = R.group_aggregate(keys, {"mn": ("min", li["l_extendedprice"][m]), "mx": ("max", li["l_extendedprice"][m]),
                                  "s": ("sum", (li["l_quantity"] + li["l_tax"])[m])})
    gid = exp["a"].astype(int) * 2 + exp["b"].astype(int)
    acc = host(st.acc)
    assert np.array_equal(acc[gid, 0], exp["mn"]) and np.array_equal(acc[gid, 1], exp["mx"])
    np.testing.assert_allclose(acc[gid, 2], exp["s"], rtol=RTOL)
    # revenue-by-one-key plan: the typed "rev1" plan and the runtime-described plan
    sch = _schema(qb, d)
    for variant, name in ((3, "fused_tma:rev1"), (7, "fused_tma:dyn")):
        st = qb.ops.DenseAggState([3], [qb.L.AGG_SUM], "cuda")
        st.update(list(d.values()), qb.E.compile_expr(qb.E.parse("l_shipdate > date '1995-03-15'"), sch), [sch["l_returnflag"].slot],
                  [qb.E.compile_expr(qb.E.parse("l_extendedprice * (1 - l_discount)"), sch)], variant=variant)
        assert qb.ops.last_variant() == name
        m = li["l_shipdate"] > G.DAY_1995_03_15
        exp = R.group_aggregate({"a": li["l_returnflag"][m]}, {"r": ("sum", (li["l_extendedprice"] * (1 - li["l_discount"]))[m]), "c": ("count", None)})
        np.testing.assert_allclose(host(st.acc)[exp["a"].astype(int), 0], exp["r"], rtol=RTOL)
        assert np.array_equal(host(st.cnt)[exp["a"].astype(int)], exp["c"])


@pytest.mark.parametrize("n", [1, 255, 1024, 1025, 300_007])
def test_dense_agg_dynamic_fused_plan(qb, n):
    """The runtime-described fused plan (csrc/scan.cu k_dense_agg_dyn_tma: same TMA tile ring as the typed Q1 plan) against
    numpy AND against the per-row interpreter, on the aggregate shapes of tpch.py that are not the three typed plans:
    Q6 (three range terms, one of them on an fp64 column, ungrouped), Q14 (CASE WHEN code IN set ... ELSE 0), Q12-like
    (two gated counts), MIN / MAX, Q1 itself forced through the dynamic plan.  SUMs within 1e-9, counts / MIN / MAX exact."""
    rng = np.random.default_rng(n)
    cols = ["l_shipdate", "l_returnflag", "l_linestatus", "l_quantity", "l_extendedprice", "l_discount", "l_tax"]
    li = G.gen_lineitem(1, 1_000_000, 1_000_000 + n, cols)
    li["p_type"] = rng.integers(0, 150, n).astype(np.uint8)
    li["ka"], li["kb"] = rng.integers(0, 25, n), rng.integers(0, 25, n)                       # int64 keys compared column to column (Q5)
    li["nat"] = rng.integers(0, 25, n).astype(np.int32)                                        # an int32-coded dictionary key
    d = {k: dev(v) for k, v in li.items()}
    types = [f"{a} {b}" for a in ("STANDARD", "SMALL", "MEDIUM", "LARGE", "ECONOMY", "PROMO") for b in range(25)]
    sch = _schema(qb, d, {"p_type": types, "nat": G.NATIONS})
    promo = np.array([t.startswith("PROMO") for t in types])[li["p_type"]]
    rev = li["l_extendedprice"] * (1 - li["l_discount"])
    cases = [
        # (predicate, group columns, [(op, expr)], numpy mask, [numpy values])
        ("l_shipdate >= date '1994-01-01' and l_shipdate < date '1995-01-01' and l_discount between 0.05 and 0.07 and l_quantity < 24", [],
         [("sum", "l_extendedprice * l_discount")],
         (li["l_shipdate"] >= G.DAY_1994_01_01) & (li["l_shipdate"] < G.DAY_1995_01_01) & (li["l_discount"] >= 0.05) & (li["l_discount"] <= 0.07) & (li["l_quantity"] < 24),
         [li["l_extendedprice"] * li["l_discount"]]),
        ("l_shipdate >= date '1995-09-01'", [],
         [("sum", "case when p_type like 'PROMO%' then l_extendedprice * (1 - l_discount) else 0 end"), ("sum", "l_extendedprice * (1 - l_discount)")],
         li["l_shipdate"] >= 9374,                                                            # date '1995-09-01'
         [np.where(promo, rev, 0.0), rev]),
        ("not l_quantity > 30", ["l_linestatus"],
         [("sum", "case when l_returnflag in ('A', 'R') then 1 else 0 end"), ("sum", "case when l_returnflag not in ('A', 'R') then 1 else 0 end"),
          ("min", "l_extendedprice"), ("max", "1 - l_discount"), ("sum", "-l_tax")],
         ~(li["l_quantity"] > 30),
         [np.isin(li["l_returnflag"], [G.RETURNFLAG_DICT.index("A"), G.RETURNFLAG_DICT.index("R")]).astype(float),
          (~np.isin(li["l_returnflag"], [G.RETURNFLAG_DICT.index("A"), G.RETURNFLAG_DICT.index("R")])).astype(float),
          li["l_extendedprice"], 1 - li["l_discount"], -li["l_tax"]]),
        ("l_shipdate <= date '1998-09-02'", ["l_returnflag", "l_linestatus"], [("sum", a) for a in Q1_AGGS], li["l_shipdate"] <= G.DAY_1998_09_02,
         [li["l_quantity"], li["l_extendedprice"], rev, rev * (1 + li["l_tax"]), li["l_discount"]]),
        # Q5's final aggregate: int64 column = int64 column, an int32-coded key; then `<`, an int64 range and both together
        ("ka = kb", ["nat"], [("sum", "l_extendedprice * (1 - l_discount)")], li["ka"] == li["kb"], [rev]),
        ("ka < kb and ka >= 3 and not ka = 7", ["l_linestatus", "l_returnflag"], [("sum", "l_extendedprice"), ("max", "l_tax")],
         (li["ka"] < li["kb"]) & (li["ka"] >= 3) & (li["ka"] != 7), [li["l_extendedprice"], li["l_tax"]]),
    ]
    sch["l_returnflag"].dictionary = G.RETURNFLAG_DICT
    sch["l_linestatus"].dictionary = G.LINESTATUS_DICT
    assert qb.E.compile_expr(qb.E.parse("ka = kb"), sch)[0][0] == qb.L.OP_CMP_COL_COL
    OPS = {"sum": qb.L.AGG_SUM, "min": qb.L.AGG_MIN, "max": qb.L.AGG_MAX}
    for pred_sql, gcols, aggs, mask, vals in cases:
        card = [len(sch[g].dictionary) for g in gcols]
        pred = qb.E.compile_expr(qb.E.parse(pred_sql), sch)
        progs = [qb.E.compile_expr(qb.E.parse(e), sch) for _, e in aggs]
        res = {}
        for variant in (7, 1):                                       # 7 = the dynamic fused plan, 1 = the interpreter
            st = qb.ops.DenseAggState(card, [OPS[o] for o, _ in aggs], "cuda")
            st.update(list(d.values()), pred, [sch[g].slot for g in gcols], progs, variant=variant)
            assert qb.ops.last_variant() == ("fused_tma:dyn" if variant == 7 else "generic"), (pred_sql, variant)
            res[variant] = (host(st.acc), host(st.cnt))
        gid = np.zeros(n, dtype=np.int64)
        for g, c in zip(gcols, card):
            gid = gid * c + li[g].astype(np.int64)
        ng = int(np.prod(card)) if card else 1
        exp_cnt = np.bincount(gid[mask], minlength=ng)
        for variant in (7, 1):
            acc, cnt = res[variant]
            assert np.array_equal(cnt, exp_cnt), (pred_sql, variant)
            for j, ((op, _), v) in enumerate(zip(aggs, vals)):
                for g in range(ng):
                    sel = mask & (gid == g)
                    if not sel.any():
                        continue
                    if op == "sum":
                        np.testing.assert_allclose(acc[g, j], v[sel].sum(), rtol=RTOL, atol=1e-9, err_msg=f"{pred_sql} agg {j} variant {variant}")
                    else:
                        assert acc[g, j] == (v[sel].min() if op == "min" else v[sel].max()), (pred_sql, j, variant)
    # default dispatch: typed plan for Q1, the dynamic plan for the others -- never the interpreter for this grammar
    st = qb.ops.DenseAggState([], [qb.L.AGG_SUM], "cuda")
    st.update(list(d.values()), qb.E.compile_expr(qb.E.parse(cases[0][0]), sch), [], [qb.E.compile_expr(qb.E.parse("l_extendedprice * l_discount"), sch)])
    assert qb.ops.last_variant() == "fused_tma:dyn"


# ------------------------------------------------------------------ K2 hash aggregate
@pytest.mark.parametrize("n,card", [(0, 10), (1, 1), (5000, 7), (200_000, 50_000), (300_000, 300_000)])
def test_hash_aggregate(qb, n, card):
    rng = np.random.default_rng(n + card)
    k0 = rng.integers(0, max(card, 1), n).astype(np.int64) * 977 - 5
    k1 = (k0 % 13).astype(np.int32)
    k2 = rng.integers(0, 2, n).astype(np.int32)
    v = rng.normal(size=n) * 1e4
    st = qb.ops.HashAggState([torch.int64, torch.int32, torch.int32], [qb.L.AGG_SUM, qb.L.AGG_MIN, qb.L.AGG_MAX], 2 * n + 16, "cuda")
    for lo in range(0, max(n, 1), 70_001):
        sl = slice(lo, lo + 70_001)
        st.update([dev(k0[sl]), dev(k1[sl]), dev(k2[sl])], [dev(v[sl])] * 3)
    keys, vals, cnt = st.finalize()
    exp = R.group_aggregate({"a": k0, "b": k1, "c": k2}, {"s": ("sum", v), "mn": ("min", v), "mx": ("max", v), "n": ("count", None)})
    got = {"a": host(keys[0]), "b": host(keys[1]), "c": host(keys[2])}
    assert len(got["a"]) == len(exp["a"])
    order = np.lexsort((got["c"], got["b"], got["a"]))
    for name in "abc":
        assert np.array_equal(got[name][order], exp[name])                 # integer keys bit-exact
    assert np.array_equal(host(cnt)[order], exp["n"])
    np.testing.assert_allclose(host(vals[0])[order], exp["s"], rtol=RTOL, atol=1e-6)
    assert np.array_equal(host(vals[1])[order], exp["mn"]) and np.array_equal(host(vals[2])[order], exp["mx"])


# ------------------------------------------------------------------ K3 partition + scatter
@pytest.mark.parametrize("n,nparts", [(0, 8), (1, 8), (4097, 2), (100_000, 8), (100_000, 7), (50_000, 1000),
                                      (1024 * 4096 + 1, 3)])          # 1025 chunks of 4096 rows: one carry of the count scan
def test_partition_matches_key_mod_n_and_is_stable(qb, n, nparts):
    rng = np.random.default_rng(1)
    key = rng.integers(0, 10_000_000, n).astype(np.int64)
    pay = np.arange(n, dtype=np.float64)
    code = rng.integers(0, 255, n).astype(np.uint8)
    dest, offs = qb.ops.partition_plan(dev(key), nparts)
    outs = qb.ops.scatter([dev(key), dev(pay), dev(code)], dest)
    offs = host(offs)
    exp = R.partition_table({"k": key, "p": pay, "c": code}, "k", nparts)
    assert offs[0] == 0 and offs[-1] == n
    for ch in range(nparts):
        lo, hi = offs[ch], offs[ch + 1]
        if ch not in exp:
            assert lo == hi
            continue
        assert np.array_equal(host(outs[0])[lo:hi], exp[ch]["k"])          # same rows, same (stable) order
        assert np.array_equal(host(outs[1])[lo:hi], exp[ch]["p"])
        assert np.array_equal(host(outs[2])[lo:hi], exp[ch]["c"])


def test_partition_by_code_many_parts(qb):
    n, nparts = 200_000, 8000
    rng = np.random.default_rng(2)
    code = np.minimum((rng.random(n) ** 2 * nparts).astype(np.int32), nparts - 1)
    dest, offs = qb.ops.partition_plan(dev(code), nparts, qb.L.PART_CODE)
    out = host(qb.ops.scatter([dev(np.arange(n, dtype=np.int64))], dest)[0])
    order = np.argsort(code, kind="stable")
    assert np.array_equal(out, order)
    assert np.array_equal(host(offs), np.concatenate([[0], np.cumsum(np.bincount(code, minlength=nparts))]))


# ------------------------------------------------------------------ K4 / K5 join
def _pairs(pi, bi):
    return set(zip(host(pi).tolist(), host(bi).tolist()))


def test_join_golden_ab(qb, golden_dir):
    g = np.load(os.path.join(golden_dir, "join_ab.npz"))
    t = qb.ops.JoinTable(len(g["key_b"]), "cuda")
    t.build(dev(g["key_b"]))
    pi, bi = t.probe(dev(g["key_a"]), qb.L.JOIN_INNER)
    assert t.check_flags() & 4                                       # duplicate build keys detected
    assert pi.numel() == int(g["n_inner"]) == 10118                   # lesson2.1.py:64-68
    assert _pairs(pi, bi) == set(zip(g["inner_ia"].tolist(), g["inner_ib"].tolist()))
    a1 = qb.ops.gather([dev(g["val1_a"])], pi)[0]
    b1 = qb.ops.gather([dev(g["val1_b"])], bi)[0]
    assert abs(float((a1 * b1).sum().item()) - float(g["dot_val1"])) <= 1e-9 * abs(float(g["dot_val1"]))
    assert t.probe(dev(g["key_a"]), qb.L.JOIN_SEMI)[0].numel() == int(g["n_semi"])
    assert t.probe(dev(g["key_a"]), qb.L.JOIN_ANTI)[0].numel() == int(g["n_anti"])
    assert t.probe(dev(g["key_a"]), qb.L.JOIN_LEFT)[0].numel() == int(g["n_left"])


@pytest.mark.parametrize("how", ["inner", "left", "semi", "anti"])
@pytest.mark.parametrize("nb,npr,dom", [(0, 1000, 100), (1000, 0, 100), (50_000, 200_000, 40_000), (30_000, 100_000, 3_000)])
def test_join_vs_oracle(qb, how, nb, npr, dom):
    rng = np.random.default_rng(nb + npr)
    bk = rng.integers(-dom, dom, nb).astype(np.int64) * 1_000_003
    pk = rng.integers(-dom, dom, npr).astype(np.int64) * 1_000_003
    t = qb.ops.JoinTable(nb, "cuda")
    for lo in range(0, nb, 17_000):                                   # several build batches share the table
        t.build(dev(bk[lo:lo + 17_000]))
    code = {"inner": qb.L.JOIN_INNER, "left": qb.L.JOIN_LEFT, "semi": qb.L.JOIN_SEMI, "anti": qb.L.JOIN_ANTI}[how]
    pi, bi = t.probe(dev(pk), code)
    li, ri = R.join_indices(pk, bk, how)
    if ri is None:
        assert sorted(host(pi).tolist()) == li.tolist()
    else:
        got = sorted(zip(host(pi).tolist(), host(bi).tolist()))
        assert got == sorted(zip(li.tolist(), ri.tolist()))
    t.check_flags()


def test_gather_handles_no_match(qb):
    src = dev(np.arange(10, dtype=np.float64) + 0.5)
    idx = dev(np.array([3, -1, 9, 0], dtype=np.int32))
    assert host(qb.ops.gather([src], idx)[0]).tolist() == [3.5, 0.0, 9.5, 0.5]


# ------------------------------------------------------------------ K7 as-of
@pytest.mark.parametrize("tag", ["0", "1", "2"])
def test_asof_golden(qb, golden_dir, tag):
    g = np.load(os.path.join(golden_dir, f"asof{tag}.npz"))
    n_by = int(max(g["t_sym"].max(), g["q_sym"].max())) + 1
    r = host(qb.ops.asof_backward(dev(g["t_time"]), dev(g["t_sym"]), dev(g["q_time"]), dev(g["q_sym"]), n_by))
    assert np.array_equal(r, g["ridx"])                               # apps/time-series/asof_join.py:6-18
    assert int((r >= 0).sum()) == int(g["n_matched"])


@pytest.mark.parametrize("nt,nq,nsym,span", [
    (0, 0, 5, 10), (0, 1000, 5, 100), (1000, 0, 5, 100), (1, 1, 1, 1), (1023, 1, 3, 50), (1, 1023, 3, 50), (1025, 1024, 7, 300),
    (5000, 20_000, 3, 400),            # 3 keys, heavy ties: nearly every left row has right rows of its key in its window, before AND after it
    (40_000, 200_000, 8000, 10**9),    # the benchmark's shape: 8000 keys, few in-window matches
    (200_000, 40_000, 200, 10**6), (70_001, 333_333, 40, 5000), (300_000, 300_000, 1, 10**5)])
def test_asof_merge_kernel(qb, nt, nq, nsym, span):
    """qk_asof_merge (csrc/asof.cu: windows of 1024 merged rows, a CTA per chunk, table in shared memory) against the oracle's
    per-key binary search, bit-exact: ties (right rows first, the LAST equal right row wins), windows that are all left or all
    right rows, keys outside [0, n_by) on either side (no match / ignored), and the STREAMING form -- the right side fed in
    batches with carry_in / carry_out / r_base -- which must give the same rows as one call."""
    rng = np.random.default_rng(nt * 31 + nq)
    lt = np.sort(rng.integers(0, span, nt)).astype(np.int64)
    rt = np.sort(rng.integers(0, span, nq)).astype(np.int64)
    lb = rng.integers(0, nsym, nt).astype(np.int32)
    rb = rng.integers(0, nsym, nq).astype(np.int32)
    exp = R.asof_backward(lt, lb, rt, rb)
    out, carry = qb.ops.asof_merge(dev(lt), dev(lb), dev(rt), dev(rb), nsym, want_carry=True)
    assert np.array_equal(host(out), exp)
    last = np.full(nsym, -1, dtype=np.int64)
    last[rb] = np.arange(nq)                                             # later rows overwrite: the newest right row of each key
    assert np.array_equal(host(carry), last)
    if nt and nq:
        # keys outside the table: such left rows get -1, such right rows are never a match
        lb2, rb2 = lb.copy(), rb.copy()
        lb2[::7] = nsym + 3; rb2[::5] = -2; lb2[3::11] = -1
        ok_r = rb2 >= 0
        sub = np.nonzero(ok_r)[0]
        e2 = R.asof_backward(lt, lb2, rt[ok_r], rb2[ok_r])
        e2 = np.where(e2 >= 0, sub[np.maximum(e2, 0)], -1) if len(sub) else np.full(nt, -1, dtype=np.int64)
        e2[(lb2 < 0) | (lb2 >= nsym)] = -1
        out2, _ = qb.ops.asof_merge(dev(lt), dev(lb2), dev(rt), dev(rb2), nsym)
        assert np.array_equal(host(out2), e2)
        # streaming: right rows in 3 batches cut at times, left rows up to each cut joined against (carry, batch)
        cuts = [int(rt[nq // 3]), int(rt[2 * nq // 3]), span + 1]
        carry_t, base, lpos, got = None, 0, 0, []
        for c in cuts:
            r_hi = int(np.searchsorted(rt, c, side="left"))              # right rows with time < c
            l_hi = int(np.searchsorted(lt, c, side="left"))
            o, carry_t = qb.ops.asof_merge(dev(lt[lpos:l_hi]), dev(lb[lpos:l_hi]), dev(rt[base:r_hi]), dev(rb[base:r_hi]), nsym,
                                           carry_in=carry_t, r_base=base, want_carry=True)
            got.append(host(o))
            base, lpos = r_hi, l_hi
        assert np.array_equal(np.concatenate(got), exp)


def test_asof_synthetic_ticks(qb):
    nt, nq, nsym = 60_000, 300_000, 500
    tr = G.gen_ticks(G.T_TRADES, nt, nsym, mean_gap_ns=5000)
    qu = G.gen_ticks(G.T_QUOTES, nq, nsym, mean_gap_ns=1000)
    r = host(qb.ops.asof_backward(dev(tr["time"]), dev(tr["symbol"]), dev(qu["time"]), dev(qu["symbol"]), nsym))
    exp = R.asof_backward(tr["time"], tr["symbol"], qu["time"], qu["symbol"])
    assert np.array_equal(r, exp)
    ridx, n_matched, checksum = Q.asof_checksum(tr, qu)
    asize = host(qb.ops.gather([dev(qu["asize"])], dev(r.astype(np.int32)))[0])
    m = r >= 0
    assert int(m.sum()) == n_matched
    assert int(np.rint(asize[m].astype(np.float64) * 100.0).sum()) == checksum


# ------------------------------------------------------------------ K8 top-k
@pytest.mark.parametrize("n,k,desc", [(5, 10, True), (1000, 10, True), (100_000, 10, True), (100_000, 100, False)])
def test_topk_candidates(qb, n, k, desc):
    rng = np.random.default_rng(n)
    v = np.round(rng.normal(size=n) * 1000, 1)         # ties exist
    idx = host(qb.ops.topk_candidates(dev(v), k, desc))
    order = np.argsort(-v if desc else v, kind="stable")
    kth = v[order[min(k, n) - 1]]
    exp = np.nonzero(v >= kth if desc else v <= kth)[0]
    assert sorted(idx.tolist()) == exp.tolist()
    for arr, dt in ((np.arange(n, dtype=np.int64) * 7 % 1013 - 500, np.int64), (rng.integers(8000, 10500, n).astype(np.int32), np.int32)):
        idx = host(qb.ops.topk_candidates(dev(arr), k, desc))
        o = np.sort(arr)[::-1] if desc else np.sort(arr)
        kth = o[min(k, n) - 1]
        assert sorted(idx.tolist()) == np.nonzero(arr >= kth if desc else arr <= kth)[0].tolist()


# ------------------------------------------------------------------ error behaviour at the C-ABI
def test_errors_are_loud(qb):
    with pytest.raises(qb.L.QkError):
        qb.ops.scan_filter_project([torch.zeros(4, dtype=torch.float64)], None, [[(qb.L.OP_COL, 0, 0, 0.0, 0)]])   # CPU tensor
    d = dev(np.zeros(8))
    with pytest.raises(qb.L.QkError, match="column slot"):
        qb.ops.scan_filter_project([d], None, [[(qb.L.OP_COL, 3, 0, 0.0, 0)]])
    with pytest.raises(qb.L.QkError, match="stack underflow"):
        qb.ops.scan_filter_project([d], [(qb.L.OP_ADD, 0, 0, 0.0, 0)], [[(qb.L.OP_COL, 0, 0, 0.0, 0)]])
    with pytest.raises(qb.L.QkError, match="integer"):
        qb.ops.partition_plan(d, 4)


# ------------------------------------------------------------------ K1 fast path: TMA-staged filter + compaction
@pytest.mark.parametrize("n", [0, 1, 255, 2303, 2304, 2305, 100_000, 1_000_003])
@pytest.mark.parametrize("pred_sql,cols", [
    ("l_shipdate > date '1995-03-15'", ["l_orderkey", "l_extendedprice", "l_discount"]),
    ("l_returnflag = 'R'", ["l_orderkey", "l_returnflag", "l_shipdate"]),
    ("l_orderkey >= 1000000", ["l_orderkey"]),
    ("l_linestatus != 'F'", ["l_linestatus", "l_tax", "l_shipdate", "l_orderkey", "l_quantity"]),
    (None, ["l_shipdate", "l_returnflag"]),
])
def test_filter_compact_tma(qb, n, pred_sql, cols):
    names = ["l_orderkey", "l_shipdate", "l_extendedprice", "l_discount", "l_returnflag", "l_linestatus", "l_tax", "l_quantity"]
    li = G.gen_lineitem(1, 3_000_000, 3_000_000 + n, names)
    d = {k: dev(v) for k, v in li.items()}
    sch = _schema(qb, d, {"l_returnflag": G.RETURNFLAG_DICT, "l_linestatus": G.LINESTATUS_DICT})
    pred = qb.E.compile_expr(qb.E.parse(pred_sql), sch) if pred_sql else None
    outs, m = qb.ops.scan_filter_project(list(d.values()), pred, [qb.E.compile_expr(qb.E.parse(c), sch) for c in cols])
    if n > 0:
        assert qb.ops.last_variant() == "compact_tma"
    mask = {"l_shipdate > date '1995-03-15'": li["l_shipdate"] > G.DAY_1995_03_15, "l_returnflag = 'R'": li["l_returnflag"] == 2,
            "l_orderkey >= 1000000": li["l_orderkey"] >= 1000000, "l_linestatus != 'F'": li["l_linestatus"] != 0,
            None: np.ones(n, bool)}[pred_sql]
    assert m == int(mask.sum())
    got = [host(o) for o in outs]
    exp = [li[c][mask] for c in cols]
    for g, e in zip(got, exp):                      # stable: input row order is preserved, bit-exact
        assert np.array_equal(g, e)
    for g, e in zip(got, exp):
        assert g.dtype == e.dtype


# ------------------------------------------------------------------ semi-join reduction (Bloom) fused into the scan
@pytest.mark.parametrize("nparts", [1, 2, 8])
@pytest.mark.parametrize("n_probe,n_build", [(1000, 0), (300_000, 20_000), (1_000_003, 150_000)])
def test_bloom_semijoin_scan(qb, nparts, n_probe, n_build):
    li = G.gen_lineitem(1, 0, n_probe, ["l_orderkey", "l_shipdate", "l_extendedprice"])
    od = G.gen_orders(1, 0, n_build, ["o_orderkey"])
    d = {k: dev(v) for k, v in li.items()}
    sch = _schema(qb, d)
    words = qb.ops.Bloom.words_for(max(1, n_build // nparts + 1))
    bf = qb.ops.Bloom.build(dev(od["o_orderkey"]) if n_build else None, words, nparts, "cuda")
    pred = qb.E.compile_expr(qb.E.parse("l_shipdate > date '1995-03-15'"), sch)
    projs = [qb.E.compile_expr(qb.E.parse(c), sch) for c in ("l_extendedprice", "l_orderkey")]
    outs, m = qb.ops.scan_filter_project(list(d.values()), pred, projs, bloom=(bf, 1))
    assert qb.ops.last_variant() == "compact_tma+bloom"
    mask = li["l_shipdate"] > G.DAY_1995_03_15
    member = np.isin(li["l_orderkey"], od["o_orderkey"])
    got_keys, got_price = host(outs[1]), host(outs[0])
    must = mask & member
    # no false negatives, stable order, survivors are a subset of the predicate's rows
    surv = np.zeros(n_probe, bool)
    pos = np.nonzero(mask)[0]
    exp_all = li["l_orderkey"][mask]
    j = 0
    idx = []
    for k in got_keys.tolist():                      # survivors appear in input order: walk both lists
        while exp_all[j] != k:
            j += 1
        idx.append(pos[j]); j += 1
    surv[idx] = True
    assert np.array_equal(got_price, li["l_extendedprice"][surv])
    assert not np.any(must & ~surv), "Bloom filter lost a joining row"
    fp = int((surv & ~member).sum())
    assert fp <= 0.05 * max(1, int(mask.sum())) + 5, f"false-positive rate too high: {fp} of {int(mask.sum())}"
