"""OrderedStream.pattern_recognize without a GPU: the brute-force oracle of tests/pattern_cases.py against hand-worked cases, the
kernel's search (as restated by tests/pattern_shim.py) against the oracle, the split of event predicates and the link compiler,
and the API cases through the planner and executors on the shim."""
import datetime

import numpy as np
import pyarrow as pa
import pytest
import torch

import cpu_shim
import pattern_cases as P
import pattern_shim
from quokka_b200 import _lib as L
from quokka_b200 import expr as E


def _t(times, vals, keys=None):
    n = len(times)
    return pa.table({"t": np.array(times, np.int64), "k": np.array(keys if keys is not None else [0] * n, np.int64),
                     "v": np.array(vals, np.float64)})


# ------------------------------------------------------------------ the oracle, by hand
def test_oracle_hand_worked():
    t = _t([1, 2, 3, 4, 6], [5, 1, 7, 1, 9])
    # starts at v > 4: t=1 (b at 2, c at 3), t=3 (b at 4, c at 6), t=6 (no later rows)
    assert P.pattern_recognize(t, "t", [("a", "v > 4"), ("b", "v < 2"), ("c", "v > 4")], 10, "k") == [(0, 1, 2, 3), (0, 3, 4, 6)]
    # maxspan 2 closes the span at t0 + 2: only the first start still completes
    assert P.pattern_recognize(t, "t", [("a", "v > 4"), ("b", "v < 2"), ("c", "v > 4")], 2, "k") == [(0, 1, 2, 3)]
    # a link: c must exceed a; from t=1 (v=5) that is t=3 (7); from t=3 (v=7) it is t=6 (9)
    assert P.pattern_recognize(t, "t", [("a", "v > 4"), ("b", "v < 2"), ("c", "c.v > a.v")], 10, "k") == [(0, 1, 2, 3), (0, 3, 4, 6)]
    # rows between bound rows are skipped freely; the smallest (t1, t2) wins, not the first b
    t2 = _t([0, 1, 2, 3, 4], [0, 3, 1, 2, 9])
    assert P.pattern_recognize(t2, "t", [("a", "v = 0"), ("b", "v > 0"), ("c", "c.v > b.v + 5")], 10, "k") == [(0, 0, 1, 4)]
    # keys are independent; a start row never binds a later event
    t3 = _t([0, 0, 1, 1], [1, 1, 1, 1], keys=[0, 1, 0, 1])
    assert P.pattern_recognize(t3, "t", [("a", None), ("b", "v = 1")], 5, "k") == [(0, 0, 1), (1, 0, 1)]
    # equal times never chain
    assert P.pattern_recognize(_t([0, 0], [1, 1]), "t", [("a", None), ("b", None)], 5, "k") == []


def test_oracle_lexicographic_rule():
    # two tied b rows: the smaller completion wins whichever row comes first
    t = _t([1, 1, 2, 2, 5, 9], [1, 2, 10, 20, 15, 25])
    ev = [("a", "v = 1"), ("b", "v >= 2"), ("c", "c.v > b.v")]
    assert P.pattern_recognize(t, "t", ev, 100, "k") == [(0, 1, 2, 5)]
    assert P.pattern_recognize(t.take(pa.array([0, 1, 3, 2, 4, 5])), "t", ev, 100, "k") == [(0, 1, 2, 5)]
    # the cap path: a tied b binds c earlier than the best's c, after which d may lie beyond the best's d
    t = _t(P.CAP_TABLE["t"], P.CAP_TABLE["v"])
    assert P.pattern_recognize(t, "t", P.CAP_EVENTS, 20, "k") == [(0, 1, 2, 3, 12)]


def test_oracle_nulls():
    t = pa.table({"t": np.array([0, 1, 2], np.int64), "k": np.zeros(3, np.int64), "v": pa.array([1.0, None, 3.0])})
    assert P.pattern_recognize(t, "t", [("a", None), ("b", "v > 0 or v < 0")], 5, "k") == [(0, 0, 2), (0, 1, 2)]
    # a NULL in the row bound to a makes b's link false: the start at t=1 has no match
    assert P.pattern_recognize(t, "t", [("a", None), ("b", "v > a.v - 100")], 5, "k") == [(0, 0, 2)]


# ------------------------------------------------------------------ the search against the oracle
def _search(tab, time_col, events, maxspan, by, budget=1 << 30):
    return P.search(pattern_shim.pattern_search, tab, time_col, events, maxspan, by, budget)


@pytest.mark.parametrize("m", [2, 3, 4, 5])
@pytest.mark.parametrize("seed", range(12))
def test_search_against_oracle(m, seed):
    nulls = seed % 3 == 0
    tab = P.random_stream(seed * 7 + m, n=45 if m < 5 else 30, keys=2 + seed % 3, tmax=25, nulls=nulls)
    ev = P.random_events(seed * 13 + m, m)
    for span in (0, 3, 8, 30):
        assert _search(tab, "time", ev, span, "sym") == P.pattern_recognize(tab, "time", ev, span, "sym"), (ev, span)


def test_search_lexicographic_rule():
    """The search on the two hand-worked tie cases, in both row orders."""
    t = _t([1, 1, 2, 2, 5, 9], [1, 2, 10, 20, 15, 25])
    ev = [("a", "v = 1"), ("b", "v >= 2"), ("c", "c.v > b.v")]
    for tab in (t, t.take(pa.array([0, 1, 3, 2, 4, 5]))):
        assert _search(tab, "t", ev, 100, "k") == [(0, 1, 2, 5)]
    t = _t(P.CAP_TABLE["t"], P.CAP_TABLE["v"])
    for tab in (t, t.take(pa.array([0, 2, 1, 3, 4, 5, 6]))):
        assert _search(tab, "t", P.CAP_EVENTS, 20, "k") == [(0, 1, 2, 3, 12)]


@pytest.mark.parametrize("m", [3, 4, 5])
def test_search_against_oracle_dense_ties(m):
    """Many rows per timestamp and chained link programs, so that tied rows lead to different completions: the caps of the
    best match, and when they are lifted, decide the answer."""
    for seed in range(100):
        tab = P.tie_stream(seed * 5 + m)
        ev = P.tie_events(seed * 11 + m, m)
        for span in (3, 10):
            assert _search(tab, "time", ev, span, "sym") == P.pattern_recognize(tab, "time", ev, span, "sym"), (seed, ev, span)


def test_pruning_keeps_row_local_patterns_linear():
    """A row-local-only pattern whose middle event matches everywhere and whose last never does: with the rule that a level no
    later program reads ends with its first binding, every start tests each row of its span about once."""
    n = 300
    tab = pa.table({"t": np.arange(n, dtype=np.int64), "k": np.zeros(n, np.int64), "v": np.ones(n)})
    ev = [("a", "v = 1"), ("b", "v = 1"), ("c", "v = 1"), ("d", "v = 2")]
    assert _search(tab, "t", ev, 50, "k", budget=3 * 51) == []
    with pytest.raises(L.QkError, match="tested more than"):
        _search(tab, "t", [("a", "v = 1"), ("b", "v = 1"), ("c", "c.v >= b.v"), ("d", "d.v = 2 + 0 * c.v")], 50, "k", budget=3 * 51)


# ------------------------------------------------------------------ predicate split and link compilation
SCHEMA = ["t", "k", "px", "sz", "sym"]


def test_split_pattern():
    p = E.split_pattern([("a", "px > 1 and a.sz < 3"), ("b", "b.px > a.px and sz = 2"), ("c", None if False else "px < b.px * a.px")],
                        SCHEMA, "k")
    assert p.names == ["a", "b", "c"]
    assert p.local[0].sql() == "((px > 1) and (sz < 3))" and p.link[0] is None
    assert p.local[1].sql() == "(sz = 2)" and p.link[1].sql() == "(px > a.px)"
    assert p.local[2] is None and p.link[2].sql() == "(px < (b.px * a.px))"
    assert p.columns == {"px", "sz"}
    assert E.pattern_prefilter(p) is None                                        # c has no row-local part
    q = E.split_pattern([("a", "px > 5"), ("b", "px < 1 and b.px > a.px"), ("c", "px > 5")], SCHEMA, "k")
    assert E.pattern_prefilter(q).sql() == "(((px > 5) or (px < 1)) or (px > 5))"
    r = E.split_pattern([("a", "px > 5"), ("b", "sz < 1")], SCHEMA, "k")
    assert E.pattern_prefilter(r) is None                                        # different columns: a NULL would drop rows


@pytest.mark.parametrize("events,msg", [
    ([("a", "px > b.px"), ("b", "px > 1")], "later event"),
    ([("a", "px > 1"), ("b", "px > z.px")], "names no event"),
    ([("a", "px > 1"), ("a", "px > 2")], "used for two events"),
    ([("a", "px > 1"), ("b", "nope > 2")], "unknown column"),
    ([("a", "px > 1"), ("b", "a.nope > 2")], "unknown column"),
    ([("a", "px > 1"), ("b", None)], "only the first event"),
    ([("a.x", "px > 1"), ("b", "px > 2")], "identifier"),
    ([("k", "px > 1"), ("b", "px > 2")], "`by` column"),
    ([("a", "px > 1")], "2 to 8"),
    ([(c, "px > 1") for c in "abcdefghi"], "2 to 8"),
])
def test_split_rejects(events, msg):
    with pytest.raises(E.ExprError, match=msg):
        E.split_pattern(events, SCHEMA, "k")


def test_compile_link():
    sch = {"px": E.ColumnInfo(0, L.QK_F64), "sz": E.ColumnInfo(1, L.QK_I64), "sym": E.ColumnInfo(2, L.QK_I32, ["x", "y"])}
    names = ["a", "b", "c"]
    slots = {"px": 0, "sz": 1, "sym": 2}
    p = E.split_pattern([("a", "px > 0"), ("b", "b.px > a.px * 1.005"), ("c", "case when a.sz > 1 then -px else px end <= b.px")],
                        ["px", "sz", "sym"], "k")
    assert E.compile_link(p.link[1], 1, names, slots, sch) == [(L.OP_COL, 0, 1, 0.0, 0), (L.OP_COL, 0, 0, 0.0, 0), (L.OP_CONST, 0, 0, 1.005, 0),
                                                            (L.OP_MUL, 0, 0, 0.0, 0), (L.OP_GT, 0, 0, 0.0, 0)]
    prog = E.compile_link(p.link[2], 2, names, slots, sch)
    assert [x[0] for x in prog] == [L.OP_COL, L.OP_CONST, L.OP_GT, L.OP_COL, L.OP_NEG, L.OP_COL, L.OP_SELECT, L.OP_COL, L.OP_LE]
    assert prog[0][2] == 0 and prog[3][2] == 2 and prog[7][2] == 1
    bad = E.split_pattern([("a", "px > 0"), ("b", "sym = a.sym")], ["px", "sym"], "k")
    with pytest.raises(E.ExprError, match="string column"):
        E.compile_link(bad.link[1], 1, ["a", "b"], slots, sch)
    bad = E.split_pattern([("a", "px > 0"), ("b", "px in (1, a.px)")], ["px"], "k")
    with pytest.raises(E.ExprError, match="not supported"):
        E.compile_link(bad.link[1], 1, ["a", "b"], slots, sch)
    deep = " + ".join(f"a.px * {i}" for i in range(30))
    bad = E.split_pattern([("a", "px > 0"), ("b", f"px > {deep}")], ["px"], "k")
    with pytest.raises(E.ExprError):
        E.compile_link(bad.link[1], 1, ["a", "b"], slots, sch)


def test_link_errors_while_the_plan_is_built(monkeypatch):
    """Ops outside the link subset and programs over the kernel's limits fail when pattern_recognize is called, before any row is
    read; a string column read across events (its type is known only when rows arrive) fails when the search runs."""
    cpu_shim.install(monkeypatch)
    from quokka_b200.df import QuokkaContext
    qc = QuokkaContext()
    tab = pa.table({"t": np.arange(4, dtype=np.int64), "k": np.zeros(4, np.int64), "v": np.arange(4.0), "s": ["x", "y", "x", "y"]})
    s = qc.from_arrow_sorted(tab, "t")
    with pytest.raises(E.ExprError, match="not supported"):
        s.pattern_recognize("t", [("a", None), ("b", "v in (1, a.v)")], 5, "k")
    big = " and ".join(f"v > a.v + {i}" for i in range(8))             # 47 nodes per event: 141 over three events
    with pytest.raises(E.ExprError, match="nodes; at most 128"):
        s.pattern_recognize("t", [("a", None), ("b", big), ("c", big.replace("a.v", "b.v")), ("d", big.replace("a.v", "c.v"))], 5, "k")
    r = s.pattern_recognize("t", [("a", None), ("b", "s = a.s")], 5, "k")
    with pytest.raises(E.ExprError, match="string column"):
        r.collect()


def test_maxspan_and_by_arguments(monkeypatch):
    cpu_shim.install(monkeypatch)
    from quokka_b200.df import QuokkaContext
    qc = QuokkaContext()
    s = qc.from_arrow_sorted(_t([0, 1], [1, 2]), "t")
    with pytest.raises(E.ExprError, match="maxspan"):
        s.pattern_recognize("t", [("a", None), ("b", None)], -1, "k")
    with pytest.raises(E.ExprError, match="maxspan"):
        s.pattern_recognize("t", [("a", None), ("b", None)], 1.5, "k")
    with pytest.raises(Exception, match="by column"):
        s.pattern_recognize("t", [("a", None), ("b", None)], 1, None)
    with pytest.raises(AssertionError):
        s.pattern_recognize("v", [("a", None), ("b", None)], 1, "k")


def test_explain_and_prefilter_pushdown(monkeypatch, capsys):
    cpu_shim.install(monkeypatch)
    from quokka_b200.df import QuokkaContext
    qc = QuokkaContext()
    s = qc.from_arrow_sorted(_t([0, 1], [1, 2]), "t").pattern_recognize("t", [("a", "v > 1"), ("b", "v < 0 and b.v < a.v")], 5, "k")
    assert s.schema == ["k", "a", "b"] and s.sorted_by == "a"
    s.explain()
    out = capsys.readouterr().out
    assert "pattern_recognize [a: (v > 1), b: (v < 0) and (v < a.v)] maxspan=5 by=k" in out
    assert "filter ((v > 1) or (v < 0))" in out


# ------------------------------------------------------------------ the API on the shim
@pytest.fixture
def qc(monkeypatch):
    cpu_shim.install(monkeypatch)
    from quokka_b200.df import QuokkaContext
    return QuokkaContext()


@pytest.mark.parametrize("case", P.API_CASES + P.SINGLE_RANK_CASES, ids=lambda c: c.__name__)
def test_api_case(qc, case):
    case(qc)


def test_timedelta_on_date_column(qc):
    d = pa.array(np.array([0, 1, 3, 10], np.int32), pa.int32()).cast(pa.date32())
    t = pa.table({"d": d, "k": np.zeros(4, np.int64), "v": np.array([1.0, 2.0, 3.0, 4.0])})
    got = P.check(qc, t, "d", [("a", "v = 1"), ("b", "v > 2")], datetime.timedelta(days=3), "k")
    assert got == [(0, 0, 3)]
