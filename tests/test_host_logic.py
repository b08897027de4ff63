"""Host-side units that need neither a GPU nor the kernel shim: the SQL-subset parser / compiler, the edge-op
algebra, predicate push-down, aggregate decomposition, column / dictionary plumbing and the readers' lineage."""
import datetime

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest
import torch

from quokka_b200 import _lib as L
from quokka_b200 import expr as E
from quokka_b200.columns import DeviceColumn, DeviceTable, DictionaryRegistry, concat_tables, unify_dictionaries
from quokka_b200.datastream import (DataStream, FilterNode, JoinNode, MapNode, SourceNode, decompose_aggs, push_filters)
from quokka_b200.dataset import InputArrowDataset, InputParquetDataset, InputSortedParquetDataset
from quokka_b200.edge import EdgeOps


def days(s):
    return (datetime.date.fromisoformat(s) - datetime.date(1970, 1, 1)).days


def test_parser_folds_dates_and_intervals():
    assert E.parse("d <= date '1998-12-01' - interval '90' day").sql() == "(d <= date '1998-09-02')"       # tpch.py:108
    assert E.parse("d < date '1994-01-01' + interval '1' year").args[1].value == days("1995-01-01")          # tpch.py:230
    assert E.parse("d < date '1993-07-01' + interval '3' month").args[1].value == days("1993-10-01")
    assert E.parse("d < date '2000-01-31' + interval '1' month").args[1].value == days("2000-02-29")         # clamped
    assert E.parse("x between 0.06 - 0.01 and 0.06 + 0.01").sql() == "((x >= 0.049999999999999996) and (x <= 0.06999999999999999))"
    assert E.parse("a in (1, 2)").sql() == "(a in (1, 2))"
    assert E.parse(E.parse("not a in (1, 2)").sql()) == E.parse("a not in (1, 2)")            # the SQL text round-trips
    assert E.parse("a not in (1, 2)").kind == "un"
    assert E.parse("r_name == 'ASIA'").sql() == "(r_name = 'ASIA')"
    assert E.parse("-3 * 2").value == -6
    with pytest.raises(E.ExprError):
        E.parse("a +")
    with pytest.raises(E.ExprError):
        E.parse("a ; drop")


def test_compiler_emits_exact_integer_compares_and_resolves_strings():
    sch = {"d": E.ColumnInfo(0, L.QK_I32, None, True), "k": E.ColumnInfo(1, L.QK_I64), "x": E.ColumnInfo(2, L.QK_F64),
           "s": E.ColumnInfo(3, L.QK_U8, ["AUTOMOBILE", "BUILDING"]), "k2": E.ColumnInfo(4, L.QK_I64)}
    assert E.compile_expr(E.parse("d > date '1995-03-15'"), sch) == [(L.OP_CMP_COL_IMM, 0, L.CMP_GT, 0.0, 9204)]
    assert E.compile_expr(E.parse("9204 < d"), sch) == [(L.OP_CMP_COL_IMM, 0, L.CMP_GT, 0.0, 9204)]         # flipped
    assert E.compile_expr(E.parse("s = 'BUILDING'"), sch) == [(L.OP_CMP_COL_IMM, 3, L.CMP_EQ, 0.0, 1)]
    assert E.compile_expr(E.parse("s = 'NOPE'"), sch) == [(L.OP_CMP_COL_IMM, 3, L.CMP_EQ, 0.0, -1)]        # matches nothing
    # range terms on ONE integer column fold into one closed-range node: the scan keeps its compaction fast path (and Bloom filter)
    assert E.compile_expr(E.parse("d >= date '1994-01-01' and d < date '1994-01-01' + interval '1' year"), sch) == [(L.OP_RANGE_COL_IMM, 0, 0, 9130.0, 8766)]
    assert E.compile_expr(E.parse("d between date '1995-01-01' and date '1996-12-31'"), sch) == [(L.OP_RANGE_COL_IMM, 0, 0, 9861.0, 9131)]
    assert E.compile_expr(E.parse("d > 5 and d <= 9 and d < 8"), sch) == [(L.OP_RANGE_COL_IMM, 0, 0, 7.0, 6)]
    assert E.compile_expr(E.parse("d > 9 and d < 3"), sch) == [(L.OP_RANGE_COL_IMM, 0, 0, 0.0, 1)]                   # empty
    assert [p[0] for p in E.compile_expr(E.parse("d > 5 or d < 3"), sch)] == [L.OP_CMP_COL_IMM, L.OP_CMP_COL_IMM, L.OP_OR]
    assert [p[0] for p in E.compile_expr(E.parse("d > 5 and k < 3"), sch)] == [L.OP_CMP_COL_IMM, L.OP_CMP_COL_IMM, L.OP_AND]      # two columns
    assert E.compile_expr(E.parse("k = k2"), sch) == [(L.OP_CMP_COL_COL, 1, L.CMP_EQ | (4 << 8), 0.0, 0)]   # Q5 post-join predicate
    prog = E.compile_expr(E.parse("x * (1 - x) > 0.5"), sch)
    assert [p[0] for p in prog] == [L.OP_COL, L.OP_CONST, L.OP_COL, L.OP_SUB, L.OP_MUL, L.OP_CONST, L.OP_GT]
    assert E.compile_expr(E.parse("cast(x * 100 as int)"), sch)[-1][0] == L.OP_RINT
    with pytest.raises(E.ExprError, match="unknown column"):
        E.compile_expr(E.parse("zzz > 1"), sch)
    with pytest.raises(E.ExprError, match="dictionary"):
        E.compile_expr(E.parse("x = 'a'"), sch)


def test_case_like_extract_and_booleans():
    """The rest of sql_utils.evaluate's node set (pyquokka/sql_utils.py:131-149 LIKE, :161-168 CASE, :204-211 EXTRACT)."""
    sch = {"a": E.ColumnInfo(0, L.QK_I64), "b": E.ColumnInfo(1, L.QK_F64), "d": E.ColumnInfo(2, L.QK_I32, None, True),
           "s": E.ColumnInfo(3, L.QK_I32, ["PROMO BRUSHED", "STANDARD", "PROMO X", "ECONOMY PROMO", "A.C"])}
    # every new construct prints as SQL that parses back to the same tree (aggregate decomposition goes through text)
    for t in ("case when a > 1 then b * 2 when a < 0 then 0 else 7 end", "s like 'PROMO%' or cast(b as int) = 3",
              "sum(case when s like '%PROMO' then b else 0 end)", "extract(month from d)", "not s like 'A_C'"):
        n = E.parse(t)
        assert E.parse(n.sql()) == n, t
    # EXTRACT(year) in a comparison folds to a date range (which row-group statistics can prune on)
    assert E.parse("extract(year from d) = 1995").sql() == "((d >= date '1995-01-01') and (d < date '1996-01-01'))"
    assert E.parse("1996 > extract(year from d)").sql() == "(d < date '1996-01-01')"
    assert E.parse("extract(year from d) >= 1995 and extract(year from d) <= 1996").sql() == \
        "((d >= date '1995-01-01') and (d < date '1997-01-01'))"
    assert E.parse("extract(year from d) != 1995").sql() == "((d < date '1995-01-01') or (d >= date '1996-01-01'))"
    # EXTRACT as a value: one unary node on the days-since-epoch value (year / month / day of month)
    prog = E.compile_expr(E.parse("extract(month from d) = 3"), sch)
    assert [p[0] for p in prog] == [L.OP_COL, L.OP_EXTRACT, L.OP_CONST, L.OP_EQ] and prog[1][2] == 1
    import cpu_shim as _shim
    days = np.array([0, 58, 59, 365, 11016, 19782, -1, -366], dtype=np.int32)      # 1970-01-01, 02-28, 03-01, 1971-01-01, 2000-02-29, 2024-02-29, 1969-12-31, 1968-12-31
    for part, exp in (("year", [1970, 1970, 1970, 1971, 2000, 2024, 1969, 1968]), ("month", [1, 2, 3, 1, 2, 2, 12, 12]), ("day", [1, 28, 1, 1, 29, 29, 31, 31])):
        got = _shim.eval_prog(E.compile_expr(E.parse(f"extract({part} from d)"), sch), [None, None, days, None], len(days))
        assert got.tolist() == exp, part
    # CASE = cond then else SELECT: the condition is compiled (and evaluated) once
    prog = E.compile_expr(E.parse("case when a > 1 then b * 2 else 0 end"), sch)
    assert [p[0] for p in prog] == [L.OP_CMP_COL_IMM, L.OP_COL, L.OP_CONST, L.OP_MUL, L.OP_CONST, L.OP_SELECT]
    with pytest.raises(E.ExprError, match="ELSE"):
        E.parse("case when a > 1 then 2 end")
    # LIKE is resolved against the dictionary on the host: % and _ wildcards, regex metacharacters are literals
    def codes(pat):
        prog = E.compile_expr(E.parse(f"s like '{pat}'"), sch)
        assert len(prog) == 1                       # ONE node whatever the number of matching dictionary values
        op, slot, a1, _, imm_i = prog[0]
        if op == L.OP_CMP_COL_IMM:
            return [imm_i]
        assert op == L.OP_IN_SET and slot == 3 and imm_i >> a1 == 0
        return [c for c in range(a1) if (imm_i >> c) & 1]
    assert codes("PROMO%") == [0, 2] and codes("%PROMO") == [3] and codes("%PROMO%") == [0, 2, 3] and codes("STANDARD") == [1]
    assert codes("PROMO _") == [2] and codes("A.C") == [4] and codes("A_C") == [4] and codes("AxC") == [-1] and codes("%") == [0, 1, 2, 3, 4]
    with pytest.raises(E.ExprError, match="dictionary"):
        E.compile_expr(E.parse("b like 'x%'"), sch)
    assert E.compile_expr(E.parse("true"), sch) == [(L.OP_CONST, 0, 0, 1.0, 0)] and E.parse("false").value == 0
    # Q14's shape at TPC-H size: 25 of 150 p_type values match 'PROMO%' -- still one node, inside the kernel's limits
    # (round 1 expanded this to 108 nodes, which the device library refuses)
    types = [f"{a} {b} {c}" for a in ("STANDARD", "SMALL", "MEDIUM", "LARGE", "ECONOMY", "PROMO")
             for b in ("ANODIZED", "BURNISHED", "PLATED", "POLISHED", "BRUSHED") for c in ("TIN", "NICKEL", "BRASS", "STEEL", "COPPER")]
    sch2 = {"p_type": E.ColumnInfo(0, L.QK_U8, types), "x": E.ColumnInfo(1, L.QK_F64), "y": E.ColumnInfo(2, L.QK_F64)}
    q14 = E.compile_expr(E.parse("case when p_type like 'PROMO%' then x * (1 - y) else 0 end"), sch2)
    assert len(q14) == 8 and q14[0][0] == L.OP_IN_SET and q14[0][2] == 150 and bin(q14[0][4]).count("1") == 25
    E.check_call(3, None, [q14, q14], "test")
    # IN over strings / small integers is the same single node; other IN lists stay an OR-chain of exact compares
    assert [p[0] for p in E.compile_expr(E.parse("s in ('STANDARD', 'A.C', 'nope')"), sch)] == [L.OP_IN_SET]
    assert [p[0] for p in E.compile_expr(E.parse("a in (1, 5, 9)"), sch)] == [L.OP_IN_SET]
    assert [p[0] for p in E.compile_expr(E.parse("a in (-1, 5)"), sch)] == [L.OP_CMP_COL_IMM, L.OP_CMP_COL_IMM, L.OP_OR]
    # programs the kernels would refuse fail on the host, in the compiler (48 nodes / 8 stack slots) ...
    with pytest.raises(E.ExprError, match="at most 48"):
        E.compile_expr(E.parse(" + ".join(["b"] * 30)), sch)
    with pytest.raises(E.ExprError, match="stack"):
        E.compile_expr(E.parse("b" + " + (b" * 9 + ")" * 9), sch)
    # ... and per call (112 nodes in total, 16 columns, 16 expressions)
    long = E.compile_expr(E.parse(" + ".join(["b"] * 20)), sch)
    with pytest.raises(E.ExprError, match="in total"):
        E.check_call(4, long, [long, long], "test")
    with pytest.raises(E.ExprError, match="input columns"):
        E.check_call(17, None, [], "test")
    # the interpreter shim agrees with numpy on CASE
    import cpu_shim
    cols = [np.array([0, 2, 5, -1]), np.array([1.5, 2.5, -3.0, 4.0]), np.zeros(4, np.int32), np.zeros(4, np.int32)]
    got = cpu_shim.eval_prog(E.compile_expr(E.parse("case when a > 1 then b * 2 when a < 0 then 0 else 7 end"), sch), cols, 4)
    assert np.array_equal(got, np.array([7.0, 5.0, -6.0, 0.0]))


def test_edge_ops_compose_like_filter_map_select_rename():
    raw = ["a", "b", "c"]
    ops = EdgeOps()
    ops.with_columns({"d": E.parse("a * (1 - b)")}, raw)
    ops.filter(E.parse("d > 3 and c = 1"), raw)                      # refers to the computed column
    ops.rename({"d": "disc"}, raw)
    ops.select(["disc", "c"], raw)
    assert ops.visible(raw) == ["disc", "c"]
    assert ops.pred.sql() == "(((a * (1 - b)) > 3) and (c = 1))"     # predicate rewritten over RAW columns
    assert ops.required_raw(raw) == {"a", "b", "c"}
    with pytest.raises(L.QkError):
        ops.select(["nope"], raw)
    # no kernel is needed for pure column plumbing
    t = DeviceTable({"a": DeviceColumn(torch.arange(3)), "b": DeviceColumn(torch.arange(3.0))})
    out = EdgeOps().select(["b"], ["a", "b"]).rename({"b": "z"}, ["a", "b"]).apply(t)
    assert out.column_names == ["z"] and out["z"].data is t["b"].data


def _src(schema, rows):
    return SourceNode(object(), schema, rows)


def test_predicate_pushdown_through_joins_and_maps():
    li, od, cu = _src(["l_orderkey", "l_shipdate", "l_price"], 600), _src(["o_orderkey", "o_custkey", "o_orderdate"], 150), _src(["c_custkey", "c_seg"], 15)
    j1 = JoinNode(li, od, "l_orderkey", "o_orderkey", "inner", "_2")
    j2 = JoinNode(cu, j1, "c_custkey", "o_custkey", "inner", "_2")
    top = FilterNode(j2, E.parse("c_seg = 1 and o_orderdate < 9204 and l_shipdate > 9204 and l_price > c_custkey"))
    out = push_filters(top, [])
    assert out.kind == "filter" and out.pred.sql() == "(l_price > c_custkey)"        # spans both sides: stays above
    j2n = out.parents[0]
    assert j2n.parents[0].kind == "filter" and j2n.parents[0].pred.sql() == "(c_seg = 1)"
    j1n = j2n.parents[1]
    assert j1n.parents[0].pred.sql() == "(l_shipdate > 9204)" and j1n.parents[1].pred.sql() == "(o_orderdate < 9204)"
    # a filter on a computed column stays above the map, one on a raw column goes below it
    m = MapNode(li, {"rev": E.parse("l_price * 2")})
    out = push_filters(FilterNode(m, E.parse("rev > 10 and l_shipdate > 5")), [])
    assert out.kind == "filter" and out.pred.sql() == "(rev > 10)" and out.parents[0].parents[0].kind == "filter"
    # nothing is pushed to the right side of a non-inner join
    lj = JoinNode(li, od, "l_orderkey", "o_orderkey", "left", "_2")
    out = push_filters(FilterNode(lj, E.parse("o_orderdate < 3")), [])
    assert out.kind == "filter" and out.parents[0].parents[1].kind == "source"


def test_aggregate_decomposition_matches_the_reference_rules():
    items = E.parse_select_list("sum(a) as s, avg(b) as m, count(*) as n, sum(a) / sum(c) as r, avg(a) as m2, min(c) as lo")
    partial, final = decompose_aggs(items)
    ops = [(op, None if arg is None else arg.sql()) for op, arg, _ in partial]
    # AVG -> SUM + COUNT(*), identical partials computed once (sum(a) and count(*) are shared)
    assert ops == [("sum", "a"), ("sum", "b"), ("count", None), ("sum", "c"), ("min", "c")]
    assert "(SUM(e1_agg) / SUM(e2_agg)) AS m" in final and "SUM(e2_agg) AS n" in final and "MIN(e4_agg) AS lo" in final
    with pytest.raises(L.QkError, match="alias"):
        decompose_aggs(E.parse_select_list("sum(a)"))
    with pytest.raises(L.QkError, match="not an aggregation"):
        decompose_aggs(E.parse_select_list("a + 1 as x"))


def test_datastream_api_surface_and_schema_rules():
    class Ctx:
        exec_config = {}
    a = DataStream(Ctx(), _src(["k", "v"], 10))
    b = DataStream(Ctx(), _src(["k2", "v"], 10))
    j = a.join(b, left_on="k", right_on="k2")
    assert j.schema == ["k", "v", "v_2"]                                   # clash gets the suffix (datastream.py:1506-1519)
    assert a.join(b, left_on="k", right_on="k2", how="semi").schema == ["k", "v"]
    with pytest.raises(AssertionError):
        a.filter_sql("zzz > 1")                                            # datastream.py:374-375
    with pytest.raises(AssertionError):
        a.with_columns_sql("v * 2 as v")                                   # new names must not clash (:1276)
    with pytest.raises(AssertionError):
        a.join(b, on="k")
    g = a.groupby("k").agg({"v": ["sum", "avg"], "*": "count"})
    assert g.schema == ["k", "v_sum", "v_avg", "count"]                    # datastream.py:1863-1883
    with pytest.raises(AssertionError):
        a.groupby("k", orderby=["v"])                                      # orderby must be group keys (:1640-1643)
    with pytest.raises(NotImplementedError):
        a.with_columns({"x": lambda df: df})
    assert a.top_k("v", 3).schema == ["k", "v"]


def test_columns_arrow_roundtrip_dictionaries_and_validity():
    reg = DictionaryRegistry()
    t1 = pa.table({"s": pa.array(["b", "a", "b"]), "d": pa.array([1, 2, 3], pa.int32()).cast(pa.date32()), "x": [1.5, 2.5, 3.5],
                   "f": pa.array([True, False, True])})
    t2 = pa.table({"s": pa.array(["c", "a"]), "d": pa.array([4, 5], pa.int32()).cast(pa.date32()), "x": [4.5, 5.5], "f": pa.array([False, False])})
    a = DeviceTable.from_arrow(t1, "cpu", reg)
    b = DeviceTable.from_arrow(t2, "cpu", reg)
    assert a["s"].dictionary is b["s"].dictionary and a["s"].dictionary == ["b", "a", "c"]     # one code space per column
    both = concat_tables([a, b])
    back = both.to_arrow()
    assert back["s"].to_pylist() == ["b", "a", "b", "c", "a"] and back["d"].type == pa.date32() and back["f"].to_pylist() == [True, False, True, False, False]
    # independent dictionaries are unified by VALUE
    u, (p, q) = unify_dictionaries([DeviceColumn(torch.tensor([0, 1]), ["x", "y"]), DeviceColumn(torch.tensor([0, 1]), ["y", "z"])])
    assert u == ["x", "y", "z"] and p.data.tolist() == [0, 1] and q.data.tolist() == [1, 2]
    # "no match" rows become Arrow nulls
    v = DeviceTable({"k": DeviceColumn(torch.tensor([1, 2, 3])), "r": DeviceColumn(torch.tensor([7.0, 0.0, 9.0]), valid=torch.tensor([1, 0, 1], dtype=torch.uint8))})
    assert v.to_arrow()["r"].to_pylist() == [7.0, None, 9.0]
    assert v.drop_nulls is not None
    with pytest.raises(L.QkError, match="nulls"):
        DeviceTable.from_arrow(pa.table({"x": pa.array([1, None])}), "cpu")
    with pytest.raises(L.QkError, match="ragged"):
        DeviceTable({"a": DeviceColumn(torch.zeros(2)), "b": DeviceColumn(torch.zeros(3))})


def test_readers_deal_lineage_like_the_reference(tmp_path):
    tbl = pa.table({"time": np.arange(1000, dtype=np.int64), "v": np.arange(1000.0)})
    for i in range(4):
        pq.write_table(tbl.slice(i * 250, 250), tmp_path / f"part-{i}.parquet", row_group_size=50)
    r = InputParquetDataset(str(tmp_path) + "/*", row_groups_per_batch=2)
    st = r.get_own_state(3)
    units = [u for ch in st.values() for batch in ch for u in batch]
    assert len(units) == 20 and len(set(units)) == 20                      # every row group exactly once
    assert [len(sum(st[c], [])) for c in range(3)] == [7, 7, 6]            # round robin (unordered_readers.py:34-38)
    assert r.num_rows() == 1000 and r.schema().names == ["time", "v"]
    s = InputSortedParquetDataset(str(tmp_path) + "/*", "time", row_groups_per_batch=4)
    st = s.get_own_state(2)
    first = [pq.ParquetFile(f).read_row_group(g)["time"][0].as_py() for f, g in sum(st[0], []) + sum(st[1], [])]
    assert first == sorted(first)                                          # channel c = c-th contiguous time range
    a = InputArrowDataset(tbl, batch_rows=300).get_own_state(2)
    assert a == {0: [(0, 300), (300, 500)], 1: [(500, 800), (800, 1000)]}


def test_decimal_columns_become_exact_fp64():
    """DECIMAL(10,2) measures of the Spark-written TPC-H set (benchmark/spark/convert.py:11-14) on the host reader path."""
    import decimal
    cents = np.array([1234, 7, -97459795, 626378585, 0, 999999999], dtype=np.int64)
    arr = pa.array([decimal.Decimal(int(c)).scaleb(-2) for c in cents], pa.decimal128(10, 2))
    t = DeviceTable.from_arrow(pa.table({"p": arr, "q": arr.cast(pa.decimal128(12, 3))}), torch.device("cpu"))
    assert t["p"].data.dtype == torch.float64 and np.array_equal(t["p"].data.numpy(), cents / 100.0)
    assert np.array_equal(t["q"].data.numpy(), (cents * 10) / 1000.0)
    sliced = DeviceTable.from_arrow(pa.table({"p": arr.slice(2, 3)}), torch.device("cpu"))          # non-zero Arrow offset
    assert np.array_equal(sliced["p"].data.numpy(), cents[2:5] / 100.0)
    with pytest.raises(L.QkError, match="64-bit"):
        DeviceTable.from_arrow(pa.table({"p": pa.array([decimal.Decimal(1)], pa.decimal128(30, 2))}), torch.device("cpu"))


def test_random_expressions_compile_to_what_they_mean():
    """Differential test of the expression compiler: random SQL over integer / float / date / dictionary columns is parsed,
    compiled to a postfix program and run by the interpreter shim (the numpy mirror of libqk's interpreter, op for op);
    the same text is evaluated directly by a tiny tree-walking evaluator over numpy.  Both must agree exactly."""
    import cpu_shim
    rng = np.random.default_rng(42)
    n = 500
    data = {"a": rng.integers(-5, 6, n), "b": rng.integers(0, 100, n).astype(np.float64) / 4, "c": rng.integers(0, 3, n).astype(np.int32),
            "d": (8000 + rng.integers(0, 1200, n)).astype(np.int32), "s": rng.integers(0, 4, n).astype(np.int32)}
    words = ["PROMO TIN", "STANDARD", "PROMO BRASS", "ECONOMY"]
    sch = {"a": E.ColumnInfo(0, L.QK_I64), "b": E.ColumnInfo(1, L.QK_F64), "c": E.ColumnInfo(2, L.QK_I32),
           "d": E.ColumnInfo(3, L.QK_I32, None, True), "s": E.ColumnInfo(4, L.QK_I32, words)}
    cols = [data[k] for k in ("a", "b", "c", "d", "s")]

    def num(depth):
        r = rng.random()
        if depth <= 0 or r < 0.3:
            return str(rng.choice(["a", "b", "c", str(int(rng.integers(-3, 9))), f"{rng.integers(0, 50) / 4}"]))
        if r < 0.75:
            return f"({num(depth - 1)} {rng.choice(['+', '-', '*'])} {num(depth - 1)})"
        if r < 0.85:
            return f"(- {num(depth - 1)})"
        return f"(case when {boolean(depth - 1)} then {num(depth - 1)} else {num(depth - 1)} end)"

    def boolean(depth):
        r = rng.random()
        if depth <= 0 or r < 0.35:
            k = rng.integers(0, 6)
            if k == 0:
                return f"{num(0)} {rng.choice(['<', '<=', '>', '>=', '=', '<>'])} {num(1)}"
            if k == 1:
                return f"a {rng.choice(['in', 'not in'])} ({', '.join(str(int(v)) for v in rng.integers(-5, 6, 3))})"
            if k == 2:
                return f"b {rng.choice(['between', 'not between'])} {rng.integers(0, 10)} and {rng.integers(10, 25)}"
            if k == 3:
                return f"s {rng.choice(['=', '<>'])} '{rng.choice(words + ['NOPE'])}'"
            if k == 4:
                return f"s {rng.choice(['like', 'not like'])} '{rng.choice(['PROMO%', '%BRASS', '%O%', 'STANDAR_', 'zzz'])}'"
            return rng.choice(["d >= date '1993-01-01'", "d < date '1992-06-01' + interval '3' month", "extract(year from d) = 1993",
                               "extract(year from d) <= 1992", "a = c", "c < a", "true", "false"])
        if r < 0.8:
            return f"({boolean(depth - 1)} {rng.choice(['and', 'or'])} {boolean(depth - 1)})"
        return f"(not {boolean(depth - 1)})"

    import re as _re

    def like(pattern):
        rx = _re.compile("".join(".*" if ch == "%" else "." if ch == "_" else _re.escape(ch) for ch in pattern), _re.S)
        return np.array([bool(rx.fullmatch(w)) for w in words])

    def ev(node):                                   # direct evaluation of the parsed tree
        k = node.kind
        if k == "col":
            return data[node.value].astype(np.float64)
        if k in ("num", "date"):
            return np.full(n, float(node.value))
        if k == "un":
            v = ev(node.args[0])
            return -v if node.value == "neg" else (v == 0).astype(np.float64)
        if k == "func" and node.value == "case":
            c, x, y = (ev(a) for a in node.args)
            return np.where(c != 0, x, y)
        if k == "func" and node.value == "in":
            x = ev(node.args[0])
            return np.isin(x, [float(it.value) for it in node.args[1:]]).astype(np.float64)
        a, b = node.args
        op = node.value
        if op == "like":
            return like(b.value)[data[a.value]].astype(np.float64)
        if b.kind == "str" or a.kind == "str":
            col_, lit = (a, b) if b.kind == "str" else (b, a)
            code = words.index(lit.value) if lit.value in words else -1
            eq = data[col_.value] == code
            return (eq if op == "=" else ~eq).astype(np.float64)
        x, y = ev(a), ev(b)
        if op in "+-*":
            return {"+": x + y, "-": x - y, "*": x * y}[op]
        if op in ("and", "or"):
            return ((x != 0) & (y != 0) if op == "and" else (x != 0) | (y != 0)).astype(np.float64)
        return {"<": x < y, "<=": x <= y, ">": x > y, ">=": x >= y, "=": x == y, "!=": x != y}[op].astype(np.float64)

    checked = 0
    for trial in range(400):
        text = boolean(3) if trial % 2 else num(3)
        tree = E.parse(text)
        try:
            prog = E.compile_expr(tree, sch)
        except E.ExprError as err:
            assert "at most" in str(err) or "stack" in str(err), text
            continue
        depth = peak = 0
        for op, *_ in prog:                          # stay inside what the device interpreter accepts
            depth += 1 if op in (L.OP_COL, L.OP_CONST, L.OP_CMP_COL_IMM, L.OP_CMP_COL_COL, L.OP_IN_SET, L.OP_RANGE_COL_IMM) else (0 if op in (L.OP_NEG, L.OP_NOT, L.OP_RINT, L.OP_EXTRACT) else (-2 if op == L.OP_SELECT else -1))
            peak = max(peak, depth)
        assert peak <= L.MAX_STACK and len(prog) <= L.MAX_EXPR_NODES      # compile_expr refuses anything the kernel would
        got = cpu_shim.eval_prog(prog, cols, n)
        assert np.array_equal(got, ev(tree)), text
        assert E.parse(tree.sql()) == tree, text      # and the printed SQL means the same tree
        checked += 1
    assert checked > 300
