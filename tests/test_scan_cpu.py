"""The scan-filter-project reference and case generator (tests/scan_cases.py) on the CPU: the reference against a per-row
Python evaluation of the parsed expression, the CPU shim's scan_filter_project against the reference, the limits the cases
sit at, and the exact lowering of an integer column compared with a literal (expr.lower_int_cmp)."""
import datetime as dt
import math

import numpy as np
import pytest
import torch

import cpu_shim
import scan_cases as S
from quokka_b200 import _lib as L
from quokka_b200 import expr as E

RANDOM = S.random_cases(160)
COMPACT = S.compact_cases(40)
ALL_CASES = S.EDGE_CASES + RANDOM + COMPACT
_ids = lambda cs: [c.name for c in cs]      # noqa: E731


# ------------------------------------------------------------------ per-row Python evaluation of the parsed tree
def _fdiv(a, b):
    if b == 0.0:
        if a == 0.0 or math.isnan(a):
            return math.nan
        return math.copysign(math.inf, a) * math.copysign(1.0, b)
    return a / b


def _py_cmp(op, a, b, row):
    """Python's own comparisons: int with int / float exactly, floats as IEEE"""
    if a.kind != "col" and b.kind == "col":
        a, b, op = b, a, E._FLIP[op]
    f = {"<": lambda x, y: x < y, "<=": lambda x, y: x <= y, ">": lambda x, y: x > y, ">=": lambda x, y: x >= y,
         "=": lambda x, y: x == y, "!=": lambda x, y: x != y}[op]
    if a.kind == "col" and b.kind == "str":
        vals = S.DICTS[a.value]
        return f(vals[int(row[a.value])], b.value)
    if a.kind == "col" and a.value in S.INT_COLS and b.kind in ("num", "date"):
        return f(int(row[a.value]), b.value)
    if a.kind == "col" and a.value in S.INT_COLS and b.kind == "col" and b.value in S.INT_COLS:
        return f(int(row[a.value]), int(row[b.value]))
    return f(_py_value(a, row), _py_value(b, row))


def _py_value(e, row):
    k = e.kind
    if k == "col":
        return float(row[e.value])
    if k in ("num", "date"):
        return float(e.value)
    if k == "un":
        a = _py_value(e.args[0], row)
        return -a if e.value == "neg" else (1.0 if a == 0 else 0.0)
    if k == "func":
        if e.value == "case":
            return _py_value(e.args[1], row) if _py_value(e.args[0], row) != 0 else _py_value(e.args[2], row)
        if e.value == "cast_int":
            x = _py_value(e.args[0], row)
            return x if not math.isfinite(x) else math.copysign(float(round(x)), x)
        if e.value.startswith("extract_"):
            days, years = int(_py_value(e.args[0], row)), 0
            while days > S.DAY_9999:                       # past datetime.date's range: the calendar repeats every 400 years
                days, years = days - 146097, years + 400
            day = dt.date(1970, 1, 1) + dt.timedelta(days=days)
            return float(day.year + years if e.value == "extract_year" else getattr(day, e.value[8:]))
        if e.value == "in":
            return 1.0 if any(_py_cmp("=", e.args[0], it, row) for it in e.args[1:]) else 0.0
    if k == "bin":
        op = e.value
        if op in "+-*/":
            a, b = _py_value(e.args[0], row), _py_value(e.args[1], row)
            return {"+": lambda: a + b, "-": lambda: a - b, "*": lambda: a * b, "/": lambda: _fdiv(a, b)}[op]()
        if op in ("and", "or"):
            a, b = _py_value(e.args[0], row) != 0, _py_value(e.args[1], row) != 0
            return 1.0 if (a and b if op == "and" else a or b) else 0.0
        if op in S.CMPS:
            return 1.0 if _py_cmp(op, e.args[0], e.args[1], row) else 0.0
        if op == "like":
            c = e.args[0].value
            return 1.0 if int(row[c]) in S._like_codes(e.args[1].value, S.DICTS[c]) else 0.0
    raise ValueError(e.sql())


def _same_scalar(g, e):
    if isinstance(e, float):
        return (math.isnan(g) and math.isnan(e)) or (g == e and math.copysign(1.0, g) == math.copysign(1.0, e))
    return g == e


@pytest.mark.parametrize("case", S.EDGE_CASES + RANDOM[:80], ids=_ids(S.EDGE_CASES + RANDOM[:80]))
def test_reference_matches_per_row_python(case):
    d = S.make_data(257, seed=11)
    mask, outs = S.reference(case, d)
    rows = [{c: d[c][i].item() for c in S.COLUMNS} for i in range(257)]
    want = [(_py_value(E.parse(case.pred), r) != 0) if case.pred else True for r in rows]
    assert mask.tolist() == want
    kept = [r for r, m in zip(rows, want) if m]
    for p, o in zip(case.projs, outs):
        node = E.parse(p)
        exp = [r[p] if p in S.FLOAT_COLS else int(r[p]) for r in kept] if p in S.COLUMNS else [_py_value(node, r) for r in kept]
        got = o.tolist()
        bad = [i for i, (g, e) in enumerate(zip(got, exp)) if not _same_scalar(g, e)]
        assert len(got) == len(exp) and not bad, f"{p}: row {bad[:1]} got {[got[i] for i in bad[:1]]} want {[exp[i] for i in bad[:1]]}"


# ------------------------------------------------------------------ the CPU shim against the reference
@pytest.mark.parametrize("case", ALL_CASES, ids=_ids(ALL_CASES))
def test_shim_matches_reference(case):
    d = S.make_data(1000, seed=5)
    mask, exp = S.reference(case, d)
    pred, projs = S.compile_case(case)
    outs, m = cpu_shim.scan_filter_project([torch.from_numpy(d[c]) for c in S.COLUMNS], pred, projs, stable=True)
    assert m == int(mask.sum())
    for p, o, e in zip(case.projs, outs, exp):
        g = o.numpy()
        assert S.same(g.view(np.uint8) if g.dtype == np.bool_ else g, e), p


def test_cases_compile_and_cover_the_opcodes():
    used = set()
    for c in ALL_CASES:
        pred, projs = S.compile_case(c)
        used |= {node[0] for prog in [pred or []] + projs for node in prog}
    assert used == set(range(L.OP_COL, L.OP_RANGE_COL_IMM + 1))
    assert sum(S.compact_shaped(*S.compile_case(c)) for c in S.EDGE_CASES + RANDOM) >= 40


def test_limit_cases_sit_at_the_limits():
    by = {c.name: c for c in S.EDGE_CASES}

    def depth(prog):
        d = top = 0
        for op, *_ in prog:
            d += 1 if op in (L.OP_COL, L.OP_CONST, L.OP_CMP_COL_IMM, L.OP_CMP_COL_COL, L.OP_IN_SET, L.OP_RANGE_COL_IMM) else \
                -2 if op == L.OP_SELECT else 0 if op in (L.OP_NEG, L.OP_NOT, L.OP_RINT, L.OP_EXTRACT) else -1
            top = max(top, d)
        return top
    assert depth(S.compile_case(by["stack_8_pred"])[0]) == L.MAX_STACK
    assert depth(S.compile_case(by["stack_8_value"])[1][0]) == L.MAX_STACK
    assert len(S.compile_case(by["nodes_48"])[0]) == L.MAX_EXPR_NODES
    pred, projs = S.compile_case(by["nodes_112"])
    assert len(pred) + sum(map(len, projs)) == L.MAX_TOTAL_NODES
    # one more slot or node is refused on the host
    sch = S.schema()
    with pytest.raises(E.ExprError, match="stack"):
        E.compile_expr(E.parse("f64 + (f32 + (i32 + (u8 + (d + (j64 + (c3 + (f64 * 2)))))))"), sch)
    with pytest.raises(E.ExprError, match="nodes"):
        E.compile_expr(E.parse(by["nodes_48"].pred.replace("i32 > 3", "not (i32 > 3)")), sch)
    with pytest.raises(E.ExprError, match="in total"):
        E.check_call(len(S.COLUMNS), pred, projs + [[(L.OP_COL, 0, 0, 0.0, 0)]])


# ------------------------------------------------------------------ exact lowering of integer column <cmp> literal
SLOT = {c: i for i, c in enumerate(S.COLUMNS)}
ALWAYS, NEVER = (L.CMP_GE, S.I64_MIN), (L.CMP_LT, S.I64_MIN)


@pytest.mark.parametrize("sql,node", [
    ("i64 < 9223372036854775808", ALWAYS),
    ("i64 <= 9223372036854775808", ALWAYS),
    ("i64 > -9223372036854775809", ALWAYS),
    ("i64 > 9223372036854775808", NEVER),
    ("i64 = 18446744073709551616", NEVER),
    ("i64 != 18446744073709551616", ALWAYS),
    ("i64 in (18446744073709551616)", NEVER),
    ("i64 <= 9223372036854775807", (L.CMP_LE, S.I64_MAX)),
    ("i64 < -9223372036854775808", (L.CMP_LT, S.I64_MIN)),
    ("i64 > 1.7e18", (L.CMP_GT, 1_700_000_000_000_000_000)),
    ("i64 > 2.5", (L.CMP_GE, 3)),
    ("i64 >= 2.5", (L.CMP_GE, 3)),
    ("i64 < 2.5", (L.CMP_LE, 2)),
    ("i64 <= -2.5", (L.CMP_LE, -3)),
    ("2.5 < i64", (L.CMP_GE, 3)),
    ("i64 = 2.5", NEVER),
    ("i64 != 2.5", ALWAYS),
    ("i64 = 2.0", (L.CMP_EQ, 2)),
    ("i64 < (1e400 - 1e400)", NEVER),
    ("i64 = (1e400 - 1e400)", NEVER),
    ("i64 != (1e400 - 1e400)", ALWAYS),
    ("i64 < 1e400", ALWAYS),
    ("i64 > 1e400", NEVER),
    ("i64 > -1e400", ALWAYS),
    ("i64 != 1e400", ALWAYS),
    ("i64 < 9.3e18", ALWAYS),
    ("i64 >= 9.223372036854775807e18", NEVER),
    ("i64 <= -9.223372036854775808e18", (L.CMP_LE, S.I64_MIN)),
    ("i64 > -9.223372036854775808e18", (L.CMP_GT, S.I64_MIN)),
    ("i32 < 3000000000", (L.CMP_LT, 3000000000)),
    ("d >= date '1900-01-01'", (L.CMP_GE, S.DAY_1900)),
])
def test_literal_lowering(sql, node):
    col = E.parse(sql).columns().pop()
    assert E.compile_expr(E.parse(sql), S.schema()) == [(L.OP_CMP_COL_IMM, SLOT[col], node[0], 0.0, node[1])]


def test_literal_lowering_of_ranges_and_sets():
    sch = S.schema()
    assert E.compile_expr(E.parse("i64 between -0.5 and 65.5"), sch) == [(L.OP_RANGE_COL_IMM, SLOT["i64"], 0, 65.0, 0)]
    assert E.compile_expr(E.parse("j64 in (1.0, 2.5, 3.0, 1e400)"), sch) == [(L.OP_IN_SET, SLOT["j64"], 4, 0.0, 0b1010)]
    prog = E.compile_expr(E.parse("i64 in (1, 18446744073709551617)"), sch)
    assert prog == [(L.OP_CMP_COL_IMM, SLOT["i64"], L.CMP_EQ, 0.0, 1)]
    prog = E.compile_expr(E.parse("i64 in (100000, 18446744073709551617)"), sch)
    assert prog == [(L.OP_CMP_COL_IMM, SLOT["i64"], L.CMP_EQ, 0.0, 100000), (L.OP_CMP_COL_IMM, SLOT["i64"], *NEVER[:1], 0.0, NEVER[1]),
                    (L.OP_OR, 0, 0, 0.0, 0)]
    # a float column against the same literals stays an fp64 compare
    assert E.compile_expr(E.parse("f64 > 2.5"), sch) == [(L.OP_COL, SLOT["f64"], 0, 0.0, 0), (L.OP_CONST, 0, 0, 2.5, 0),
                                                         (L.OP_GT, 0, 0, 0.0, 0)]


_EDGE_X = sorted(set(S.I64_EDGES + [-3, -2, 2, 3, 64, 65, 2 ** 53 + 2, 2 ** 62, -2 ** 62]))
_EDGE_V = [2 ** 63, 2 ** 63 - 1, -2 ** 63, -2 ** 63 - 1, 2 ** 64, 0, 2, -3, 2 ** 53 + 1, S.NEAR + 1, 2.5, -2.5, 0.5, -0.5, -0.0,
           1.7e18, 2.0 ** 53, 2.0 ** 63, -2.0 ** 63, 9.3e18, -9.3e18, math.inf, -math.inf, math.nan, 1e-300, 9007199254740993.0]


@pytest.mark.parametrize("op", S.CMPS)
def test_lower_int_cmp_agrees_with_python(op):
    cmp = [lambda a, b: a < b, lambda a, b: a <= b, lambda a, b: a > b, lambda a, b: a >= b, lambda a, b: a == b, lambda a, b: a != b]
    for v in _EDGE_V:
        code, imm = E.lower_int_cmp(op, v)
        assert S.I64_MIN <= imm <= S.I64_MAX
        for x in _EDGE_X:
            want = {"<": x < v, "<=": x <= v, ">": x > v, ">=": x >= v, "=": x == v, "!=": x != v}[op]
            assert cmp[code](x, imm) == want, (x, op, v, code, imm)


def test_out_of_range_immediates_are_refused_not_wrapped():
    """An ABI-level program whose integer immediate does not fit int64 fails on the host (ops and the CPU shim alike)
    instead of wrapping in the int64 field of qk_expr_node."""
    cols = [torch.zeros(4, dtype=torch.int64)]
    keep = [[(L.OP_COL, 0, 0, 0.0, 0)]]
    for prog in ([(L.OP_CMP_COL_IMM, 0, L.CMP_LT, 0.0, 1 << 63)], [(L.OP_CMP_COL_IMM, 0, L.CMP_GT, 0.0, -(1 << 63) - 1)],
                 [(L.OP_RANGE_COL_IMM, 0, 0, 5.0, -(1 << 64))], [(L.OP_RANGE_COL_IMM, 0, 0, 2.0 ** 60, 0)]):
        with pytest.raises(E.ExprError):
            cpu_shim.scan_filter_project(cols, prog, keep)
