"""Exact reference and seeded case generator for K1, the scan-filter-project kernels (csrc/scan.cu qk_scan_filter_project:
the stable and unordered postfix interpreters; csrc/compact.cu: the TMA compaction and its Bloom-reduced form).

A case is SQL text: a predicate (or None) and a list of projections over a fixed set of columns.  The text goes through
`expr.parse` / `expr.compile_expr` like every query; the reference evaluates the PARSED `expr.Node` tree, never the compiled
program, so a compiler bug cannot cancel out.  Semantics of the reference:
- an integer column (u8, bool, i32, i64, date32, dictionary codes) against a numeric literal, and IN over such literals:
  exact, as Python compares an int with an int or a float (computed in long double, which holds every int64 and every
  double); NaN: every compare false, != true;
- integer column against integer column: exact int64;
- everything else is fp64 arithmetic in numpy, in the same operation order as the postfix program (the library is built
  with -fmad=false, so values are bit-identical), with IEEE compares (NaN unordered);
- AND / OR / NOT and the predicate itself test a value != 0 (so a NaN value is true); CASE selects on condition != 0;
  CAST AS INT is rint (half to even); EXTRACT goes through datetime64;
- string `=` / `!=` / IN and LIKE on a dictionary column are resolved against the dictionary.
Constant folding (`expr.fold`: literal arithmetic, date +- interval, EXTRACT(year) compares into date ranges) happens in
`parse` and is shared with the compiler.

Importable without a GPU: tests/test_scan_cpu.py checks the reference against a per-row Python evaluation and the CPU shim
against the reference; tests/test_gpu_scan.py runs every device path."""
from __future__ import annotations

import math
import re
from dataclasses import dataclass

import numpy as np

from quokka_b200 import _lib as L
from quokka_b200 import expr as E

I32_MIN, I32_MAX = -(1 << 31), (1 << 31) - 1
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
CMPS = ("<", "<=", ">", ">=", "=", "!=")
_NP_CMP = {"<": np.less, "<=": np.less_equal, ">": np.greater, ">=": np.greater_equal, "=": np.equal, "!=": np.not_equal}
DAY_1900, DAY_9999 = -25567, 2932896                     # 1900-01-01, 9999-12-31 in days since 1970-01-01
NEAR = 1_700_000_000_000_000_000                         # an int64 nanosecond timestamp: fp64 spacing 256 around it

_WORDS = ("red", "green", "blue", "dark red", "light_blue", "teal")
DICTS = {"c3": [f"{_WORDS[i % 6]} {i}" for i in range(3)],
         "c150": [f"{_WORDS[i % 6]} {i}" for i in range(150)],
         "c3000": [f"{_WORDS[i % 6]} {i}" for i in range(3000)]}
# name -> numpy dtype; the order is the kernel's column slot order
COLUMNS = {"u8": np.uint8, "b": np.bool_, "i32": np.int32, "i64": np.int64, "j64": np.int64, "f32": np.float32,
           "f64": np.float64, "d": np.int32, "c3": np.uint8, "c150": np.uint8, "c3000": np.int32, "rid": np.int64}
INT_COLS = ("u8", "b", "i32", "i64", "j64", "d", "c3", "c150", "c3000", "rid")
FLOAT_COLS = ("f32", "f64")
QK_DTYPE = {np.dtype(np.uint8): L.QK_U8, np.dtype(np.bool_): L.QK_U8, np.dtype(np.int32): L.QK_I32,
            np.dtype(np.int64): L.QK_I64, np.dtype(np.float32): L.QK_F32, np.dtype(np.float64): L.QK_F64}


def schema() -> dict:
    return {c: E.ColumnInfo(i, QK_DTYPE[np.dtype(t)], DICTS.get(c), c == "d") for i, (c, t) in enumerate(COLUMNS.items())}


# ------------------------------------------------------------------ data
I64_EDGES = [I64_MIN, I64_MIN + 1, -(1 << 53) - 1, -(1 << 53), -(1 << 53) + 1, -1, 0, 1, (1 << 53) - 1, 1 << 53,
             (1 << 53) + 1, I64_MAX - 1, I64_MAX] + [NEAR + k for k in (-257, -256, -129, -128, -127, -1, 0, 1, 127, 128, 129, 255, 256, 257)]
I32_EDGES = [I32_MIN, I32_MIN + 1, -1, 0, 1, 63, 64, 65, I32_MAX - 1, I32_MAX]
F64_SPECIAL = [math.nan, -math.nan, 0.0, -0.0, math.inf, -math.inf, 5e-324, -5e-324, 2.2250738585072014e-308, 1.5, 2.5, -2.5,
               -0.5, 0.5, float(NEAR), 2.0 ** 53, 2.0 ** 53 + 2, 1e308, -1e308]
F32_SPECIAL = [math.nan, 0.0, -0.0, math.inf, -math.inf, 1e-45, -1e-45, 1.1754942e-38, 3.4028235e38, 0.5, 2.5, -2.5, -1.5]
DATE_EDGES = [DAY_1900, DAY_1900 + 58, DAY_1900 + 59, -306, -1, 0, 59, 10956 + 59, DAY_9999 - 1, DAY_9999]


def _pick(rng, n, dtype, parts):
    """n values of `dtype`, each drawn from one of `parts` (callables rng, k -> k values) chosen uniformly per row"""
    which = rng.integers(0, len(parts), n)
    out = np.empty(n, dtype=dtype)
    for j, f in enumerate(parts):
        sel = np.nonzero(which == j)[0]
        if len(sel):
            out[sel] = np.asarray(f(rng, len(sel))).astype(dtype)
    return out


def make_data(n: int, seed: int = 0) -> dict:
    rng = np.random.default_rng(seed)
    ch = lambda vals, t: (lambda r, k: r.choice(np.array(vals, dtype=t), k))       # noqa: E731
    d = {}
    d["u8"] = _pick(rng, n, np.uint8, [lambda r, k: r.integers(0, 256, k), lambda r, k: r.integers(0, 70, k),
                                       ch([0, 31, 32, 63, 64, 65, 76, 77, 255], np.uint8)])
    d["b"] = rng.integers(0, 2, n).astype(np.bool_)
    d["i32"] = _pick(rng, n, np.int32, [lambda r, k: r.integers(I32_MIN, I32_MAX, k, endpoint=True),
                                        lambda r, k: r.integers(-70, 70, k), ch(I32_EDGES, np.int32)])
    d["i64"] = _pick(rng, n, np.int64, [lambda r, k: r.integers(I64_MIN, I64_MAX, k, endpoint=True, dtype=np.int64),
                                        lambda r, k: r.integers(-70, 70, k), lambda r, k: NEAR + r.integers(-300, 300, k),
                                        ch(I64_EDGES, np.int64)])
    d["j64"] = _pick(rng, n, np.int64, [lambda r, k: r.integers(-70, 70, k), ch(I64_EDGES, np.int64)])
    d["f64"] = _pick(rng, n, np.float64, [lambda r, k: r.normal(0, 100, k), lambda r, k: r.integers(-140, 140, k) / 2.0,
                                          ch(F64_SPECIAL, np.float64)])
    d["f32"] = _pick(rng, n, np.float32, [lambda r, k: r.normal(0, 100, k), lambda r, k: r.integers(-140, 140, k) / 2.0,
                                          ch(F32_SPECIAL, np.float32)])
    d["d"] = _pick(rng, n, np.int32, [lambda r, k: r.integers(DAY_1900, DAY_9999, k, endpoint=True), ch(DATE_EDGES, np.int32)])
    d["c3"] = rng.integers(0, 3, n).astype(np.uint8)
    d["c150"] = rng.integers(0, 150, n).astype(np.uint8)
    d["c3000"] = rng.integers(0, 3000, n).astype(np.int32)
    d["rid"] = np.arange(n, dtype=np.int64)
    return {c: d[c] for c in COLUMNS}


# ------------------------------------------------------------------ reference
_LD = np.longdouble


def _exact_vs_literal(x: np.ndarray, op: str, v) -> np.ndarray:
    """integer array x <op> Python int / float v, exactly"""
    assert np.finfo(_LD).nmant >= 63, "the exact compare needs a long double that holds every int64"
    if isinstance(v, float) and math.isnan(v):
        return np.full(len(x), op == "!=")
    if isinstance(v, int):
        v = float(2 ** 64) if v > I64_MAX else float(-2 ** 64) if v < I64_MIN else v      # beyond every x either way
        lv = np.array([v], dtype=np.int64).astype(_LD)[0] if isinstance(v, int) else _LD(v)
    else:
        lv = _LD(v)
    return _NP_CMP[op](x.astype(np.int64).astype(_LD), lv)


def _is_int_col(n: E.Node) -> bool:
    return n.kind == "col" and n.value in INT_COLS


def _errfree(f, *a):
    with np.errstate(all="ignore"):
        return f(*a)


def _like_codes(pattern: str, values: list) -> list:
    rx = re.compile("".join(".*" if c == "%" else "." if c == "_" else re.escape(c) for c in pattern), re.S)
    return [i for i, v in enumerate(values) if rx.fullmatch(v)]


def _compare(op: str, a: E.Node, b: E.Node, d: dict, n: int) -> np.ndarray:
    if a.kind != "col" and b.kind == "col":
        a, b, op = b, a, E._FLIP[op]
    if a.kind == "col" and b.kind == "str":
        vals = DICTS[a.value]
        code = vals.index(b.value) if b.value in vals else None
        eq = d[a.value].astype(np.int64) == code if code is not None else np.zeros(n, bool)
        return eq if op == "=" else ~eq
    if _is_int_col(a) and b.kind in ("num", "date"):
        return _exact_vs_literal(d[a.value], op, b.value)
    if _is_int_col(a) and _is_int_col(b):
        return _NP_CMP[op](d[a.value].astype(np.int64), d[b.value].astype(np.int64))
    return _errfree(_NP_CMP[op], value(a, d, n), value(b, d, n))


def value(e: E.Node, d: dict, n: int) -> np.ndarray:
    """fp64 value of every row (a comparison or a logical operator is 1.0 / 0.0)"""
    k = e.kind
    if k == "col":
        return d[e.value].astype(np.float64)
    if k in ("num", "date"):
        return np.full(n, float(e.value))
    if k == "un":
        a = value(e.args[0], d, n)
        return -a if e.value == "neg" else (a == 0).astype(np.float64)
    if k == "func":
        if e.value == "case":
            c, a, b = (value(x, d, n) for x in e.args)
            return np.where(c != 0, a, b)
        if e.value == "cast_int":
            return np.rint(value(e.args[0], d, n))
        if e.value.startswith("extract_"):
            days = value(e.args[0], d, n).astype(np.int64).astype("datetime64[D]")
            part = {"year": days.astype("datetime64[Y]").astype(np.int64) + 1970,
                    "month": days.astype("datetime64[M]").astype(np.int64) % 12 + 1,
                    "day": (days - days.astype("datetime64[M]")).astype(np.int64) + 1}[e.value[8:]]
            return part.astype(np.float64)
        if e.value == "in":
            m = np.zeros(n, bool)
            for it in e.args[1:]:
                m |= _compare("=", e.args[0], it, d, n)
            return m.astype(np.float64)
    if k == "bin":
        op = e.value
        if op in ("+", "-", "*", "/"):
            a, b = value(e.args[0], d, n), value(e.args[1], d, n)
            return _errfree({"+": np.add, "-": np.subtract, "*": np.multiply, "/": np.divide}[op], a, b)
        if op in ("and", "or"):
            a, b = value(e.args[0], d, n) != 0, value(e.args[1], d, n) != 0
            return (a & b if op == "and" else a | b).astype(np.float64)
        if op in CMPS:
            return _compare(op, e.args[0], e.args[1], d, n).astype(np.float64)
        if op == "like":
            c = e.args[0].value
            return np.isin(d[c].astype(np.int64), _like_codes(e.args[1].value, DICTS[c])).astype(np.float64)
    raise ValueError(f"reference cannot evaluate {e.sql()}")


def out_dtype(proj_sql: str):
    """a bare column is copied verbatim in its own dtype (bool as uint8); anything else is an fp64 expression"""
    t = COLUMNS.get(proj_sql.strip())
    return np.dtype(np.uint8) if t is np.bool_ else np.dtype(t) if t is not None else np.dtype(np.float64)


@dataclass
class Case:
    name: str
    pred: str | None
    projs: tuple = ()


def reference(case: Case, d: dict):
    """(pass mask, [expected output arrays]) of a case over the data d"""
    n = len(d["rid"])
    mask = value(E.parse(case.pred), d, n) != 0 if case.pred else np.ones(n, bool)
    outs = []
    for p in case.projs:
        if p.strip() in COLUMNS:
            outs.append(d[p.strip()][mask].astype(out_dtype(p)))
        else:
            outs.append(value(E.parse(p), d, n)[mask])
    return mask, outs


def compile_case(case: Case):
    """(pred program or None, projection programs), checked against the limits of one kernel call"""
    sch = schema()
    pred = E.compile_expr(E.parse(case.pred), sch) if case.pred else None
    projs = [E.compile_expr(E.parse(p), sch) for p in case.projs]
    E.check_call(len(COLUMNS), pred, projs)
    return pred, projs


def compact_shaped(pred, projs) -> bool:
    """whether csrc/compact.cu takes the call (given 16-byte aligned columns and at least one row)"""
    return (1 <= len(projs) <= 8 and all(len(p) == 1 and p[0][0] == L.OP_COL for p in projs)
            and (not pred or (len(pred) == 1 and pred[0][0] in (L.OP_CMP_COL_IMM, L.OP_RANGE_COL_IMM))))


def compact_tile_rows(projs, ctas_per_sm: int = 3) -> int:
    """the tile of csrc/compact.cu try_filter_compact_tma for these verbatim projections"""
    row_bytes = sum(np.dtype(out_dtype(p)).itemsize for p in projs)
    return min(((216 * 1024 // ctas_per_sm - 1024) // 3 // row_bytes) // 256 * 256, 16 * 256)


def same(got: np.ndarray, exp: np.ndarray) -> bool:
    """bit-exact, except that every NaN equals every NaN (payloads differ between numpy and the device)"""
    if got.dtype != exp.dtype or got.shape != exp.shape:
        return False
    if got.dtype.kind != "f":
        return np.array_equal(got, exp)
    gn, en = np.isnan(got), np.isnan(exp)
    w = np.dtype(f"u{got.dtype.itemsize}")
    return np.array_equal(gn, en) and np.array_equal(got[~gn].view(w), exp[~en].view(w))


def row_keys(outs: list) -> np.ndarray:
    """the output rows as one sortable uint64 matrix (NaN canonicalised), to compare arrival-order outputs as multisets"""
    cols = []
    for o in outs:
        if o.dtype.kind == "f":
            o = np.where(np.isnan(o), np.array(np.nan, o.dtype), o)
            o = o.view(np.dtype(f"u{o.dtype.itemsize}"))
        cols.append(o.astype(np.int64).view(np.uint64) if o.dtype.kind == "i" else o.astype(np.uint64))
    m = np.stack(cols, axis=1) if cols else np.zeros((0, 0), np.uint64)
    return m[np.lexsort(m.T[::-1])] if len(cols) else m


# ------------------------------------------------------------------ hand-written cases
def _or_chain(terms):
    return " or ".join(f"({t})" for t in terms)


EDGE_CASES = [
    # defect 1: literals outside int64 (the compiler used to wrap them into the int64 immediate)
    Case("lit_2p63_lt", "i64 < 9223372036854775808", ("rid", "i64")),
    Case("lit_m2p63m1_gt", "i64 > -9223372036854775809", ("rid",)),
    Case("lit_2p64_in", "i64 in (18446744073709551616)", ("rid",)),
    Case("lit_2p64_ne", "i64 != 18446744073709551616", ("rid", "i64")),
    Case("lit_i64max_le", "i64 <= 9223372036854775807", ("rid",)),
    Case("lit_i64min_lt", "i64 < -9223372036854775808", ("rid",)),
    Case("lit_i64min_eq", "i64 = -9223372036854775808", ("rid", "i64")),
    Case("lit_i32_wide", "i32 < 3000000000", ("i32",)),
    Case("lit_u8_neg", "u8 > -1", ("u8",)),
    Case("lit_u8_256", "u8 = 256", ("u8",)),
    Case("lit_huge_in_mixed", "i64 in (1, 18446744073709551617, -9223372036854775809, 9223372036854775807)", ("rid", "i64")),
    Case("lit_huge_or", "i64 < 9223372036854775808 and f64 > 0", ("rid",)),
    # defect 2: integer column against a non-integer literal (used to be compared in fp64)
    Case("near_gt", "i64 > 1.7e18", ("rid", "i64")),
    Case("near_ge", "i64 >= 1.7e18", ("i64",)),
    Case("near_eq", "i64 = 1.7e18", ("rid",)),
    Case("near_ne", "i64 != 1.7e18", ("rid",)),
    Case("near_le", "i64 <= 1700000000000000128.0", ("i64",)),
    Case("near_between", "i64 between 1.7e18 and 1.7000000000000002e18", ("i64",)),
    Case("frac_gt", "i64 > 2.5", ("i64",)),
    Case("frac_lt", "i32 < -2.5", ("i32",)),
    Case("frac_le", "u8 <= 64.5", ("u8",)),
    Case("frac_ge", "d >= -0.5", ("d",)),
    Case("frac_eq", "i64 = 2.5", ("rid",)),
    Case("frac_ne", "j64 != 2.5", ("j64",)),
    Case("integral_float_eq", "j64 = 2.0", ("j64",)),
    Case("float_2p53", "i64 > 9007199254740993.0", ("i64",)),        # the literal rounds to 2^53 when it is read
    Case("float_beyond_i64", "i64 < 9.3e18", ("rid",)),
    Case("float_below_i64", "i64 > -9.3e18", ("rid",)),
    Case("float_i64max", "i64 >= 9.223372036854775807e18", ("i64",)),   # = 2^63: above every int64
    Case("float_i64min", "i64 <= -9.223372036854775808e18", ("i64",)),  # = -2^63
    Case("inf_lt", "i64 < 1e400", ("rid",)),
    Case("minf_lt", "i64 < -1e400", ("rid",)),
    Case("inf_ne", "i32 != 1e400", ("rid",)),
    Case("nan_eq", "i64 = (1e400 - 1e400)", ("rid",)),
    Case("nan_ne", "i64 != (1e400 - 1e400)", ("rid",)),
    Case("nan_lt", "u8 < (1e400 - 1e400)", ("rid",)),
    Case("frac_between", "i64 between -0.5 and 65.5", ("i64", "rid")),
    Case("frac_in", "j64 in (1.0, 2.5, 3.0, -1e400)", ("j64",)),
    Case("frac_in_big", "i64 in (1.7e18, 9007199254740992.0, 0.5)", ("rid", "i64")),
    # IN_SET at its bitmap boundaries
    Case("set_64_bits", "u8 in (0, 5, 63)", ("u8",)),
    Case("set_65_bits", "u8 in (1, 64)", ("u8", "rid")),
    Case("set_77_bits", "u8 in (3, 31, 32, 76)", ("u8",)),
    Case("set_96_bits", "i32 in (0, 31, 32, 95)", ("i32",)),
    Case("set_256_bits", "u8 in (0, 255)", ("u8",)),
    Case("set_neg_codes", "i32 in (1, 5, 63)", ("i32",)),
    Case("set_neg_literal", "i32 in (-1, 5, 63)", ("i32",)),
    Case("set_not", "not (u8 in (2, 64, 65))", ("u8",)),
    Case("set_bool", "b in (1)", ("b", "rid")),
    Case("dict_in", "c150 in ('red 0', 'teal 149', 'green 61', 'nope')", ("c150",)),
    Case("dict_like_wide", "c3000 like '%7'", ("c3000", "rid")),
    Case("dict_like_64", "c150 like 'red %'", ("c150",)),
    Case("dict_like_none", "c150 like 'purple%'", ("c150",)),
    Case("dict_not_like", "c3000 not like 'dark%'", ("c3000",)),
    Case("dict_eq", "c3 = 'green 1'", ("c3", "rid")),
    Case("dict_ne_absent", "c3 != 'purple'", ("c3",)),
    Case("dict_eq_absent", "c3000 = 'purple'", ("c3000",)),
    # empty and full ranges
    Case("range_empty", "i64 between 5 and 4", ("i64",)),
    Case("range_full_i32", "i32 between -2147483648 and 2147483647", ("i32",)),
    Case("range_full_date", "d between date '1900-01-01' and date '9999-12-31'", ("d",)),
    Case("range_full_i64", "i64 >= -9223372036854775808", ("rid",)),
    Case("range_u8", "u8 between 0 and 255", ("u8",)),
    Case("range_2p53", "i64 between -9007199254740992 and 9007199254740992", ("i64",)),
    Case("range_beyond_2p53", "i64 between -9007199254740993 and 9007199254740993", ("i64",)),
    Case("range_neg_merge", "not (i64 >= 0 and i64 < 64)", ("i64",)),
    Case("range_date", "d >= date '1969-03-01' and d < date '1970-03-01'", ("d", "rid")),
    # EXTRACT before and after 1970
    Case("extract_year_lt", "extract(year from d) < 1950", ("d",)),
    Case("extract_year_eq", "extract(year from d) = 1900", ("d",)),
    Case("extract_month", "extract(month from d) = 2", ("d", "extract(day from d)")),
    Case("extract_values", None, ("extract(year from d)", "extract(month from d)", "extract(day from d)")),
    Case("extract_shifted", "extract(day from d + 1) = 1", ("extract(year from d - 366)",)),
    # floats: NaN, ±0, ±inf, subnormals
    Case("f64_zero", "f64 = 0", ("f64",)),
    Case("f64_neg_zero", "f64 = -0.0", ("f64",)),
    Case("f64_nan_rows", "not (f64 = f64)", ("f64", "rid")),
    Case("f64_ne_self", "f64 != f64", ("rid",)),
    Case("f64_inf", "f64 = 1e400 or f64 = -1e400", ("f64",)),
    Case("f64_subnormal", "f64 > 0 and f64 < 1e-307", ("f64",)),
    Case("f32_subnormal", "f32 > 0 and f32 < 1e-40", ("f32",)),
    Case("f32_nan", "f32 != f32", ("f32", "rid")),
    Case("f32_vs_f64", "f32 < f64", ("f32", "f64")),
    Case("f64_nan_literal", "f64 < (1e400 - 1e400)", ("rid",)),
    Case("f64_nan_truthy", "f64 * 0 + 1", ("rid",)),                    # NaN, inf * 0 = NaN: a NaN predicate value passes
    # arithmetic projections (bit-exact)
    Case("arith", "b = 1", ("f64 * f32 - i32 / 7", "-(f64)", "i64 + 1", "u8 / (f64 - f64)")),
    Case("rint", None, ("cast(f64 as int)", "cast(f32 * 3 as int)", "cast(i64 as int)")),
    Case("case_select", "u8 < 128", ("case when f64 > 0 then f64 else -f64 end", "case when b = 1 then 1 / f64 else i32 end")),
    Case("cmp_value", None, ("(f64 < 0) + (i64 > 1.7e18) * 2 + (c3 = 'red 0') * 4",)),
    Case("colcol", "i64 < j64", ("i64", "j64")),
    Case("colcol_eq", "j64 = i64 or u8 >= i32", ("rid",)),
    Case("colcol_mixed_width", "u8 > c150 and i32 != d", ("u8", "c150", "i32", "d")),
    # count only
    Case("count_only_interp", "f64 > 0", ()),
    Case("count_only_cmp", "i64 > 0", ()),
    Case("count_only_none", None, ()),
    # program limits: stack depth 8, 48 nodes, 112 nodes over the call
    Case("stack_8_pred", "u8 < 1 or (u8 < 2 or (u8 < 3 or (u8 < 4 or (u8 < 5 or (u8 < 6 or (u8 < 7 or u8 > 250))))))", ("u8",)),
    Case("stack_8_value", None, ("f64 + (f32 + (i32 + (u8 + (d + (j64 + (c3 + f64))))))",)),
    Case("nodes_48", "not (" + _or_chain([f"i64 = {k}" for k in range(-11, 12)]) + " or i32 > 3)", ("i64",)),
    Case("nodes_112", "not (" + _or_chain([f"u8 = {k}" for k in range(0, 240, 10)]) + ")",
         ("(" + " + ".join(["f64"] * 8) + ") * (" + " + ".join(["f32"] * 8) + ") - (" + " + ".join(["i32"] * 8) + ")",
          "case when c150 > 3 then " + " - ".join(["u8"] * 7) + " else -d end")),
    # verbatim projections of every dtype
    Case("all_columns", "c3 != 1", tuple(COLUMNS)[:8]),
]


# ------------------------------------------------------------------ random cases
_INT_LITS = [0, 1, -1, 2, 63, 64, 65, 255, 256, -70, 70, 2147483647, -2147483648, 2147483648, 9007199254740992,
             9007199254740993, -9007199254740993, NEAR, NEAR + 1, NEAR - 128, 9223372036854775807, 9223372036854775808,
             -9223372036854775808, -9223372036854775809, 18446744073709551616, -36893488147419103232]
_FLOAT_LITS = ["0.0", "-0.0", "0.5", "-0.5", "2.5", "-2.5", "64.5", "1e400", "-1e400", "(1e400 - 1e400)", "1.7e18",
               "1.7000000000000002e18", "9.3e18", "-9.3e18", "9007199254740993.0", "1e-310", "3.4028235e38", "100.25"]
_NUM_COLS = ("u8", "b", "i32", "i64", "j64", "f32", "f64", "d", "c3", "c150", "c3000")


class _Gen:
    def __init__(self, rng):
        self.r = rng

    def pick(self, xs):
        return xs[int(self.r.integers(0, len(xs)))]

    def int_lit(self):
        return str(self.pick(_INT_LITS)) if self.r.random() < 0.6 else str(int(self.r.integers(-80, 80)))

    def lit(self):
        return self.pick(_FLOAT_LITS) if self.r.random() < 0.5 else self.int_lit()

    def icol(self):
        return self.pick(("u8", "b", "i32", "i64", "j64", "d", "c3", "c150", "c3000"))

    def term(self, depth):
        r = self.r.random()
        if r < 0.18:
            return f"{self.icol()} {self.pick(CMPS)} {self.int_lit()}"
        if r < 0.30:
            return f"{self.icol()} {self.pick(CMPS)} {self.pick(_FLOAT_LITS)}"
        if r < 0.36:
            return f"{self.int_lit()} {self.pick(CMPS)} {self.icol()}"
        if r < 0.44:
            return f"{self.icol()} between {self.int_lit()} and {self.lit()}"
        if r < 0.52:
            k = int(self.r.integers(1, 6))
            return f"{self.icol()} in ({', '.join(self.lit() for _ in range(k))})"
        if r < 0.58:
            return f"{self.icol()} {self.pick(CMPS)} {self.icol()}"
        if r < 0.66:
            return f"{self.pick(FLOAT_COLS)} {self.pick(CMPS)} {self.lit()}"
        if r < 0.74:
            c = self.pick(("c3", "c150", "c3000"))
            v = self.pick(DICTS[c]) if self.r.random() < 0.8 else "purple"
            return f"{c} {self.pick(('=', '!='))} '{v}'"
        if r < 0.79:
            c = self.pick(("c3", "c150", "c3000"))
            return f"{c} in ({', '.join(repr(self.pick(DICTS[c])) for _ in range(int(self.r.integers(1, 5))))})"
        if r < 0.84:
            c = self.pick(("c150", "c3000"))
            pat = self.pick(("red%", "%7", "%e_n%", "_r%", "dark red 1%", "%", "teal 14_", "%blue%"))
            return f"{c} {self.pick(('like', 'not like'))} '{pat}'"
        if r < 0.90 and depth > 0:
            return f"extract({self.pick(('year', 'month', 'day'))} from d) {self.pick(CMPS)} {int(self.r.integers(1, 32))}"
        return f"{self.value(max(depth - 1, 0))} {self.pick(CMPS)} {self.value(max(depth - 1, 0))}"

    def pred(self, depth):
        r = self.r.random()
        if depth <= 0 or r < 0.4:
            return self.term(depth)
        if r < 0.55:
            return f"not ({self.pred(depth - 1)})"
        return f"({self.pred(depth - 1)}) {self.pick(('and', 'or'))} ({self.pred(depth - 1)})"

    def value(self, depth):
        r = self.r.random()
        if depth <= 0 or r < 0.3:
            return self.pick(_NUM_COLS) if self.r.random() < 0.75 else self.lit()
        if r < 0.6:
            return f"({self.value(depth - 1)} {self.pick('+-*/')} {self.value(depth - 1)})"
        if r < 0.67:
            return f"(-{self.value(depth - 1)})"
        if r < 0.74:
            return f"cast({self.value(depth - 1)} as int)"
        if r < 0.81:
            return f"extract({self.pick(('year', 'month', 'day'))} from d{self.pick(('', ' + 1', ' - 400'))})"
        if r < 0.92:
            return f"case when {self.pred(depth - 1)} then {self.value(depth - 1)} else {self.value(depth - 1)} end"
        return f"({self.pred(depth - 1)})"

    def case(self, i):
        pred = None if self.r.random() < 0.08 else self.pred(int(self.r.integers(0, 4)))
        projs = []
        for _ in range(int(self.r.integers(0, 5))):
            projs.append(self.pick(tuple(COLUMNS)) if self.r.random() < 0.5 else self.value(int(self.r.integers(0, 4))))
        return Case(f"rand{i}", pred, tuple(projs))


def random_cases(n: int, seed: int = 1) -> list:
    """n seeded cases from the grammar above, each within the limits of one kernel call (check_call)"""
    g = _Gen(np.random.default_rng(seed))
    out = []
    while len(out) < n:
        c = g.case(len(out))
        try:
            compile_case(c)
        except E.ExprError:
            continue
        out.append(c)
    return out


def compact_cases(n: int, seed: int = 2) -> list:
    """seeded cases of the TMA compaction's shape: one integer compare / range (or none) and 1-8 verbatim columns"""
    g = _Gen(np.random.default_rng(seed))
    out = []
    while len(out) < n:
        r = g.r.random()
        pred = (None if r < 0.1 else f"{g.icol()} {g.pick(CMPS)} {g.lit()}" if r < 0.7
                else f"{g.icol()} between {g.int_lit()} and {g.lit()}")
        cols = list(g.r.permutation(list(COLUMNS))[:int(g.r.integers(1, 9))])
        c = Case(f"compact{len(out)}", pred, tuple(cols))
        if compact_shaped(*compile_case(c)):
            out.append(c)
    return out
