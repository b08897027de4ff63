"""SQL-subset expressions: parser, normaliser and compiler to libqk postfix programs.

Replaces the sqlglot dependency of the reference (pyquokka/sql_utils.py:86-223 `evaluate`,
:225-287 `parquet_condition_decomp`, :299-413 aggregate decomposition) for the subset the judged
queries use (SURVEY.md Appendix E): arithmetic + - * /, comparisons, AND / OR / NOT, BETWEEN, IN,
`date 'YYYY-MM-DD'`, `interval 'n' day|month|year` (folded on the host), string literals against
dictionary columns (resolved to codes on the host), CAST(x AS INT), aggregate calls
SUM / AVG / MIN / MAX / COUNT(*) with aliases.
"""
from __future__ import annotations

import datetime as _dt
import math
import re
from dataclasses import dataclass
from typing import Any

from . import _lib as L


class ExprError(ValueError):
    pass


# ------------------------------------------------------------------ IR
@dataclass(frozen=True)
class Node:
    kind: str                 # col | num | str | date | interval | bin | un | func | agg | star
    value: Any = None
    args: tuple = ()

    def columns(self) -> set:
        if self.kind == "col":
            return {self.value}
        out = set()
        for a in self.args:
            out |= a.columns()
        return out

    def has_agg(self) -> bool:
        return self.kind == "agg" or any(a.has_agg() for a in self.args)

    def sql(self) -> str:
        k = self.kind
        if k == "col":
            return self.value
        if k == "num":
            return repr(self.value)
        if k == "str":
            return "'" + self.value + "'"
        if k == "date":
            return "date '" + (_dt.date(1970, 1, 1) + _dt.timedelta(days=self.value)).isoformat() + "'"
        if k == "interval":
            return f"interval '{self.value[0]}' {self.value[1]}"
        if k == "bin":
            return f"({self.args[0].sql()} {self.value} {self.args[1].sql()})"
        if k == "func" and self.value == "case":
            return f"(case when {self.args[0].sql()} then {self.args[1].sql()} else {self.args[2].sql()} end)"
        if k == "func" and self.value.startswith("extract_"):
            return f"extract({self.value[8:]} from {self.args[0].sql()})"
        if k == "func" and self.value == "cast_int":
            return f"cast({self.args[0].sql()} as int)"
        if k == "func" and self.value == "in":
            return f"({self.args[0].sql()} in ({', '.join(a.sql() for a in self.args[1:])}))"
        if k == "bin" and self.value == "like":
            return f"({self.args[0].sql()} like {self.args[1].sql()})"
        if k == "un":
            return f"({'-' if self.value == 'neg' else self.value} {self.args[0].sql()})"
        if k == "star":
            return "*"
        return f"{self.value}({', '.join(a.sql() for a in self.args)})"


def col(name): return Node("col", name)
def num(v): return Node("num", v)
def binop(op, a, b): return Node("bin", op, (a, b))


# ------------------------------------------------------------------ tokenizer / parser
_TOKEN = re.compile(r"\s*(?:(\d+\.\d*(?:[eE][-+]?\d+)?|\.\d+|\d+(?:[eE][-+]?\d+)?)|([A-Za-z_][A-Za-z_0-9.]*)|'((?:[^']|'')*)'|(<=|>=|<>|!=|==|[-+*/()<>=,]))")
_KEYWORDS = {"and", "or", "not", "between", "in", "as", "date", "interval", "cast", "is", "null", "like", "case", "when", "then",
             "else", "end", "extract", "from", "true", "false"}
_AGGS = {"sum", "avg", "min", "max", "count", "mean"}


def tokenize(s: str):
    pos, out = 0, []
    s = s.strip()
    while pos < len(s):
        m = _TOKEN.match(s, pos)
        if not m or m.end() == pos:
            raise ExprError(f"cannot tokenize {s[pos:pos + 20]!r}")
        if m.group(1) is not None:
            t = m.group(1)
            out.append(("num", float(t) if any(c in t for c in ".eE") else int(t)))
        elif m.group(2) is not None:
            w = m.group(2)
            out.append(("kw", w.lower()) if w.lower() in _KEYWORDS else ("id", w))
        elif m.group(3) is not None:
            out.append(("str", m.group(3).replace("''", "'")))
        else:
            out.append(("op", m.group(4)))
        pos = m.end()
    return out


class Parser:
    def __init__(self, text: str):
        self.toks = tokenize(text)
        self.i = 0

    def peek(self):
        return self.toks[self.i] if self.i < len(self.toks) else ("eof", None)

    def next(self):
        t = self.peek()
        self.i += 1
        return t

    def accept(self, kind, val=None):
        t = self.peek()
        if t[0] == kind and (val is None or t[1] == val):
            self.i += 1
            return True
        return False

    def expect(self, kind, val=None):
        if not self.accept(kind, val):
            raise ExprError(f"expected {val or kind}, got {self.peek()}")

    # precedence climbing: or < and < not < comparison < additive < multiplicative < unary
    def parse_or(self):
        e = self.parse_and()
        while self.accept("kw", "or"):
            e = binop("or", e, self.parse_and())
        return e

    def parse_and(self):
        e = self.parse_not()
        while self.accept("kw", "and"):
            e = binop("and", e, self.parse_not())
        return e

    def parse_not(self):
        if self.accept("kw", "not"):
            return Node("un", "not", (self.parse_not(),))
        return self.parse_cmp()

    def parse_cmp(self):
        e = self.parse_add()
        t = self.peek()
        if t[0] == "op" and t[1] in ("<", "<=", ">", ">=", "=", "==", "!=", "<>"):
            self.next()
            op = {"==": "=", "<>": "!="}.get(t[1], t[1])
            return binop(op, e, self.parse_add())
        neg = False
        if t == ("kw", "not"):
            nxt = self.toks[self.i + 1] if self.i + 1 < len(self.toks) else None
            if nxt in (("kw", "between"), ("kw", "in"), ("kw", "like")):
                self.next()
                neg = True
                t = self.peek()
        if t == ("kw", "like"):
            self.next()
            pat = self.next()
            if pat[0] != "str":
                raise ExprError("LIKE needs a string pattern")
            r = Node("bin", "like", (e, Node("str", pat[1])))
            return Node("un", "not", (r,)) if neg else r
        if t == ("kw", "between"):
            self.next()
            lo = self.parse_add()
            self.expect("kw", "and")
            hi = self.parse_add()
            r = binop("and", binop(">=", e, lo), binop("<=", e, hi))
            return Node("un", "not", (r,)) if neg else r
        if t == ("kw", "in"):
            self.next()
            self.expect("op", "(")
            items = [self.parse_add()]
            while self.accept("op", ","):
                items.append(self.parse_add())
            self.expect("op", ")")
            r = Node("func", "in", (e, *items))
            return Node("un", "not", (r,)) if neg else r
        return e

    def parse_add(self):
        e = self.parse_mul()
        while True:
            t = self.peek()
            if t[0] == "op" and t[1] in "+-":
                self.next()
                e = binop(t[1], e, self.parse_mul())
            else:
                return e

    def parse_mul(self):
        e = self.parse_unary()
        while True:
            t = self.peek()
            if t[0] == "op" and t[1] in "*/":
                self.next()
                e = binop(t[1], e, self.parse_unary())
            else:
                return e

    def parse_unary(self):
        if self.accept("op", "-"):
            return Node("un", "neg", (self.parse_unary(),))
        if self.accept("op", "+"):
            return self.parse_unary()
        return self.parse_atom()

    def parse_atom(self):
        t = self.next()
        if t[0] == "num":
            return num(t[1])
        if t[0] == "str":
            return Node("str", t[1])
        if t == ("op", "("):
            e = self.parse_or()
            self.expect("op", ")")
            return e
        if t == ("kw", "date"):
            s = self.next()
            if s[0] != "str":
                raise ExprError("date literal needs a string")
            return Node("date", (_dt.date.fromisoformat(s[1]) - _dt.date(1970, 1, 1)).days)
        if t == ("kw", "interval"):
            s = self.next()
            n = int(s[1]) if s[0] in ("str", "num") else None
            u = self.next()
            if n is None or u[0] != "id":
                raise ExprError("bad interval literal")
            unit = u[1].lower().rstrip("s")
            if unit not in ("day", "month", "year"):
                raise ExprError(f"unsupported interval unit {u[1]}")
            return Node("interval", (n, unit))
        if t in (("kw", "true"), ("kw", "false")):
            return num(1 if t[1] == "true" else 0)
        if t == ("kw", "case"):
            # CASE WHEN c1 THEN a1 [WHEN c2 THEN a2 ...] ELSE b END, nested right to left
            arms = []
            while self.accept("kw", "when"):
                c = self.parse_or()
                self.expect("kw", "then")
                arms.append((c, self.parse_or()))
            if not arms:
                raise ExprError("CASE needs at least one WHEN")
            if not self.accept("kw", "else"):
                raise ExprError("CASE without ELSE yields NULL, which the hot path does not carry")
            e = self.parse_or()
            self.expect("kw", "end")
            for c, a in reversed(arms):
                e = Node("func", "case", (c, a, e))
            return e
        if t == ("kw", "extract"):
            self.expect("op", "(")
            part = self.next()
            if part[0] != "id" or part[1].lower() not in ("year", "month", "day"):
                raise ExprError("EXTRACT supports year / month / day")
            self.expect("kw", "from")
            e = self.parse_add()
            self.expect("op", ")")
            return Node("func", "extract_" + part[1].lower(), (e,))
        if t == ("kw", "cast"):
            self.expect("op", "(")
            e = self.parse_or()
            self.expect("kw", "as")
            ty = self.next()
            self.expect("op", ")")
            tyname = str(ty[1]).lower()
            if tyname in ("int", "integer", "bigint", "int64", "int32"):
                return Node("func", "cast_int", (e,))
            if tyname in ("double", "float", "float64", "real"):
                return e
            raise ExprError(f"unsupported cast target {ty[1]}")
        if t[0] == "id":
            name = t[1]
            if self.accept("op", "("):
                fname = name.lower()
                if self.accept("op", "*"):
                    args = (Node("star"),)
                elif self.peek() == ("op", ")"):
                    args = ()
                else:
                    args = [self.parse_or()]
                    while self.accept("op", ","):
                        args.append(self.parse_or())
                    args = tuple(args)
                self.expect("op", ")")
                if fname in _AGGS:
                    return Node("agg", "avg" if fname == "mean" else fname, args)
                return Node("func", fname, args)
            return col(name)
        raise ExprError(f"unexpected token {t}")


def parse(text: str) -> Node:
    p = Parser(text)
    e = p.parse_or()
    if p.peek()[0] != "eof":
        raise ExprError(f"trailing tokens in {text!r}: {p.toks[p.i:]}")
    return fold(e)


def parse_select_list(text: str):
    """'expr as name, expr as name' -> [(Node, alias | None)].  Commas inside parentheses are kept."""
    p = Parser(text)
    out = []
    while True:
        e = p.parse_or()
        alias = None
        if p.accept("kw", "as"):
            t = p.next()
            if t[0] != "id":
                raise ExprError("alias must be an identifier")
            alias = t[1]
        out.append((fold(e), alias))
        if not p.accept("op", ","):
            break
    if p.peek()[0] != "eof":
        raise ExprError(f"trailing tokens in {text!r}")
    return out


# ------------------------------------------------------------------ constant folding (dates, intervals, numbers)
def _add_interval(days: int, n: int, unit: str, sign: int) -> int:
    d = _dt.date(1970, 1, 1) + _dt.timedelta(days=days)
    n *= sign
    if unit == "day":
        d = d + _dt.timedelta(days=n)
    else:
        months = d.year * 12 + (d.month - 1) + (n if unit == "month" else 12 * n)
        y, m = divmod(months, 12)
        # clamp the day like SQL engines do (DuckDB / Postgres)
        last = [31, 29 if (y % 4 == 0 and (y % 100 != 0 or y % 400 == 0)) else 28, 31, 30, 31, 30, 31, 31, 30, 31, 30, 31][m]
        d = _dt.date(y, m + 1, min(d.day, last))
    return (d - _dt.date(1970, 1, 1)).days


def fold(e: Node) -> Node:
    if not e.args:
        return e
    args = tuple(fold(a) for a in e.args)
    e = Node(e.kind, e.value, args)
    if e.kind == "bin" and e.value in "+-*/":
        a, b = args
        if a.kind == "date" and b.kind == "interval" and e.value in "+-":
            return Node("date", _add_interval(a.value, b.value[0], b.value[1], 1 if e.value == "+" else -1))
        if a.kind == "num" and b.kind == "num":
            v = {"+": a.value + b.value, "-": a.value - b.value, "*": a.value * b.value,
                 "/": (a.value / b.value) if b.value != 0 else float("nan")}[e.value]
            return num(v)
    if e.kind == "un" and e.value == "neg" and args[0].kind == "num":
        return num(-args[0].value)
    if e.kind == "bin" and e.value in _FLIP_CMP:
        r = _fold_extract_year(e)
        if r is not None:
            return r
    return e


_FLIP_CMP = {"<": ">", "<=": ">=", ">": "<", ">=": "<=", "=": "=", "!=": "!="}


def _fold_extract_year(e: Node):
    """extract(year from d) <cmp> Y  ->  a range test on the days-since-epoch value of d: the only use the judged
    queries make of EXTRACT in predicates, and a form row-group statistics can prune on."""
    a, b, op = e.args[0], e.args[1], e.value
    if not (a.kind == "func" and a.value == "extract_year"):
        a, b, op = b, a, _FLIP_CMP[op]
    if not (a.kind == "func" and a.value == "extract_year" and b.kind == "num" and float(b.value).is_integer()):
        return None
    y, d = int(b.value), a.args[0]
    if not 1 <= y <= 9998:
        return None
    start = Node("date", (_dt.date(y, 1, 1) - _dt.date(1970, 1, 1)).days)
    nxt = Node("date", (_dt.date(y + 1, 1, 1) - _dt.date(1970, 1, 1)).days)
    if op == "=":
        return binop("and", binop(">=", d, start), binop("<", d, nxt))
    if op == "!=":
        return binop("or", binop("<", d, start), binop(">=", d, nxt))
    return {"<": binop("<", d, start), "<=": binop("<", d, nxt), ">": binop(">=", d, nxt), ">=": binop(">=", d, start)}[op]


def integer_valued(e: Node) -> bool:
    """Expressions whose fp64 result is an exact integer by construction (usable as group keys after a cast)."""
    return e.kind == "func" and (e.value.startswith("extract_") or e.value == "cast_int")


def conjuncts(e: Node) -> list:
    """Top-level AND terms (the reference converts to CNF first, pyquokka/datastream.py:368-370; the
    judged predicates are already conjunctions)."""
    if e.kind == "bin" and e.value == "and":
        return conjuncts(e.args[0]) + conjuncts(e.args[1])
    return [e]


def and_all(terms: list) -> Node | None:
    out = None
    for t in terms:
        out = t if out is None else binop("and", out, t)
    return out


def rename(e: Node, mapping: dict) -> Node:
    if e.kind == "col":
        return col(mapping.get(e.value, e.value))
    return Node(e.kind, e.value, tuple(rename(a, mapping) for a in e.args))


def substitute(e: Node, defs: dict) -> Node:
    """Inline computed columns (with_columns) into an expression."""
    if e.kind == "col" and e.value in defs:
        return defs[e.value]
    return Node(e.kind, e.value, tuple(substitute(a, defs) for a in e.args))


# ------------------------------------------------------------------ compiler to postfix programs
@dataclass
class ColumnInfo:
    slot: int
    dtype: int                        # QK_*
    dictionary: list | None = None     # value list for dictionary-coded string columns
    is_date: bool = False


_CMP = {"<": L.CMP_LT, "<=": L.CMP_LE, ">": L.CMP_GT, ">=": L.CMP_GE, "=": L.CMP_EQ, "!=": L.CMP_NE}
_FLIP = {"<": ">", "<=": ">=", ">": "<", ">=": "<=", "=": "=", "!=": "!="}
_FCMP = {"<": L.OP_LT, "<=": L.OP_LE, ">": L.OP_GT, ">=": L.OP_GE, "=": L.OP_EQ, "!=": L.OP_NE}
_ARITH = {"+": L.OP_ADD, "-": L.OP_SUB, "*": L.OP_MUL, "/": L.OP_DIV}
_INT_DTYPES = (L.QK_U8, L.QK_I32, L.QK_I64)


_I64_MIN, _I64_MAX = -(1 << 63), (1 << 63) - 1
_ALWAYS, _NEVER = (L.CMP_GE, _I64_MIN), (L.CMP_LT, _I64_MIN)     # x >= INT64_MIN, x < INT64_MIN: true / false for every x


def lower_int_cmp(op: str, v) -> tuple:
    """(compare code, int64 immediate) of `x <op> v` for an integer column x and a numeric literal v (Python int or float),
    decided exactly, as Python compares an int with an int or a float: a fractional bound becomes the integer bound that
    selects the same rows (x < 2.5 is x <= 2), a literal outside int64 or a NaN / inf decides every row at once (NaN: every
    compare false, != true), and the result always fits the node's int64 immediate.  Without this an int64 column would be
    compared in fp64 (1.7e18 + 1 rounds to 1.7e18) or against a literal that wraps when it is stored."""
    if isinstance(v, float):
        if math.isnan(v):
            return _ALWAYS if op == "!=" else _NEVER
        if math.isinf(v):
            v = _I64_MAX + 1 if v > 0 else _I64_MIN - 1      # beyond every x, like any literal outside int64
        elif not v.is_integer():
            if op in ("=", "!="):
                return _ALWAYS if op == "!=" else _NEVER
            op, v = ("<=", math.floor(v)) if op in ("<", "<=") else (">=", math.ceil(v))
    v = int(v)
    if v > _I64_MAX:
        return _ALWAYS if op in ("<", "<=", "!=") else _NEVER
    if v < _I64_MIN:
        return _ALWAYS if op in (">", ">=", "!=") else _NEVER
    return _CMP[op], v


def compile_expr(e: Node, schema: dict) -> list:
    """Postfix program [(op, a0, a1, imm, imm_i)] over the column slots in `schema` (name -> ColumnInfo)."""
    out: list = []

    def ci(name) -> ColumnInfo:
        if name not in schema:
            raise ExprError(f"unknown column {name!r}; available: {sorted(schema)}")
        return schema[name]

    def emit(n: Node):
        k = n.kind
        if k == "col":
            out.append((L.OP_COL, ci(n.value).slot, 0, 0.0, 0))
        elif k == "num":
            out.append((L.OP_CONST, 0, 0, float(n.value), 0))
        elif k == "date":
            out.append((L.OP_CONST, 0, 0, float(n.value), 0))
        elif k == "str":
            raise ExprError("a string literal can only be compared with a dictionary column")
        elif k == "interval":
            raise ExprError("interval arithmetic must fold to a date literal")
        elif k == "un":
            emit(n.args[0])
            out.append((L.OP_NEG if n.value == "neg" else L.OP_NOT, 0, 0, 0.0, 0))
        elif k == "func":
            if n.value == "cast_int":
                emit(n.args[0])
                out.append((L.OP_RINT, 0, 0, 0.0, 0))
            elif n.value == "case":
                # cond then else SELECT: the condition is evaluated once; both arms are evaluated for every row but an
                # unselected arm that is inf / NaN does not reach the result
                c, a, b = n.args
                emit(c); emit(a); emit(b)
                out.append((L.OP_SELECT, 0, 0, 0.0, 0))
            elif n.value == "in":
                emit_in(n.args[0], n.args[1:])
            elif n.value.startswith("extract_"):
                # EXTRACT(year | month | day FROM date) as a VALUE (group keys, select lists); comparisons of the year with a
                # constant never get here: fold() turned them into date ranges
                emit(n.args[0])
                out.append((L.OP_EXTRACT, 0, {"year": 0, "month": 1, "day": 2}[n.value[8:]], 0.0, 0))
            else:
                raise ExprError(f"unsupported function {n.value}")
        elif k == "bin":
            a, b = n.args
            op = n.value
            if op in _ARITH:
                emit(a); emit(b)
                out.append((_ARITH[op], 0, 0, 0.0, 0))
            elif op in ("and", "or"):
                start = len(out)
                emit(a)
                mid = len(out)
                emit(b)
                if op == "and" and mid - start == 1 and len(out) - mid == 1:
                    merged = _merge_ranges(out[start], out[mid])          # x >= a AND x < b on one integer column: ONE range node
                    if merged is not None:
                        del out[start:]
                        out.append(merged)
                        return
                out.append((L.OP_AND if op == "and" else L.OP_OR, 0, 0, 0.0, 0))
            elif op in _CMP:
                emit_cmp(op, a, b)
            elif op == "like":
                emit_like(a, b)
            else:
                raise ExprError(f"unsupported operator {op}")
        else:
            raise ExprError(f"cannot compile {k} node here")

    def emit_like(a, b):
        """col LIKE 'pattern' on a dictionary-coded column: the pattern is matched against the dictionary on the
        host, the row test is `code in {matching codes}` (pyquokka/sql_utils.py:131-149 handles the same four shapes
        through Polars string kernels)."""
        if a.kind != "col" or ci(a.value).dictionary is None:
            raise ExprError("LIKE needs a dictionary-coded string column on the left")
        info = ci(a.value)
        rx = re.compile("".join(".*" if ch == "%" else "." if ch == "_" else re.escape(ch) for ch in b.value), re.S)
        emit_set(info, [i for i, v in enumerate(info.dictionary) if isinstance(v, str) and rx.fullmatch(v)])

    def emit_set(info, codes):
        """`code in {codes}` as ONE node whatever the size of the set: a bitmap indexed by the code (QK_OP_IN_SET).  The
        bitmap travels as a Python int in imm_i; ops._Progs keeps it inline when it spans <= 64 bits and uploads it to
        the device otherwise."""
        codes = sorted(set(int(c) for c in codes if c >= 0))
        if not codes:
            out.append((L.OP_CMP_COL_IMM, info.slot, L.CMP_EQ, 0.0, -1))
        elif len(codes) == 1:
            out.append((L.OP_CMP_COL_IMM, info.slot, L.CMP_EQ, 0.0, codes[0]))
        else:
            bitmap = 0
            for c in codes:
                bitmap |= 1 << c
            out.append((L.OP_IN_SET, info.slot, codes[-1] + 1, 0.0, bitmap))

    def emit_in(a, items):
        """x IN (literals): dictionary columns resolve the strings to codes, small non-negative integer sets become one
        bitmap test, anything else is the OR-chain of equalities the reference's sqlglot tree also is."""
        if a.kind == "col":
            info = ci(a.value)
            if info.dictionary is not None and all(it.kind == "str" for it in items):
                emit_set(info, [info.dictionary.index(it.value) for it in items if it.value in info.dictionary])
                return
            if info.dtype in _INT_DTYPES and all(it.kind in ("num", "date") for it in items):
                # the integers the column can equal: a fractional, NaN, infinite or out-of-int64 literal matches no row
                vals = [v for c, v in (lower_int_cmp("=", it.value) for it in items) if c == L.CMP_EQ]
                if vals and all(0 <= v < (1 << 16) for v in vals):
                    emit_set(info, vals)
                    return
        for j, it in enumerate(items):
            emit_cmp("=", a, it)
            if j:
                out.append((L.OP_OR, 0, 0, 0.0, 0))

    def emit_cmp(op, a, b):
        if a.kind != "col" and b.kind == "col":
            a, b, op = b, a, _FLIP[op]
        if a.kind == "col":
            info = ci(a.value)
            if b.kind == "str":
                if info.dictionary is None:
                    raise ExprError(f"column {a.value} is not dictionary-coded; cannot compare with a string")
                if op not in ("=", "!="):
                    raise ExprError("only = / != are supported against string literals")
                code = info.dictionary.index(b.value) if b.value in info.dictionary else -1
                out.append((L.OP_CMP_COL_IMM, info.slot, _CMP[op], 0.0, code))
                return
            if info.dtype in _INT_DTYPES and b.kind in ("num", "date"):
                cmp, v = lower_int_cmp(op, b.value)
                out.append((L.OP_CMP_COL_IMM, info.slot, cmp, 0.0, v))
                return
            if info.dtype in _INT_DTYPES and b.kind == "col" and ci(b.value).dtype in _INT_DTYPES:
                out.append((L.OP_CMP_COL_COL, info.slot, _CMP[op] | (ci(b.value).slot << 8), 0.0, 0))
                return
        emit(a); emit(b)
        out.append((_FCMP[op], 0, 0, 0.0, 0))

    emit(e)
    check_program(out)
    return out


def _as_range(node):
    """(slot, lo, hi) of a non-negated integer range node, or None."""
    op, a0, a1, imm, imm_i = node
    if op == L.OP_RANGE_COL_IMM and not a1:
        return a0, int(imm_i), int(imm)
    if op == L.OP_CMP_COL_IMM:
        v = int(imm_i)
        if a1 == L.CMP_LT: return a0, _I64_MIN, v - 1
        if a1 == L.CMP_LE: return a0, _I64_MIN, v
        if a1 == L.CMP_GT: return a0, v + 1, _I64_MAX
        if a1 == L.CMP_GE: return a0, v, _I64_MAX
        if a1 == L.CMP_EQ: return a0, v, v
    return None


def _merge_ranges(x, y):
    """Two range tests on the same integer column, ANDed -> one QK_OP_RANGE_COL_IMM node (closed interval), when both bounds are
    finite and fit the node (|bound| <= 2^53: the upper bound travels in the node's fp64 immediate)."""
    rx, ry = _as_range(x), _as_range(y)
    if rx is None or ry is None or rx[0] != ry[0]:
        return None
    lo, hi = max(rx[1], ry[1]), min(rx[2], ry[2])
    if lo > hi:
        lo, hi = 1, 0                               # empty
    if abs(lo) > (1 << 53) or abs(hi) > (1 << 53):
        return None
    return (L.OP_RANGE_COL_IMM, rx[0], 0, float(hi), lo)


def check_program(prog, what: str = "expression") -> None:
    """The limits the kernels enforce (include/qk.h QK_MAX_EXPR_NODES / QK_MAX_STACK; csrc/scan.cu pack_programs):
    checked where the program is made, so that the planner fails on the host -- and in the CPU test shim -- exactly where
    the device library would."""
    if len(prog) > L.MAX_EXPR_NODES:
        raise ExprError(f"{what} compiles to {len(prog)} nodes; the scan kernels take at most {L.MAX_EXPR_NODES}")
    depth = 0
    for op, _a0, _a1, imm, imm_i in prog:
        # an integer immediate is stored in an int64 field, which would wrap a larger one silently (lower_int_cmp keeps the
        # compiler's inside it); a range's upper bound travels in the fp64 immediate, exact up to 2^53
        if op in (L.OP_CMP_COL_IMM, L.OP_RANGE_COL_IMM) and not _I64_MIN <= int(imm_i) <= _I64_MAX:
            raise ExprError(f"{what}: integer immediate {imm_i} outside int64")
        if op == L.OP_RANGE_COL_IMM and not -(1 << 53) <= imm <= (1 << 53):
            raise ExprError(f"{what}: range upper bound {imm} outside +-2^53")
        if op in (L.OP_COL, L.OP_CONST, L.OP_CMP_COL_IMM, L.OP_CMP_COL_COL, L.OP_IN_SET, L.OP_RANGE_COL_IMM):
            depth += 1
        elif op == L.OP_SELECT:
            depth -= 2
        elif op not in (L.OP_NEG, L.OP_NOT, L.OP_RINT, L.OP_EXTRACT):
            depth -= 1
        if depth > L.MAX_STACK:
            raise ExprError(f"{what} needs more than {L.MAX_STACK} stack slots")


def check_call(ncols: int, pred, exprs, who: str = "scan") -> None:
    """What csrc/scan.cu pack_programs accepts for ONE kernel call: <= MAX_COLS input columns, <= MAX_PROJ expressions,
    <= MAX_EXPR_NODES nodes each, <= MAX_TOTAL_NODES nodes together, <= MAX_STACK stack slots.  Shared by quokka_b200.ops
    and the CPU test shim, so that a plan the device library would refuse also fails on the host."""
    if ncols > L.MAX_COLS:
        raise ExprError(f"{who}: {ncols} input columns; one kernel call takes at most {L.MAX_COLS}")
    exprs = list(exprs or [])
    if len(exprs) > L.MAX_PROJ:
        raise ExprError(f"{who}: {len(exprs)} expressions; one kernel call takes at most {L.MAX_PROJ}")
    total = 0
    for k, prog in enumerate([pred] + exprs):
        prog = prog or []
        check_program(prog, f"{who}: expression {k}")
        total += len(prog)
        for op, a0, a1, *_ in prog:
            slots = [a0] if op in (L.OP_COL, L.OP_CMP_COL_IMM, L.OP_IN_SET, L.OP_RANGE_COL_IMM) else [a0, a1 >> 8] if op == L.OP_CMP_COL_COL else []
            if any(not 0 <= s_ < ncols for s_ in slots):
                raise ExprError(f"{who}: column slot out of range in expression {k}")
    if total > L.MAX_TOTAL_NODES:
        raise ExprError(f"{who}: programs hold {total} nodes in total; one kernel call takes at most {L.MAX_TOTAL_NODES}")


# ------------------------------------------------------------------ pattern predicates (OrderedStream.pattern_recognize)
@dataclass
class PatternPredicates:
    """The events of a pattern, split the way the search runs them.  local[e]: the conjuncts of event e that read only the row
    being bound (plain column names), or None = every row; link[e]: the conjuncts that read an earlier event's row, whose columns
    are `name.col` (that event's bound row) or `col` (the row being bound), or None."""
    names: list
    local: list
    link: list
    columns: set


def split_pattern(events, schema, by: str) -> PatternPredicates:
    """Resolves the `name.col` qualifiers of every event predicate (the event's own name = the row being bound, an earlier
    event's name = that event's bound row) and splits each predicate into row-local and link conjuncts (the reference's
    event_prefilters / event_dependent_filters, pyquokka/executors/cep_executors.py:35-75).  A reference to a later event, an
    unknown event or column, a repeated or malformed name, or a missing predicate after the first event is an ExprError."""
    events = list(events)
    if not 2 <= len(events) <= L.PATTERN_MAX_EVENTS:
        raise ExprError(f"a pattern has 2 to {L.PATTERN_MAX_EVENTS} events, got {len(events)}")
    names = []
    for ev in events:
        if not (isinstance(ev, (tuple, list)) and len(ev) == 2):
            raise ExprError("every event is a (name, predicate) pair")
        name = ev[0]
        if not isinstance(name, str) or not re.fullmatch(r"[A-Za-z_][A-Za-z_0-9]*", name):
            raise ExprError(f"event name {name!r} must be an identifier without '.'")
        if name in names:
            raise ExprError(f"event name {name!r} is used for two events")
        if name == by:
            raise ExprError(f"event name {name!r} equals the `by` column")
        names.append(name)
    schema = set(schema)
    local, link, columns = [], [], set()
    for i, (name, pred) in enumerate(events):
        if pred is None:
            if i > 0:
                raise ExprError(f"event {name!r}: only the first event may have no predicate")
            local.append(None)
            link.append(None)
            continue
        node = parse(pred) if isinstance(pred, str) else getattr(pred, "node", pred)
        if not isinstance(node, Node):
            raise ExprError(f"event {name!r}: a predicate is a SQL string or an Expression")

        def resolve(n):
            if n.kind != "col":
                return Node(n.kind, n.value, tuple(resolve(a) for a in n.args)) if n.args else n
            q, c = n.value.split(".", 1) if "." in n.value else (None, n.value)
            if q is not None and q != name:
                if q not in names:
                    raise ExprError(f"event {name!r}: {n.value!r} names no event")
                if names.index(q) > i:
                    raise ExprError(f"event {name!r}: {n.value!r} refers to the later event {q!r}")
            if c not in schema:
                raise ExprError(f"event {name!r}: unknown column {c!r}")
            columns.add(c)
            return col(c if q is None or q == name else f"{q}.{c}")

        terms = conjuncts(resolve(node))
        loc = [t for t in terms if not any("." in c for c in t.columns())]
        lnk = [t for t in terms if any("." in c for c in t.columns())]
        local.append(and_all(loc))
        link.append(and_all(lnk))
    return PatternPredicates(names, local, link, columns)


def pattern_prefilter(p: PatternPredicates):
    """The OR of the events' row-local parts (cep_executors.py:77-81): a row it rejects can bind no event.  None when an event
    has no row-local part, or when the parts read different columns -- a filter over a column that may hold NULLs drops every
    row where it reads one, which is only right when every event would read that column too."""
    if any(x is None for x in p.local) or len({frozenset(x.columns()) for x in p.local}) != 1:
        return None
    out = None
    for x in p.local:
        out = x if out is None else binop("or", out, x)
    return out


def compile_link(e: Node, ev: int, names: list, slots: dict, schema: dict) -> list:
    """Postfix program of event `ev`'s link conjuncts for qk_pattern_search: QK_OP_COL a0 = slots[column], a1 = the event whose
    bound row is read (ev for the row being bound).  Only arithmetic, NEG, the float compares, AND / OR / NOT and CASE, in fp64;
    string columns and literals are rejected."""
    out: list = []

    def emit(n: Node):
        k = n.kind
        if k == "col":
            q, c = n.value.split(".", 1) if "." in n.value else (names[ev], n.value)
            if names.index(q) > ev:
                raise ExprError(f"event {names[ev]!r}: {n.value!r} refers to a later event")
            info = schema[c]
            if info.dictionary is not None:
                raise ExprError(f"event {names[ev]!r}: string column {c!r} cannot be read across events")
            out.append((L.OP_COL, slots[c], names.index(q), 0.0, 0))
        elif k in ("num", "date"):
            out.append((L.OP_CONST, 0, 0, float(n.value), 0))
        elif k == "un":
            emit(n.args[0])
            out.append((L.OP_NEG if n.value == "neg" else L.OP_NOT, 0, 0, 0.0, 0))
        elif k == "bin" and n.value in _ARITH:
            emit(n.args[0]); emit(n.args[1])
            out.append((_ARITH[n.value], 0, 0, 0.0, 0))
        elif k == "bin" and n.value in _FCMP:
            emit(n.args[0]); emit(n.args[1])
            out.append((_FCMP[n.value], 0, 0, 0.0, 0))
        elif k == "bin" and n.value in ("and", "or"):
            emit(n.args[0]); emit(n.args[1])
            out.append((L.OP_AND if n.value == "and" else L.OP_OR, 0, 0, 0.0, 0))
        elif k == "func" and n.value == "case":
            for a in n.args:
                emit(a)
            out.append((L.OP_SELECT, 0, 0, 0.0, 0))
        else:
            raise ExprError(f"event {names[ev]!r}: {n.sql()} is not supported in a predicate that reads an earlier event "
                            "(arithmetic, comparisons, AND / OR / NOT and CASE over numeric columns)")

    emit(e)
    check_program(out, f"event {names[ev]!r}")
    return out


def compile_links(p: PatternPredicates, schema: dict | None = None):
    """(link columns, one program per event) for qk_pattern_search, with the limits the kernel enforces: at most QK_MAX_COLS link
    columns and PATTERN_MAX_LINK_NODES nodes over all programs.  schema = None checks a plan before any row has arrived: every
    column is taken as numeric, so only a string column is left to be found when the rows' types are known."""
    lcols = sorted({c.split(".", 1)[-1] for x in p.link if x is not None for c in x.columns()})
    if len(lcols) > L.MAX_COLS:
        raise ExprError(f"pattern: predicates that read earlier events read {len(lcols)} columns; at most {L.MAX_COLS}")
    if schema is None:
        schema = {c: ColumnInfo(i, L.QK_F64) for i, c in enumerate(lcols)}
    slots = {c: i for i, c in enumerate(lcols)}
    links = [compile_link(x, e, p.names, slots, schema) if x is not None else [] for e, x in enumerate(p.link)]
    total = sum(len(x) for x in links)
    if total > L.PATTERN_MAX_LINK_NODES:
        raise ExprError(f"pattern: predicates that read earlier events compile to {total} nodes; at most {L.PATTERN_MAX_LINK_NODES}")
    return lcols, links
