"""The dense-aggregate reference and plan generator (tests/dense_agg_cases.py) on the CPU: the reference against a per-row
Python evaluation of the compiled programs, the CPU shim's DenseAggState against the reference, and the routing of
dictionary groupings that the dense kernel cannot hold (edge.PartialAgg -> ops.dense_agg_fits)."""
import math

import numpy as np
import pytest
import torch

import cpu_shim
import dense_agg_cases as D
from quokka_b200 import _lib as L


# ------------------------------------------------------------------ per-row brute force over the compiled programs
def _row_eval(prog, row):
    """One row of a postfix program (include/qk.h QK_OP_*), in Python floats / ints: an evaluation independent of the
    numpy reference, so a plan whose SQL text and numpy meaning disagree fails here."""
    st = []
    cmp = [lambda a, b: a < b, lambda a, b: a <= b, lambda a, b: a > b, lambda a, b: a >= b, lambda a, b: a == b, lambda a, b: a != b]
    for op, a0, a1, imm, imm_i in prog:
        if op == L.OP_COL:
            st.append(float(row[a0]))
        elif op == L.OP_CONST:
            st.append(float(imm))
        elif op in (L.OP_ADD, L.OP_SUB, L.OP_MUL):
            b, a = st.pop(), st.pop()
            try:
                st.append(a + b if op == L.OP_ADD else a - b if op == L.OP_SUB else a * b)
            except OverflowError:
                st.append(math.copysign(math.inf, a) * math.copysign(1.0, b))
        elif op == L.OP_NEG:
            st.append(-st.pop())
        elif L.OP_LT <= op <= L.OP_NE:
            b, a = st.pop(), st.pop()
            st.append(1.0 if cmp[op - L.OP_LT](a, b) else 0.0)
        elif op == L.OP_AND:
            b, a = st.pop(), st.pop()
            st.append(1.0 if a != 0 and b != 0 else 0.0)
        elif op == L.OP_NOT:
            st.append(1.0 if st.pop() == 0 else 0.0)
        elif op == L.OP_SELECT:
            b, a, c = st.pop(), st.pop(), st.pop()
            st.append(a if c != 0 else b)
        elif op == L.OP_IN_SET:
            code = int(row[a0])
            st.append(1.0 if 0 <= code < a1 and (int(imm_i) >> code) & 1 else 0.0)
        elif op == L.OP_CMP_COL_IMM:
            st.append(1.0 if cmp[a1](int(row[a0]), int(imm_i)) else 0.0)
        elif op == L.OP_RANGE_COL_IMM:
            x = int(row[a0])
            st.append(1.0 if (int(imm_i) <= x <= int(imm)) != bool(a1) else 0.0)
        elif op == L.OP_CMP_COL_COL:
            st.append(1.0 if cmp[a1 & 0xff](int(row[a0]), int(row[a1 >> 8])) else 0.0)
        else:
            raise ValueError(op)
    assert len(st) == 1
    return st[0]


def _brute(plan, d):
    names, pred, gslots, progs = D.compile_plan(plan, d)
    n = len(d[names[0]])
    cols = [d[c] for c in names]
    ng = plan.n_groups
    cnt = [0] * ng
    vals = [[[] for _ in plan.aggs] for _ in range(ng)]
    for i in range(n):
        row = [c[i].item() for c in cols]
        if pred is not None and _row_eval(pred, row) == 0:
            continue
        g = 0
        for s, card in zip(gslots, plan.cards):
            g = g * card + int(row[s])
        cnt[g] += 1
        for j, p in enumerate(progs):
            vals[g][j].append(_row_eval(p, row))
    acc = np.zeros((ng, max(1, len(plan.aggs))))
    for g in range(ng):
        for j, a in enumerate(plan.aggs):
            v = [x for x in vals[g][j] if not (a.op != "sum" and math.isnan(x))]
            if a.op == "sum":
                fin = all(math.isfinite(x) for x in v)
                acc[g, j] = math.fsum(v) if fin else sum(v)
            else:
                acc[g, j] = (min(v) if a.op == "min" else max(v)) if v else (math.inf if a.op == "min" else -math.inf)
    return acc, np.array(cnt)


@pytest.mark.parametrize("seed", range(12))
def test_reference_matches_per_row_evaluation(seed):
    """Generated plans (both walks' type mixes, both data modes) at 300 rows: mask, group id and every per-row value of
    the reference equal a row-by-row evaluation of the programs expr.compile_expr makes from the plan's SQL text."""
    rng = np.random.default_rng(seed)
    mode = "dyadic" if seed % 3 else "tpch"
    d = D.make_data(300, 1000 + seed, mode)
    for k in range(6):
        plan = D.random_plan(rng, d, fast=bool(k % 2))
        ref = D.reference(plan, d)
        acc, cnt = _brute(plan, d)
        D.check(plan, acc, cnt, ref, exact=True, tag=f"seed {seed} plan {k}")


def test_reference_edges_per_row():
    """Hand-made edges the generator seldom draws: open / closed fp bounds at a value and its nextafter neighbours, ±0,
    NaN, ±inf data and constants, the smallest subnormal, int32 columns against constants beyond ±2^31, int64 columns at
    their extremes, an empty BETWEEN, 64- and 65-bit sets with codes beyond the set and negative codes, NOT of every
    kind, and MIN / MAX over NaN (skipped) and ±0."""
    c = 0.5
    f = np.array([c, np.nextafter(c, 1), np.nextafter(c, 0), 0.0, -0.0, np.nan, np.inf, -np.inf, 5e-324, -5e-324, 1.0, -1.0])
    n = len(f)
    d = {"f": f, "i32": np.array([D.I32_MIN, D.I32_MAX, 0, -1, 1, 7, 8, 9, 100, -100, 3, 4], np.int32),
         "i64": np.array([D.I64_MIN, D.I64_MAX, 0, -1, 1, 7, 8, 9, 100, -100, 3, 4], np.int64),
         "c32": np.array([-1, 0, 1, 63, 64, 65, 200, 2, 3, 4, 5, 6], np.int32),
         "k": (np.arange(n) % 3).astype(np.uint8)}
    terms = [D.fcmp("f", op, k) for op in D.CMPS for k in (c, np.inf, -np.inf, 0.0, -0.0, 5e-324)] + \
            [D.irange("i32", op, k) for op in D.CMPS for k in (D.I32_MIN - 1, D.I32_MAX + 1, 1 << 40, -(1 << 40), 7)] + \
            [D.irange("i64", op, k) for op in D.CMPS for k in (D.I64_MIN, D.I64_MAX, 0)] + \
            [D.between("i32", 9, 3), D.inset("c32", range(0, 64, 3)), D.inset("c32", [0, 64]), D.inset("c32", [1, 63]),
             D.colcol("i32", "<", "i64")]
    aggs = [D.Agg("sum", [D.f_col("f")]), D.Agg("min", [D.f_col("f")]), D.Agg("max", [D.f_neg("f")]),
            D.Agg("sum", [D.f_kminus(1.0, "f"), D.f_col("f")])]
    for t in terms + [t.negate() for t in terms]:
        plan = D.Plan([t], [("k", 3)], aggs)
        acc, cnt = _brute(plan, d)
        D.check(plan, acc, cnt, D.reference(plan, d), exact=True)


@pytest.mark.parametrize("mode", ["dyadic", "tpch"])
@pytest.mark.parametrize("seed", range(4))
def test_cpu_shim_dense_state_matches_reference(mode, seed):
    """cpu_shim.DenseAggState, which the CPU suite's DataStream programs run on, against the reference for generated plans:
    bit for bit on dyadic data, within n_g * 2^-53 * sum|x| on TPC-H data; then two batches into one state (MIN / MAX of
    groups first seen in the second batch)."""
    rng = np.random.default_rng(100 + seed)
    n = 20_000
    d = D.make_data(n, 2000 + seed, mode)
    for k in range(25):
        plan = D.random_plan(rng, d, fast=bool(k % 2))
        names, pred, gslots, progs = D.compile_plan(plan, d)
        st = cpu_shim.DenseAggState(plan.cards, plan.agg_ops, "cpu")
        st.update([torch.from_numpy(d[c]) for c in names], pred, gslots, progs)
        D.check(plan, st.acc.numpy(), st.cnt.numpy(), D.reference(plan, d), exact=mode == "dyadic", tag=f"shim {k}")
    # batches: the first one only holds group 0 of the first key
    plan = D.Plan([D.fcmp("fa", ">", -3.0)], [("k8a", 3), ("k8b", 2)],
                  [D.Agg("min", [D.f_col("fb")]), D.Agg("max", [D.f_col("fb"), D.f_col("fc")]), D.Agg("sum", [D.f_col("fc")])])
    names, pred, gslots, progs = D.compile_plan(plan, d)
    first = d["k8a"] == 0
    st = cpu_shim.DenseAggState(plan.cards, plan.agg_ops, "cpu")
    for sel in (first, ~first):
        st.update([torch.from_numpy(np.ascontiguousarray(d[c][sel])) for c in names], pred, gslots, progs)
    D.check(plan, st.acc.numpy(), st.cnt.numpy(), D.reference(plan, d), exact=mode == "dyadic", tag="batches")


def test_cpu_shim_min_max_skip_nan_like_the_kernels():
    """agg_combine is fmin / fmax: a NaN row does not poison a group's MIN / MAX, a group of NaN rows keeps the identity."""
    v = np.array([np.nan, 2.0, -1.0, np.nan, np.nan, 0.0, -0.0])
    g = np.array([0, 0, 0, 1, 1, 2, 2], np.uint8)
    progs = [[(L.OP_COL, 0, 0, 0.0, 0)], [(L.OP_COL, 0, 0, 0.0, 0)]]
    st = cpu_shim.DenseAggState([3], [L.AGG_MIN, L.AGG_MAX], "cpu")
    st.update([torch.from_numpy(v), torch.from_numpy(g)], None, [1], progs)
    acc = st.acc.numpy()
    assert acc[0].tolist() == [-1.0, 2.0] and acc[1].tolist() == [math.inf, -math.inf] and acc[2].tolist() == [0.0, 0.0]


def test_dense_agg_fits_is_the_interpreters_bound():
    from quokka_b200 import ops
    for nagg in range(L.MAX_AGGS + 1):
        top = 200 * 1024 // ((nagg * 8 + 4) * 256)
        assert ops.dense_agg_fits(top, nagg) and not ops.dense_agg_fits(top + 1, nagg), nagg
    assert [200 * 1024 // ((a * 8 + 4) * 256) for a in (0, 1, 4)] == [200, 66, 22]
    assert not ops.dense_agg_fits(0, 1) and not ops.dense_agg_fits(1, L.MAX_AGGS + 1)


@pytest.fixture
def qc(monkeypatch):
    cpu_shim.install(monkeypatch)
    from quokka_b200.df import QuokkaContext
    return QuokkaContext()


@pytest.mark.parametrize("pred", D.ROUTING_PREDS)
@pytest.mark.parametrize("nsum", D.ROUTING_AGGS)
@pytest.mark.parametrize("n_groups", D.ROUTING_GROUPS)
def test_dictionary_groupby_routing(qc, monkeypatch, n_groups, nsum, pred):
    """groupby(<dictionary column>) of 66, 67, 150 and 1 024 values: the partial aggregate takes the dense kernel only
    when ops.dense_agg_fits says the interpreter can hold the grouping, else the per-row path; the result equals pandas
    either way (it raised `groups x aggregates exceed the shared-memory dense path` before)."""
    from quokka_b200 import ops
    paths = D.routing_case(qc, monkeypatch, n_groups, nsum, pred)
    want = "shim-dense" if ops.dense_agg_fits(n_groups, nsum) else "rows"
    assert set(paths) == {want}, (paths, n_groups, nsum)
