"""Every device path of qk_scan_filter_project against the exact reference of tests/scan_cases.py:
- the stable interpreter (k_filter_count -> k_count_offsets -> k_filter_project_stable): bit-exact, in input order;
- the unordered interpreter (k_filter_project_unordered): the same multiset of rows;
- the TMA compaction (csrc/compact.cu, "compact_tma"), reached by an integer compare / range (or no predicate) and 1-8
  verbatim 16-byte aligned columns: bit-exact, in input order;
- its fall-backs to the interpreter: a misaligned view (t[1:]), more than 8 columns, an expression projection;
- the Bloom-reduced compaction (qk_scan_filter_project_sj, "compact_tma+bloom"): no false negatives, survivors in order.
After every call with rows the test asserts which kernel ran.  Sizes cover the warp, CTA, chunk (2048 rows) and TMA tile
edges, two carries of k_count_offsets' 1024-chunk tiles (4 300 000 rows), and 2^31 - 1 rows of uint8 (the largest call)."""
import functools

import numpy as np
import pytest
import torch

import scan_cases as S

pytestmark = pytest.mark.gpu

RANDOM = S.random_cases(120)
COMPACT = S.compact_cases(24)
_ids = lambda cs: [c.name for c in cs]      # noqa: E731


@pytest.fixture(scope="module")
def qk():
    from quokka_b200 import _lib, ops
    _lib.lib()
    return ops


@functools.lru_cache(maxsize=2)
def data(n, seed=0):
    return S.make_data(n, seed)


def device_columns(d, misaligned=False):
    """the columns in slot order; misaligned = views that start one element into their allocation"""
    out = []
    for c in S.COLUMNS:
        t = torch.from_numpy(d[c]).cuda()
        if misaligned:
            buf = torch.empty(len(t) + 1, dtype=t.dtype, device=t.device)
            buf[1:] = t
            t = buf[1:]
        out.append(t)
    return out


def run_paths(qk, case, d, misaligned_too=True, tag=""):
    """Runs `case` on every path that can take it and checks each against the reference."""
    n = len(d["rid"])
    mask, exp = S.reference(case, d)
    pred, projs = S.compile_case(case)
    shaped = S.compact_shaped(pred, projs)
    for misaligned in (False, True) if misaligned_too else (False,):
        cols = device_columns(d, misaligned)
        for stable in (True, False):
            outs, m = qk.scan_filter_project(cols, pred, projs, stable=stable)
            got = [o.cpu().numpy() for o in outs]
            variant = qk.last_variant()
            where = f"{tag} {case.name} n={n} stable={stable} misaligned={misaligned} via {variant}"
            if n > 0:
                assert variant == ("compact_tma" if shaped and not misaligned else "filter_interpreter"), where
            assert m == int(mask.sum()), where
            if stable or variant == "compact_tma":
                for p, g, e in zip(case.projs, got, exp):
                    assert S.same(g, e), f"{where}: {p}"
            else:
                assert np.array_equal(S.row_keys(got), S.row_keys(exp)), where


# ------------------------------------------------------------------ hand-written and generated cases
@pytest.mark.parametrize("n", [1, 257, 4099])
@pytest.mark.parametrize("case", S.EDGE_CASES, ids=_ids(S.EDGE_CASES))
def test_edge_cases(qk, case, n):
    run_paths(qk, case, data(n, 3))


@pytest.mark.parametrize("case", RANDOM, ids=_ids(RANDOM))
def test_random_cases(qk, case):
    run_paths(qk, case, data(3001, 4))


@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, 255, 256, 257, 2047, 2048, 2049, 100_003])
def test_sizes(qk, n):
    by = {c.name: c for c in S.EDGE_CASES}
    for name in ("near_gt", "set_77_bits", "arith", "count_only_interp", "count_only_cmp", "all_columns", "dict_like_wide",
                 "lit_2p63_lt", "range_empty"):
        run_paths(qk, by[name], data(n, 5))


@pytest.mark.parametrize("case", COMPACT, ids=_ids(COMPACT))
def test_compact_tile_edges(qk, case):
    """every generated compaction case at the edges of its TMA tile (one CTA's chunk is a whole number of tiles; the last
    chunk's ragged tail is read from global memory)"""
    tile = S.compact_tile_rows(case.projs)
    for n in (tile - 1, tile, tile + 1, 3 * tile + 17):
        run_paths(qk, case, data(n, 6), misaligned_too=n == tile + 1)


@pytest.mark.parametrize("n", [1_000_003, 4_300_000])
def test_large(qk, n):
    """Above 2 097 152 rows the stable interpreter's chunk-count scan walks more than one 1024-chunk tile and carries its
    running total from one to the next."""
    d = data(n, 7)
    by = {c.name: c for c in S.EDGE_CASES}
    for case in (by["near_gt"], by["arith"], by["count_only_interp"], by["set_65_bits"], by["colcol"],
                 S.Case("sparse", "i64 = 0 or u8 = 77", ("rid", "f64")), S.Case("sparse_compact", "u8 = 77", ("rid", "c150"))):
        run_paths(qk, case, d, tag="large")


# ------------------------------------------------------------------ fall-backs out of the TMA compaction
def test_more_than_8_columns_fall_back(qk):
    d = data(20_011, 8)
    case = S.Case("nine_columns", "c3 != 1", tuple(S.COLUMNS)[:9])
    assert not S.compact_shaped(*S.compile_case(case))
    run_paths(qk, case, d)
    eight = S.Case("eight_columns", "c3 != 1", tuple(S.COLUMNS)[:8])
    assert S.compact_shaped(*S.compile_case(eight))
    run_paths(qk, eight, d)


def test_expression_projection_falls_back(qk):
    d = data(20_011, 8)
    run_paths(qk, S.Case("expr_proj", "i64 > 1.7e18", ("rid", "i64 + 0")), d)


def test_negated_range_node(qk):
    """QK_OP_RANGE_COL_IMM with a1 = 1 is `not (lo <= x <= hi)`: accepted by the ABI and both kernels, never emitted by the
    compiler (which writes NOT around the node)."""
    d = data(30_007, 9)
    slot = {c: i for i, c in enumerate(S.COLUMNS)}
    for col, lo, hi in (("i64", 0, 64), ("u8", 31, 77), ("i32", -70, 70), ("d", 0, 0), ("i64", 5, 4), ("j64", -(1 << 53), 1 << 53)):
        x = d[col].astype(np.int64)
        mask = ~((x >= lo) & (x <= hi))
        pred = [(S.L.OP_RANGE_COL_IMM, slot[col], 1, float(hi), lo)]
        for misaligned in (False, True):
            cols = device_columns(d, misaligned)
            for stable in (True, False):
                outs, m = qk.scan_filter_project(cols, pred, [[(S.L.OP_COL, slot["rid"], 0, 0.0, 0)]], stable=stable)
                assert qk.last_variant() == ("filter_interpreter" if misaligned else "compact_tma")
                assert m == int(mask.sum())
                got = outs[0].cpu().numpy()
                assert np.array_equal(got if stable or not misaligned else np.sort(got), d["rid"][mask]), (col, lo, hi, misaligned, stable)


# ------------------------------------------------------------------ the Bloom-reduced compaction
@pytest.mark.parametrize("n,nparts", [(1, 1), (2049, 2), (300_007, 8), (1_000_003, 3)])
def test_bloom(qk, n, nparts):
    d = data(n, 10)
    rng = np.random.default_rng(n)
    keys = rng.choice(d["rid"], size=max(1, n // 5), replace=False) if n else d["rid"]
    bf = qk.Bloom.build(torch.from_numpy(keys).cuda(), qk.Bloom.words_for(max(1, len(keys) // nparts + 1)), nparts, "cuda")
    member = np.isin(d["rid"], keys)
    cases = [c for c in COMPACT if c.pred is not None][:6] + [S.Case("bloom_none", None, ("f64",)), S.Case("bloom_near", "i64 > 1.7e18", ("i32",))]
    for case in cases:
        case = S.Case(case.name, case.pred, tuple(p for p in case.projs if p != "rid")[:7] + ("rid",))
        mask, _ = S.reference(case, d)
        pred, projs = S.compile_case(case)
        cols = device_columns(d)
        outs, m = qk.scan_filter_project(cols, pred, projs, bloom=(bf, len(projs) - 1))
        assert qk.last_variant() == "compact_tma+bloom", case.name
        got = [o.cpu().numpy() for o in outs]
        rid = got[-1]
        assert m == len(rid)
        assert np.all(np.diff(rid) > 0), f"{case.name}: survivors out of input order"
        assert mask[rid].all(), f"{case.name}: a survivor fails the predicate"
        assert np.array_equal(np.intersect1d(rid, np.nonzero(mask & member)[0]), np.nonzero(mask & member)[0]), \
            f"{case.name}: the Bloom filter lost a row whose key is on the build side"
        for p, g in zip(case.projs, got):
            assert S.same(g, d[p][rid].astype(S.out_dtype(p))), f"{case.name}: {p}"


# ------------------------------------------------------------------ the largest call: 2^31 - 1 rows
def test_largest_call_u8(qk):
    """One call of 2^31 - 1 uint8 rows per path (the most nrows the ABI takes), checked against torch on the device."""
    from quokka_b200 import _lib as L, expr as E
    n = (1 << 31) - 1
    gen = torch.Generator(device="cuda").manual_seed(31)
    x = torch.randint(0, 256, (n,), dtype=torch.uint8, device="cuda", generator=gen)
    sch = {"x": E.ColumnInfo(0, L.QK_U8)}
    proj = [E.compile_expr(E.parse("x"), sch)]
    for sql, stable, variant in (("x < 100", True, "compact_tma"), ("x < 100 or x > 250", True, "filter_interpreter"),
                                 ("x < 100 or x > 250", False, "filter_interpreter")):
        mask = (x < 100) | (x > 250) if "or" in sql else x < 100
        want = int(mask.sum())
        outs, m = qk.scan_filter_project([x], E.compile_expr(E.parse(sql), sch), proj, stable=stable)
        assert qk.last_variant() == variant
        assert m == want, (sql, stable)
        if stable:
            assert torch.equal(outs[0], x[mask]), (sql, stable)
        else:
            assert torch.equal(torch.bincount(outs[0], minlength=256), torch.bincount(x[mask], minlength=256)), sql
        del outs, mask
        torch.cuda.empty_cache()
