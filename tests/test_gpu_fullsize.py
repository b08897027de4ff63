"""Parity at sizes the numpy oracle cannot reach in seconds, through size-independent properties and an
independent fp64 computation on the device with torch ops (torch here is the CHECKER, the kernels under
test are libqk's).  SF-10-shaped inputs (60 M lineitem rows); the SF-100 run itself is checked the same
way inside bench.py (sum of group counts = rows passing the filter)."""
import numpy as np
import pytest
import torch

from oracle import queries as OQ
from oracle import tpch_gen as G

pytestmark = pytest.mark.gpu
RTOL = 1e-9


@pytest.fixture(scope="module")
def qb():
    from quokka_b200 import _lib, expr, ops, synth
    _lib.lib()
    return type("QB", (), dict(L=_lib, E=expr, ops=ops, synth=synth))


def test_q1_sf10_typed_dyn_and_interpreter_against_independent_fp64(qb):
    sf, names = 10, ["l_shipdate", "l_returnflag", "l_linestatus", "l_quantity", "l_extendedprice", "l_discount", "l_tax"]
    cols = {c: qb.synth.column(c, sf) for c in names}
    n = cols["l_shipdate"].numel()
    assert n == 60_000_000
    sch = {c: qb.E.ColumnInfo(i, qb.ops.qk_dtype(t)) for i, (c, t) in enumerate(cols.items())}
    pred = qb.E.compile_expr(qb.E.parse("l_shipdate <= date '1998-12-01' - interval '90' day"), sch)
    aggs = [qb.E.compile_expr(qb.E.parse(a), sch) for a in
            ("l_quantity", "l_extendedprice", "l_extendedprice * (1 - l_discount)",
             "l_extendedprice * (1 - l_discount) * (1 + l_tax)", "l_discount")]
    for variant in (0, 7, 1):
        st = qb.ops.DenseAggState([3, 2], [qb.L.AGG_SUM] * 5, "cuda")
        st.update(list(cols.values()), pred, [1, 2], aggs, variant=variant)
        m = cols["l_shipdate"] <= G.DAY_1998_09_02
        g = (cols["l_returnflag"].long() * 2 + cols["l_linestatus"].long())[m]
        cnt = torch.bincount(g, minlength=6)
        assert torch.equal(st.cnt, cnt)                                   # bit-exact counts, 59 M rows
        assert int(st.cnt.sum()) == int(m.sum())
        ext, disc, tax, qty = (cols[c][m] for c in ("l_extendedprice", "l_discount", "l_tax", "l_quantity"))
        ref = [qty, ext, ext * (1 - disc), ext * (1 - disc) * (1 + tax), disc]
        for j, v in enumerate(ref):
            exp = torch.bincount(g, weights=v, minlength=6)
            assert torch.allclose(st.acc[:, j], exp, rtol=RTOL, atol=0), (variant, j)
    # linearity: Q1(whole) = Q1(first half) + Q1(second half), to the last bit of the integer part
    half = n // 2 // 1024 * 1024
    a = qb.ops.DenseAggState([3, 2], [qb.L.AGG_SUM] * 5, "cuda")
    a.update([t[:half] for t in cols.values()], pred, [1, 2], aggs)
    a.update([t[half:] for t in cols.values()], pred, [1, 2], aggs)
    assert torch.equal(a.cnt, st.cnt) and torch.allclose(a.acc, st.acc, rtol=1e-12)


def test_q3_sf1_datastream_vs_oracle():
    import pyarrow as pa
    from quokka_b200 import synth
    from quokka_b200.columns import DeviceColumn, DeviceTable
    from quokka_b200.df import QuokkaContext
    sf = 1

    def tab(names):
        return DeviceTable({n: DeviceColumn(synth.column(n, sf), synth.DICTIONARIES.get(n),
                                            pa.date32() if n in synth.DATE_COLUMNS else None) for n in names})
    li = tab(["l_orderkey", "l_shipdate", "l_extendedprice", "l_discount"])
    od = tab(["o_orderkey", "o_custkey", "o_orderdate", "o_shippriority"])
    cu = tab(["c_custkey", "c_mktsegment"])
    qc = QuokkaContext()
    d = qc.from_device(li).join(qc.from_device(od), left_on="l_orderkey", right_on="o_orderkey")
    d = qc.from_device(cu).join(d, left_on="c_custkey", right_on="o_custkey")
    d = d.filter_sql("c_mktsegment = 'BUILDING' and o_orderdate < date '1995-03-15' and l_shipdate > date '1995-03-15'")
    g = d.groupby(["l_orderkey", "o_orderdate", "o_shippriority"]).agg_sql("sum(l_extendedprice * (1 - l_discount)) as revenue")
    full = g.collect()
    top = g.top_k(["revenue", "o_orderdate"], 10, descending=[True, False]).collect()
    etop, eg = OQ.q3(G.gen_lineitem(sf, columns=["l_orderkey", "l_shipdate", "l_extendedprice", "l_discount"]),
                     G.gen_orders(sf), G.gen_customer(sf))
    assert full.num_rows == len(eg["l_orderkey"]) > 10_000
    order = np.argsort(full["l_orderkey"].to_numpy(), kind="stable")
    assert np.array_equal(full["l_orderkey"].to_numpy()[order], eg["l_orderkey"])
    np.testing.assert_allclose(full["revenue"].to_numpy()[order], eg["revenue"], rtol=RTOL)
    assert np.array_equal(top["l_orderkey"].to_numpy(), etop["l_orderkey"])


def test_join_partition_asof_properties_at_scale(qb):
    n = 50_000_000
    # --- join: unique build keys probed by themselves in another order -> exactly one match each
    keys = qb.synth.column("o_orderkey", 100, 0, n)                        # sparse, unique
    perm = torch.randperm(n, device="cuda")
    t = qb.ops.JoinTable(n, "cuda")
    t.build(keys)
    pi, bi = t.probe(keys[perm].contiguous(), qb.L.JOIN_INNER)
    assert pi.numel() == n and t.check_flags() == 0
    assert torch.equal(bi.long()[torch.argsort(pi)], perm)                  # probe row i found build row perm[i]
    assert t.probe((keys[:1_000_000] + 9).contiguous(), qb.L.JOIN_SEMI)[0].numel() == 0   # keys+9 are never order keys
    del t, pi, bi, perm
    # --- partition: placement = key % n, stable, a permutation
    for nparts in (8, 5):
        dest, offs = qb.ops.partition_plan(keys, nparts)
        out, src = qb.ops.scatter([keys, torch.arange(n, device="cuda", dtype=torch.int64)], dest)
        offs = offs.cpu().tolist()
        assert offs[0] == 0 and offs[-1] == n
        for p in range(nparts):
            seg, idx = out[offs[p]:offs[p + 1]], src[offs[p]:offs[p + 1]]
            assert bool((seg % nparts == p).all())
            assert bool((idx[1:] > idx[:-1]).all())                       # stable: original order inside a partition
        del dest, out, src
    # --- as-of: the match is the newest quote of the symbol not after the trade
    nq, nt, nsym = 40_000_000, 8_000_000, 8000
    q = qb.synth.ticks(qb.synth.T_QUOTES, nq, nsym, gap=1000, columns=["time", "symbol"])
    tr = qb.synth.ticks(qb.synth.T_TRADES, nt, nsym, gap=5000, columns=["time", "symbol"])
    r = qb.ops.asof_backward(tr["time"], tr["symbol"], q["time"], q["symbol"], nsym)
    ok = r >= 0
    ri = r[ok].long()
    assert bool((q["symbol"][ri] == tr["symbol"][ok]).all())
    assert bool((q["time"][ri] <= tr["time"][ok]).all())
    # no newer quote of the same symbol at or before the trade: check against a sort-based successor table
    order = torch.argsort(q["symbol"].long() * (1 << 42) + q["time"])       # (symbol, time) order; times < 2^42
    rank_of = torch.empty_like(order)
    rank_of[order] = torch.arange(nq, device="cuda")
    nxt = rank_of[ri] + 1
    has_next = nxt < nq
    nrow = order[nxt.clamp(max=nq - 1)]
    same = has_next & (q["symbol"][nrow] == tr["symbol"][ok])
    assert bool((q["time"][nrow][same] > tr["time"][ok][same]).all())
    # unmatched trades really have no earlier quote of their symbol
    first_time = torch.full((nsym,), 1 << 62, dtype=torch.int64, device="cuda")
    first_time.scatter_reduce_(0, q["symbol"].long(), q["time"], reduce="amin")
    assert bool((tr["time"][~ok] < first_time[tr["symbol"][~ok].long()]).all())
