"""The judged queries restated on the numpy oracle (TEST INFRASTRUCTURE -- see oracle/__init__.py).

Query text: the reference's apps/tpc-h/tpch.py:106-120 (Q1), :168-175 (Q3), :223-236 (Q5),
cross-checked with the canonical SQL in apps/tpc-h/tpch_ref.py:15-38, :89-115, :142-169;
as-of: apps/tpc-h/range.py:10-16.  Inputs are numpy column dicts (oracle/tpch_gen.py); string
columns are dictionary codes and the literals are resolved to codes here, as the product does.
"""
from __future__ import annotations

import numpy as np

from . import relops as R
from . import tpch_gen as G


def q1(li: dict) -> dict:
    """filter l_shipdate <= date '1998-12-01' - interval '90' day; group by returnflag, linestatus;
    8 aggregates (tpch.py:108-117).  Result sorted by the two keys."""
    m = li["l_shipdate"] <= G.DAY_1998_09_02
    ext, disc, tax, qty = (li[c][m] for c in ("l_extendedprice", "l_discount", "l_tax", "l_quantity"))
    disc_price = ext * (1 - disc)
    charge = ext * (1 - disc) * (1 + tax)
    keys = {"l_returnflag": li["l_returnflag"][m], "l_linestatus": li["l_linestatus"][m]}
    return R.group_aggregate(keys, {
        "sum_qty": ("sum", qty), "sum_base_price": ("sum", ext),
        "sum_disc_price": ("sum", disc_price), "sum_charge": ("sum", charge),
        "avg_qty": ("avg", qty), "avg_price": ("avg", ext), "avg_disc": ("avg", disc),
        "count_order": ("count", None)})


def q3_joined(li: dict, od: dict, cu: dict) -> dict:
    """Pushed-down filters + the reference's join chain (lineitem probe; orders then customer builds:
    pyquokka/logical.py:459-506): returns the joined, filtered rows before aggregation."""
    building = G.SEGMENT_DICT.index("BUILDING")
    cm = cu["c_mktsegment"] == building
    om = od["o_orderdate"] < G.DAY_1995_03_15
    lm = li["l_shipdate"] > G.DAY_1995_03_15
    l = {c: li[c][lm] for c in ("l_orderkey", "l_extendedprice", "l_discount")}
    o = {c: od[c][om] for c in ("o_orderkey", "o_custkey", "o_orderdate", "o_shippriority")}
    c = {"c_custkey": cu["c_custkey"][cm]}
    j1 = R.join_tables(l, o, "l_orderkey", "o_orderkey", "inner")
    j2 = R.join_tables(j1, c, "o_custkey", "c_custkey", "inner")
    return j2


def q3(li: dict, od: dict, cu: dict, k: int = 10) -> dict:
    """group by (l_orderkey, o_orderdate, o_shippriority) sum(ext*(1-disc)) as revenue; top 10 by
    revenue desc, o_orderdate asc (tpch.py:171-173)."""
    j = q3_joined(li, od, cu)
    rev = j["l_extendedprice"] * (1 - j["l_discount"])
    g = R.group_aggregate({c: j[c] for c in ("l_orderkey", "o_orderdate", "o_shippriority")},
                          {"revenue": ("sum", rev)})
    return R.top_k(g, ["revenue", "o_orderdate"], k, [True, False]), g


def q5(li: dict, od: dict, cu: dict, su: dict) -> dict:
    """tpch.py:223-236: ASIA nations (eager), customer x nations (broadcast join), then orders,
    lineitem, supplier (shuffled joins), post-join s_nationkey = c_nationkey, 1994 orders,
    sum(revenue) by n_name.  Result keyed by nation key (n_name resolved by the caller)."""
    asia = G.REGIONS.index("ASIA")
    nk = np.array([i for i, r in enumerate(G.NATION_REGION) if r == asia], dtype=np.int64)
    c = {"c_custkey": cu["c_custkey"], "c_nationkey": cu["c_nationkey"]}
    j = R.join_tables(c, {"n_nationkey": nk}, "c_nationkey", "n_nationkey", "semi")
    om = (od["o_orderdate"] >= G.DAY_1994_01_01) & (od["o_orderdate"] < G.DAY_1995_01_01)
    o = {"o_orderkey": od["o_orderkey"][om], "o_custkey": od["o_custkey"][om]}
    j = R.join_tables(j, o, "c_custkey", "o_custkey", "inner")
    l = {c_: li[c_] for c_ in ("l_orderkey", "l_suppkey", "l_extendedprice", "l_discount")}
    j = R.join_tables(j, l, "o_orderkey", "l_orderkey", "inner")
    j = R.join_tables(j, su, "l_suppkey", "s_suppkey", "inner")
    m = j["s_nationkey"] == j["c_nationkey"]
    rev = (j["l_extendedprice"] * (1 - j["l_discount"]))[m]
    return R.group_aggregate({"n_nationkey": j["c_nationkey"][m]}, {"revenue": ("sum", rev)})


def asof_checksum(trades: dict, quotes: dict):
    """trades.join_asof(quotes, on=time, by=symbol) then sum(cast(asize*100 as int))
    (apps/tpc-h/range.py:13-15).  Returns (right index per trade, #matched, checksum)."""
    ridx = R.asof_backward(trades["time"], trades["symbol"], quotes["time"], quotes["symbol"])
    m = ridx >= 0
    # DuckDB CAST(double AS INTEGER) rounds to nearest (half away from zero)
    v = quotes["asize"][ridx[m]].astype(np.float64) * 100.0
    s = int(np.sum(np.where(v >= 0, np.floor(v + 0.5), np.ceil(v - 0.5)).astype(np.int64)))
    return ridx, int(m.sum()), s


# ---------------------------------------------------------------- multi-threaded Arrow (Acero) arm
def q1_acero(tbl):
    """Same Q1 on pyarrow compute + Acero hash aggregate (multi-threaded) -- the CPU arm that
    bench.py times (`cpu_baseline`, `--impl reference`): Arrow C++ is the engine the reference scans
    with (pyquokka/dataset/unordered_readers.py:98-99) and the same family as its Polars/DuckDB
    executors, which are not installable here."""
    import pyarrow as pa
    import pyarrow.compute as pc
    t = tbl.filter(pc.less_equal(tbl["l_shipdate"], pa.scalar(G.DAY_1998_09_02, pa.int32()).cast(tbl.schema.field("l_shipdate").type)))
    one = pa.scalar(1.0)
    dp = pc.multiply(t["l_extendedprice"], pc.subtract(one, t["l_discount"]))
    ch = pc.multiply(dp, pc.add(one, t["l_tax"]))
    t = t.append_column("disc_price", dp).append_column("charge", ch)
    g = t.group_by(["l_returnflag", "l_linestatus"], use_threads=False).aggregate([
        ("l_quantity", "sum"), ("l_extendedprice", "sum"), ("disc_price", "sum"), ("charge", "sum"),
        ("l_discount", "sum"), ([], "count_all")])
    return g


def q1_acero_batched(tbl, batch_rows: int = 2_000_000, threads: int | None = None):
    """Q1 the way the reference executes it on CPU: the scan is cut into batches, every batch gets the
    filter + projection + PARTIAL aggregate on its own worker (`partition_fn` with the folded DuckDB partial
    aggregate, pyquokka/core.py:152-195 / datastream.py:795-801; one worker per channel), the partials are
    concatenated and aggregated once more (SQLAggExecutor.done, sql_executors.py:592-599).  Arrow compute
    kernels are single-threaded per array, so batch-level parallelism is what uses all host cores."""
    import os
    from concurrent.futures import ThreadPoolExecutor
    import pyarrow as pa
    threads = threads or os.cpu_count() or 1
    n = tbl.num_rows
    parts = [tbl.slice(lo, min(batch_rows, n - lo)) for lo in range(0, n, batch_rows)]
    with ThreadPoolExecutor(max_workers=threads) as ex:
        partials = list(ex.map(q1_acero, parts))
    allp = pa.concat_tables(partials)
    return allp.group_by(["l_returnflag", "l_linestatus"]).aggregate([
        ("l_quantity_sum", "sum"), ("l_extendedprice_sum", "sum"), ("disc_price_sum", "sum"), ("charge_sum", "sum"),
        ("l_discount_sum", "sum"), ("count_all", "sum")])
