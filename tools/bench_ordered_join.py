#!/usr/bin/env python
"""Order-preserving join benchmark (DataStream.join(maintain_sort_order="left") / qk_join_probe_ordered, csrc/join.cu) on one
GPU; one JSON line.

  python tools/bench_ordered_join.py [--rows 200000000] [--symbols 8000] [--sf 10] [--reps 10] [--steps 2]

Input: device-generated quotes (synth.ticks: time-sorted, `symbols` symbols interleaved) and a symbol table with one row per
symbol (sector, lot size).
  K  qk_join_probe_ordered against qk_join_probe on the same keys and table, kernels alone: the cost of the order
  D  from_device(quotes, sorted_by="time").join(symbols, on="symbol", maintain_sort_order="left"), the whole program, against
     today's way to the same ordered rows, join(...) followed by sort("time")
  L  a large build side: TPC-H lineitem (SF `sf`) sorted by l_shipdate joined to orders on the order key, ordered against
     join + sort("l_shipdate")
Each leg's two results are compared: ties in the sort column may come in another order after the sort, so the sort column is
compared row for row and every other column by its sum (fp64 sums to 1e-9 relative).
Bytes are the algorithm's (csrc/join.cu): the unordered probe reads the key and one 32-byte sector of the table per probe row
and writes 8 B per pair; the ordered probe reads key and sector twice (count and write pass), writes and reads a 4-byte count
and an 8-byte offset per row, and writes 8 B per pair.  The HBM fraction is against the H100 SXM data sheet's 3.35 TB/s.  The
card's name, power limit and SM clock are read in the same run; without a GPU the script fails.  Nothing is written to disk."""
from __future__ import annotations

import argparse
import functools
import json
import math
import os
import sys

TOOLS = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(TOOLS))
sys.path.insert(0, TOOLS)                                                     # benchkit, also when loaded as a module

import torch

import benchkit
from benchkit import HBM_PEAK_TBS, event_ms, wall
from quokka_b200 import _lib as L
from quokka_b200 import ops

card = functools.partial(benchkit.card, clocks=True)                         # with the SM clock now and at most


def model_bytes(n: int, key_bytes: int, pairs: int, ordered: bool) -> int:
    """Algorithmic bytes of one probe of n keys giving `pairs` pairs: see the module docstring."""
    per_row = 2 * (key_bytes + 32) + 2 * 4 + 2 * 8 if ordered else key_bytes + 32
    return n * per_row + pairs * 8


def leg(name, n, nbytes, ms, extra=None):
    out = {"leg": name, "rows": n, "ms": ms, "rows_per_s": n / (ms / 1e3), "algorithmic_bytes": nbytes,
           "gb_per_s": nbytes / (ms / 1e3) / 1e9, "hbm_frac_of_3.35TBs_datasheet": nbytes / (HBM_PEAK_TBS * 1e12) / (ms / 1e3)}
    return out | (extra or {})


def _same_rows(a, b, order_col) -> bool:
    """The same rows in the same `order_col` order: equal times may come in another order after sort(), so the other
    columns are compared by their sums."""
    return (a.column_names == b.column_names and len(a) == len(b) and bool(torch.equal(a[order_col].data, b[order_col].data))
            and all(math.isclose(a[c].data.double().sum().item(), b[c].data.double().sum().item(), rel_tol=1e-9) for c in a.column_names))


def _program(table, dim, left_on, right_on, sorted_by, ordered):
    from quokka_b200.df import QuokkaContext
    qc = QuokkaContext()
    if ordered:
        s = qc.from_device(table, sorted_by=sorted_by).join(qc.from_device(dim), left_on=left_on, right_on=right_on,
                                                             maintain_sort_order="left")
    else:
        s = qc.from_device(table).join(qc.from_device(dim), left_on=left_on, right_on=right_on).sort(sorted_by)
    return qc.execute_node(s.node, to_arrow=False)


def main(argv=None, dev=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--rows", type=int, default=200_000_000, help="quotes")
    ap.add_argument("--symbols", type=int, default=8000)
    ap.add_argument("--sf", type=float, default=10, help="TPC-H scale factor of leg L")
    ap.add_argument("--reps", type=int, default=10, help="timed calls per kernel measurement")
    ap.add_argument("--steps", type=int, default=2, help="timed runs of each program leg")
    ap.add_argument("--legs", default="KDL")
    args = ap.parse_args(argv)
    if dev is None:
        if not torch.cuda.is_available():
            raise SystemExit("bench_ordered_join: no CUDA device (there is no CPU path to measure)")
        dev = torch.device("cuda", torch.cuda.current_device())
    from quokka_b200 import synth
    from quokka_b200.columns import DeviceColumn, DeviceTable
    n, nsym = args.rows, args.symbols
    line, clock = {"card_name_powerlimit_smclock_maxclock": card(),
                   "workload": f"{n} quotes, {nsym} symbols, joined to one row per symbol; lineitem x orders at SF-{args.sf:g}",
                   "legs": []}, []
    q = synth.ticks(synth.T_QUOTES, n, nsym, columns=["time", "symbol", "asize"], device=dev)
    sym = torch.arange(nsym, dtype=q["symbol"].dtype, device=dev)
    dim = DeviceTable({"symbol": DeviceColumn(sym), "lot": DeviceColumn((sym % 5 + 1) * 100),
                       "sector": DeviceColumn((sym % 11).to(torch.int32))})
    for name in args.legs:
        if name == "K":
            t = ops.JoinTable(nsym, dev)
            t.build(sym)
            key = q["symbol"].contiguous()
            pairs = len(t.probe(key)[0])
            ms_u = event_ms(lambda: t.probe(key, expect=n), args.reps)
            ms_o = event_ms(lambda: t.probe_ordered(key, expect=n), args.reps)
            kb = key.element_size()
            line["legs"].append(leg("K qk_join_probe (unordered)", n, model_bytes(n, kb, pairs, False), ms_u, {"pairs": pairs}))
            line["legs"].append(leg("K qk_join_probe_ordered", n, model_bytes(n, kb, pairs, True), ms_o,
                                    {"pairs": pairs, "ms_over_unordered": ms_o / ms_u}))
            clock.append(card())
            del t
        elif name == "D":
            table = DeviceTable({c: DeviceColumn(v) for c, v in q.items()})
            res_o, s_o, _ = wall(lambda: _program(table, dim, "symbol", "symbol", "time", True), args.steps)
            res_s, s_s, _ = wall(lambda: _program(table, dim, "symbol", "symbol", "time", False), args.steps)
            line["legs"].append({"leg": "D join(maintain_sort_order='left')", "rows": n, "seconds": s_o, "rows_per_s": n / s_o})
            line["legs"].append({"leg": "D join + sort('time')", "rows": n, "seconds": s_s, "rows_per_s": n / s_s,
                                 "ordered_over_join_sort": s_o / s_s, "same_rows": _same_rows(res_o, res_s, "time")})
            del table, res_o, res_s
        elif name == "L":
            del q
            li = synth.table(["l_orderkey", "l_shipdate", "l_extendedprice"], args.sf, device=dev)
            perm = ops.sort_perm(li["l_shipdate"].contiguous(), None, False)
            li = DeviceTable({c: DeviceColumn(v[perm.long()]) for c, v in li.items()})
            od = DeviceTable({c: DeviceColumn(v) for c, v in synth.table(["o_orderkey", "o_orderdate", "o_custkey"], args.sf, device=dev).items()})
            nl = len(li)
            res_o, s_o, _ = wall(lambda: _program(li, od, "l_orderkey", "o_orderkey", "l_shipdate", True), args.steps)
            res_s, s_s, _ = wall(lambda: _program(li, od, "l_orderkey", "o_orderkey", "l_shipdate", False), args.steps)
            same = _same_rows(res_o, res_s, "l_shipdate")
            line["legs"].append({"leg": "L lineitem by l_shipdate x orders, ordered", "rows": nl, "build_rows": len(od),
                                 "seconds": s_o, "rows_per_s": nl / s_o})
            line["legs"].append({"leg": "L lineitem x orders, join + sort('l_shipdate')", "rows": nl, "seconds": s_s,
                                 "rows_per_s": nl / s_s, "ordered_over_join_sort": s_o / s_s, "same_rows": same})
        torch.cuda.empty_cache()
    line["card_after_each_kernel_leg"] = clock
    print(json.dumps(line), flush=True)
    return line


if __name__ == "__main__":
    main()
