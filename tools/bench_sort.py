#!/usr/bin/env python
"""Sort benchmark (DataStream.sort / qk_sort_perm, csrc/sort.cu) on one GPU; one JSON line.

  python tools/bench_sort.py [--sf 100] [--rows 600000000] [--api-sf 30] [--asof-quotes 200000000] [--reps 10] [--steps 2]

Kernel legs, qk_sort_perm alone next to torch.sort(stable=True) returning indices, on the same seeded data, outputs compared:
  A  SF-`sf` l_shipdate (int32, ~2 500 distinct values: two live digits)
  B  `rows` random int64 (eight live digits)
  C  SF-`sf` l_extendedprice (fp64)
Program legs through the DataStream API (whole program, results left on the device):
  D  lineitem.sort(["l_shipdate", "l_extendedprice"], [False, True]) over 4 payload columns at SF-`api-sf`
  E  shuffled quotes + trades: sort("time").join_asof(...) next to the same join from the pre-sorted input
Bytes are the algorithm's (csrc/sort.cu): pass 0 reads the key and writes 12 B/row; every live pass reads 8 B/row (4 B/row for
the NULL pass) to count and reads and writes 12 B/row to scatter; the last pass writes 4 B/row (no image wanted).  The HBM
fraction is against the H100 SXM data sheet's 3.35 TB/s.  The card's name, power limit and SM clock are read in the same run;
without a GPU the script fails.  Nothing is written to disk."""
from __future__ import annotations

import argparse
import functools
import json
import os
import re
import sys

TOOLS = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(TOOLS))
sys.path.insert(0, TOOLS)                                                     # benchkit, also when loaded as a module

import torch

import benchkit
from benchkit import HBM_PEAK_TBS, event_ms, wall
from quokka_b200 import ops

card = functools.partial(benchkit.card, clocks=True)                         # with the SM clock now and at most


def model_bytes(n: int, key_bytes: int, passes: int, null_pass: bool = False) -> int:
    """Algorithmic bytes of one qk_sort_perm without image_out: see the module docstring."""
    live = passes + int(null_pass)
    if live == 0:
        return n * (key_bytes + 12 + 12 + 4)                                  # pass 0, then the copy of the row numbers
    return n * (key_bytes + 12) + n * 8 * passes + n * 4 * int(null_pass) + n * 24 * (live - 1) + n * (12 + 4)


def kernel_leg(name: str, key: torch.Tensor, reps: int, clock: list):
    n = key.numel()
    perm = ops.sort_perm(key, None, False)                                    # warm-up of this shape
    plan = ops.sort_last_plan()
    passes = int(re.search(r"passes=(\d+)/8", plan).group(1))
    ms = event_ms(lambda: ops.sort_perm(key, None, False), reps)
    clock.append(card())
    del_ws = torch.cuda.empty_cache
    del_ws()
    idx = torch.sort(key, stable=True).indices                                # warm-up, and the answer to compare with
    same = bool(torch.equal(perm.to(torch.int64), idx))
    del idx, perm
    del_ws()
    tms = event_ms(lambda: torch.sort(key, stable=True), reps)
    nbytes = model_bytes(n, key.element_size(), passes)
    return {"leg": name, "rows": n, "dtype": str(key.dtype).replace("torch.", ""), "plan": plan, "live_passes": passes, "ms": ms,
            "rows_per_s": n / (ms / 1e3), "algorithmic_bytes": nbytes, "gb_per_s": nbytes / (ms / 1e3) / 1e9,
            "hbm_frac_of_3.35TBs_datasheet": nbytes / (HBM_PEAK_TBS * 1e12) / (ms / 1e3), "torch_sort_stable_ms": tms,
            "ms_over_torch": ms / tms, "equals_torch_indices": same, "timed_calls": reps}


def run_api(args, dev):
    from quokka_b200 import synth
    from quokka_b200.columns import DeviceColumn, DeviceTable
    from quokka_b200.df import QuokkaContext
    names = ["l_shipdate", "l_extendedprice", "l_orderkey", "l_quantity", "l_discount", "l_tax"]
    table = DeviceTable({c: DeviceColumn(synth.column(c, args.api_sf, device=dev)) for c in names})
    n = len(table)

    def program():
        qc = QuokkaContext()
        s = qc.from_device(table).sort(["l_shipdate", "l_extendedprice"], [False, True])
        return qc.execute_node(s.node, to_arrow=False)
    res, secs, _ = wall(program, args.steps)
    d, p = res["l_shipdate"].data, res["l_extendedprice"].data
    ok = bool(((d[1:] > d[:-1]) | ((d[1:] == d[:-1]) & (p[1:] <= p[:-1]))).all().item()) if n > 1 else True
    return {"leg": "D", "workload": f"SF-{args.api_sf:g} lineitem.sort([l_shipdate, l_extendedprice desc]), 2 key + 4 payload columns, {n} rows",
            "rows": n, "seconds": secs, "rows_per_s": n / secs, "sorted": ok and len(res) == n}


def run_asof(args, dev):
    from quokka_b200 import synth
    from quokka_b200.columns import DeviceColumn, DeviceTable
    from quokka_b200.df import QuokkaContext
    nq, nt, nsym = args.asof_quotes, args.asof_quotes // 5, 2048
    q = synth.ticks(synth.T_QUOTES, nq, nsym, columns=["time", "symbol", "bid", "ask"], device=dev)
    t = synth.ticks(synth.T_TRADES, nt, nsym, gap=5000, columns=["time", "symbol", "size"], device=dev)
    gen = torch.Generator(device=dev)
    gen.manual_seed(99)

    def tables(cols, shuffle):
        if shuffle:
            order = torch.randperm(cols["time"].numel(), generator=gen, device=dev)
            cols = {c: v[order] for c, v in cols.items()}
        return DeviceTable({c: DeviceColumn(v) for c, v in cols.items()})
    qs, ts, qu, tu = tables(q, False), tables(t, False), tables(q, True), tables(t, True)

    def presorted():
        qc = QuokkaContext()
        s = qc.from_device(ts, sorted_by="time").join_asof(qc.from_device(qs, sorted_by="time"), on="time", by="symbol")
        return qc.execute_node(s.node, to_arrow=False)

    def sorted_here():
        qc = QuokkaContext()
        s = qc.from_device(tu).sort("time").join_asof(qc.from_device(qu).sort("time"), on="time", by="symbol")
        return qc.execute_node(s.node, to_arrow=False)
    a, sa, _ = wall(presorted, args.steps)
    b, sb, _ = wall(sorted_here, args.steps)
    # quotes of one symbol have distinct times here, so both programs match every trade with the same quote
    same = len(a) == len(b) == nt and bool(torch.equal(torch.sort(a["bid"].data.double() + a["time"].data).values,
                                                       torch.sort(b["bid"].data.double() + b["time"].data).values))
    return {"leg": "E", "workload": f"{nq} quotes + {nt} trades, {nsym} symbols, rows shuffled", "presorted_join_seconds": sa,
            "sort_then_join_seconds": sb, "sort_cost_over_join": (sb - sa) / sa, "rows_per_s_sort_then_join": (nq + nt) / sb,
            "same_matches": same}


def main(argv=None, dev=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--sf", type=float, default=100, help="scale factor of legs A and C (SF-100: 600 M rows)")
    ap.add_argument("--rows", type=int, default=600_000_000, help="rows of leg B")
    ap.add_argument("--api-sf", type=float, default=30, help="scale factor of leg D (the table, its sorted copy and the pairs are resident)")
    ap.add_argument("--asof-quotes", type=int, default=200_000_000, help="quotes of leg E (a fifth as many trades)")
    ap.add_argument("--reps", type=int, default=10, help="timed calls per kernel measurement")
    ap.add_argument("--steps", type=int, default=2, help="timed runs of each program leg")
    ap.add_argument("--legs", default="ABCDE")
    args = ap.parse_args(argv)
    if dev is None:
        if not torch.cuda.is_available():
            raise SystemExit("bench_sort: no CUDA device (there is no CPU path to measure)")
        dev = torch.device("cuda", torch.cuda.current_device())
    from quokka_b200 import synth
    line, clock = {"card_name_powerlimit_smclock_maxclock": card(), "legs": []}, []
    for leg in args.legs:
        if leg == "A":
            line["legs"].append(kernel_leg("A l_shipdate", synth.column("l_shipdate", args.sf, device=dev), args.reps, clock))
        elif leg == "B":
            gen = torch.Generator(device=dev)
            gen.manual_seed(4321)
            key = torch.randint(-(1 << 63), (1 << 63) - 1, (args.rows,), generator=gen, device=dev, dtype=torch.int64)
            line["legs"].append(kernel_leg("B random int64", key, args.reps, clock))
            del key
        elif leg == "C":
            line["legs"].append(kernel_leg("C l_extendedprice", synth.column("l_extendedprice", args.sf, device=dev), args.reps, clock))
        elif leg == "D":
            line["legs"].append(run_api(args, dev))
        elif leg == "E":
            line["legs"].append(run_asof(args, dev))
        torch.cuda.empty_cache()
    line["card_after_each_kernel_leg"] = clock
    print(json.dumps(line), flush=True)
    return line


if __name__ == "__main__":
    main()
