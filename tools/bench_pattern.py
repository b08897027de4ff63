#!/usr/bin/env python
"""Pattern-recognition benchmark (OrderedStream.pattern_recognize, qk_pattern_search in csrc/pattern.cu) on one GPU; one JSON line on
stdout.

  python tools/bench_pattern.py [--rows 100000000] [--symbols 8000] [--reps 3] [--sample 1000000] [--tiny]

Quotes are generated on the device (synth.ticks: time, symbol, bid, ask, asize).  Two legs:
  A  the announcement's row-local pattern: asize above its 90th percentile, then below its 10th, then above the 90th again;
  B  four events with link predicates: a large quote, a higher ask, a lower bid below a's and b's, an ask above c's.
Thresholds come from the data's quantiles, so the fraction of rows that start a search is stated, not accidental; maxspan covers
about 16 quotes of one symbol.  Per leg: the qk_pattern_search time (CUDA events over `reps` calls after a warm-up), the whole
DataStream program's time (host clock around collect()), rows/s, rows tested per start, starts and matches, and the bytes of one
pass over the columns the pattern reads -- a lower bound on the traffic of any implementation.  The card's name and power limit
are read in the same run.  The host arm runs the search restated in Python (tests/pattern_shim.py) on the first `sample` rows and
checks that the device answers the same, and runs the brute-force oracle of tests/pattern_cases.py (every tuple of rows, then the
smallest time vector) on the rows of `--oracle-symbols` symbols of that sample, those of median size, against the device.  Nothing is written to
disk."""
from __future__ import annotations

import argparse
import json
import os
import sys
import time as _time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))                               # benchkit, also when loaded as a module

import torch

from benchkit import HBM_PEAK_TBS, card, event_ms
from quokka_b200 import ops, synth



def sync(dev):
    if dev.type == "cuda":
        torch.cuda.synchronize()


def quotes(n, n_symbols, dev):
    q = synth.ticks(synth.T_QUOTES, n, n_symbols, columns={"time", "symbol", "bid", "ask", "asize"}, device=dev)
    return {k: q[k] for k in ("time", "symbol", "bid", "ask", "asize")}


def legs(q, n, n_symbols):
    asize = q["asize"]
    pick = asize[:: max(1, n // 1_000_000)].double()
    hi, lo = (float(torch.quantile(pick, x).item()) for x in (0.9, 0.1))
    t = q["time"]
    span = int((int(t[-1].item()) - int(t[0].item())) * n_symbols // max(1, n)) * 16
    a = [("a", f"asize > {hi!r}"), ("b", f"asize < {lo!r}"), ("c", f"asize > {hi!r}")]
    b = [("a", f"asize > {hi!r}"), ("b", "b.ask > a.ask"), ("c", "bid < a.bid and c.bid < b.bid"), ("d", "d.ask > c.ask")]
    return {"A": a, "B": b}, span, {"asize_q90": hi, "asize_q10": lo, "start_fraction": 0.1}


def run_leg(name, events, span, table, n, reps, dev, sample, oracle_symbols):
    from quokka_b200 import executors as X
    from quokka_b200.columns import DeviceTable
    from quokka_b200.df import QuokkaContext
    ex = X.CEPExecutor(table.column_names, events, "time", span, "symbol")
    a = ex.search_inputs(table, table["time"].data)
    tested = torch.zeros(1, dtype=torch.int64, device=dev)
    bound = ops.pattern_search(**a, rows_tested=tested)              # warm-up; counts the rows tested once
    sync(dev)
    n_tested = int(tested.item())
    starts = int(a["starts"].numel())
    matches = int((bound[:, 0] >= 0).sum().item())
    kernel_ms = event_ms(lambda: ops.pattern_search(**a), reps)
    touched = sorted(ex.touched_columns)
    pass_bytes = sum(table[c].data.element_size() * n for c in touched)
    qc = QuokkaContext()
    stream = qc.from_device(table, sorted_by="time")
    stream.pattern_recognize("time", events, span, "symbol").collect()            # warm-up
    sync(dev)
    t0 = _time.perf_counter()
    for _ in range(reps):
        res = stream.pattern_recognize("time", events, span, "symbol").collect()
    sync(dev)
    program_ms = (_time.perf_counter() - t0) * 1e3 / reps
    out = {"leg": name, "events": events, "maxspan": span, "starts": starts, "matches": matches, "result_rows": res.num_rows,
           "kernel_ms": kernel_ms, "program_ms": program_ms, "rows_per_s_kernel": n / (kernel_ms / 1e3),
           "rows_per_s_program": n / (program_ms / 1e3), "rows_tested": n_tested, "rows_tested_per_start": n_tested / max(1, starts),
           "one_pass_bytes": pass_bytes, "one_pass_ms_at_hbm_peak": pass_bytes / (HBM_PEAK_TBS * 1e12) * 1e3,
           "touched_columns": touched}
    out["host_arm"] = host_arm(events, span, table, sample, dev, oracle_symbols)
    return out


def host_arm(events, span, table, sample, dev, oracle_symbols):
    """The search restated in Python on the first `sample` rows (labelled as a host number) and whether the device agrees; then
    the brute-force oracle of tests/pattern_cases.py on the rows of `oracle_symbols` symbols of typical size among them, against
    the device."""
    import numpy as np
    import pyarrow as pa
    import pyarrow.compute as pc
    import pattern_cases as P
    import pattern_shim
    tab = table.slice(0, sample).to_arrow()
    t0 = _time.perf_counter()
    host = P.search(pattern_shim.pattern_search, tab, "time", events, span, "symbol")
    host_s = _time.perf_counter() - t0
    device = P.search(ops.pattern_search, tab, "time", events, span, "symbol", device=dev)
    # the oracle enumerates every tuple of a span: it takes the symbols whose row counts in the sample are nearest the median
    # (a few hot symbols hold many times the average rows per span)
    counts = np.bincount(tab["symbol"].to_numpy())
    present = np.nonzero(counts)[0]
    med = np.median(counts[present])
    pick = present[np.argsort(np.abs(counts[present] - med), kind="stable")[:oracle_symbols]]
    few = tab.filter(pc.is_in(tab["symbol"], pa.array(pick.astype(np.int32))))
    oracle = P.pattern_recognize(few, "time", events, span, "symbol")
    return {"rows": tab.num_rows, "matches": len(host), "host_python_search_s": host_s,
            "label": "host restatement of the search in Python (tests/pattern_shim.py), not a GPU number",
            "device_equals_host": device == host,
            "oracle_rows": few.num_rows, "oracle_matches": len(oracle),
            "device_equals_oracle": P.search(ops.pattern_search, few, "time", events, span, "symbol", device=dev) == oracle}


def main(argv=None, dev=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--symbols", type=int, default=8000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sample", type=int, default=1_000_000)
    ap.add_argument("--legs", default="A,B")
    ap.add_argument("--oracle-symbols", type=int, default=8, help="symbols of the sample (those of median size) the brute-force oracle checks")
    ap.add_argument("--tiny", action="store_true", help="20 000 rows, 50 symbols, a 5 000-row sample")
    args = ap.parse_args(argv)
    if args.tiny:
        args.rows, args.symbols, args.sample = 20_000, 50, 5_000
    dev = dev or torch.device("cuda")
    from quokka_b200.columns import DeviceColumn, DeviceTable
    q = quotes(args.rows, args.symbols, dev)
    table = DeviceTable({k: DeviceColumn(v) for k, v in q.items()})
    pats, span, thresholds = legs(q, args.rows, args.symbols)
    out = {"bench": "pattern_recognize", "card": card(), "rows": args.rows, "symbols": args.symbols, "reps": args.reps,
           "thresholds": thresholds, "legs": []}
    for name in args.legs.split(","):
        out["legs"].append(run_leg(name, pats[name], span, table, args.rows, args.reps, dev, min(args.sample, args.rows),
                                   args.oracle_symbols))
    print(json.dumps(out))
    return out


if __name__ == "__main__":
    main()
