#!/usr/bin/env python
"""Quantile-sketch benchmark (DataStream.approximate_quantile / qk_qsketch_update, csrc/quantile.cu) on one GPU; one JSON line.

  python tools/bench_quantile.py [--sf 100] [--rows 1000000] [--cols 4096] [--cpu-rows 120000000] [--reps 5]

(a) narrow: SF-`sf` lineitem generated in HBM.  lineitem.approximate_quantile(["l_tax"], 0.9) (apps/tpc-h/tpch.py:606) and the
    four columns of covariance() at [0.1, 0.5, 0.9], through the DataStream API; qk_qsketch_update alone (CUDA events, a
    roofline at 8 B per value read once); torch's exact kthvalue / sort on the same columns.  CPU arm: pyarrow's tdigest
    (delta=100, buffer_size=500, the reference plugin's parameters and code lineage) on the first `cpu-rows` rows, with the
    rank error of each method against the exact target.
(b) wide: `rows` x `cols` seeded normal f32 columns at [0.1, 0.9] (the winsorising workload of the reference's blog): the
    kernel into a fresh sketch (growth included) and into a grown one, the extraction, and torch's kthvalue per column.
The card's name and power limit are read in the same run.  Nothing is written to disk."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np
import torch

from quokka_b200 import ops

COV_COLS = ["l_quantity", "l_extendedprice", "l_discount", "l_tax"]         # apps/tpc-h/tpch.py:600-602
QS = [0.1, 0.5, 0.9]
HBM_PEAK_TBS = 3.35                                                           # H100 SXM data sheet (700 W card)


def card():
    """name and power limit of the card (a read-only query)."""
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except Exception as e:
        return f"unknown ({type(e).__name__})"


def event_ms(fn, reps):
    """CUDA-event time of one call of fn, averaged over reps calls."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def wall(fn, steps):
    """(last result, best seconds) of fn() after one untimed call, each call ending in a device synchronise."""
    fn()
    best, res = float("inf"), None
    for _ in range(max(1, steps)):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = fn()
        torch.cuda.synchronize()
        best = min(best, time.perf_counter() - t0)
    return res, best


def roofline(nbytes, seconds, what):
    return {"bound": "hbm", "frac": nbytes / (HBM_PEAK_TBS * 1e12) / seconds, "gb_per_s": nbytes / seconds / 1e9,
            "algorithmic_bytes": nbytes, "peak_tb_per_s": HBM_PEAK_TBS, "source": "H100 SXM data sheet (700 W), not measured",
            "what": what}


def nearest_rank(n, q):
    x = (n - 1) * q
    f = int(np.floor(x))
    return f + int(x - f >= 0.5)


def rank_error(sorted_x, value, q):
    """|rank of `value` - target rank| / n in the sorted sample (0 when value is the target or ties with it)."""
    n = len(sorted_x)
    r = nearest_rank(n, q)
    lo, hi = int(np.searchsorted(sorted_x, value, "left")), int(np.searchsorted(sorted_x, value, "right")) - 1
    return 0.0 if lo <= r <= hi else min(abs(lo - r), abs(hi - r)) / n


def run_narrow(args, dev):
    from quokka_b200 import synth
    from quokka_b200.columns import DeviceColumn, DeviceTable
    from quokka_b200.df import QuokkaContext
    cols = {c: synth.column(c, args.sf, device=dev) for c in COV_COLS}
    n = cols["l_tax"].numel()
    table = DeviceTable({c: DeviceColumn(v) for c, v in cols.items()})
    res606, t606 = wall(lambda: QuokkaContext().from_device(table).approximate_quantile(["l_tax"], 0.9).collect(), args.steps)
    res4, t4 = wall(lambda: QuokkaContext().from_device(table).approximate_quantile(COV_COLS, QS).collect(), args.steps)
    xs = [cols[c] for c in COV_COLS]
    sk = ops.QuantileSketch(len(xs), dev)
    sk.update(xs)
    kms = event_ms(lambda: sk.update(xs), args.reps)                        # a grown sketch: the steady state of a stream
    kms1 = event_ms(lambda: ops.QuantileSketch(1, dev).update([cols["l_tax"]]), args.reps)     # tpch.py:606, table set-up included
    ex_ms = event_ms(lambda: sk.quantiles(QS), args.reps)
    # torch's exact path: kthvalue per quantile, and one sort per column
    def kth():
        return [[float(torch.kthvalue(x.to(torch.float64), nearest_rank(n, q) + 1).values) for q in QS] for x in xs]
    exact, kth_s = wall(kth, 1)
    _, sort_s = wall(lambda: [torch.sort(x)[0][[nearest_rank(n, q) for q in QS]] for x in xs], 1)
    _, kth606_s = wall(lambda: float(torch.kthvalue(cols["l_tax"], nearest_rank(n, 0.9) + 1).values), 1)
    got = [[res4[c][i].as_py() for c in COV_COLS] for i in range(len(QS))]
    rel = max(abs(got[i][j] - exact[j][i]) / max(abs(exact[j][i]), 1e-300) for i in range(len(QS)) for j in range(len(COV_COLS)))
    out = {"workload": f"SF-{args.sf:g} lineitem, {n} rows, fp64 columns resident in HBM",
           "tpch_606_seconds": t606, "tpch_606_value": res606["l_tax"][0].as_py(), "tpch_606_exact": exact[3][2],
           "four_cols_3q_seconds": t4, "kernel_ms_4cols": kms, "kernel_ms_l_tax_fresh_sketch": kms1, "extract_ms_4cols_3q": ex_ms,
           "roofline": roofline(8 * len(xs) * n, kms / 1e3, "qk_qsketch_update alone over 4 columns: 8 B per value read once"),
           "torch_kthvalue_4cols_3q_seconds": kth_s, "torch_sort_4cols_seconds": sort_s, "torch_kthvalue_l_tax_seconds": kth606_s,
           "max_rel_err_vs_exact": rel, "exact_cols": [c for j, c in enumerate(COV_COLS) if all(got[i][j] == exact[j][i] for i in range(len(QS)))]}
    out["cpu_arm"] = run_cpu_arm(args, cols, dev)
    return out


def run_cpu_arm(args, cols, dev):
    import pyarrow as pa
    import pyarrow.compute as pc
    m = min(args.cpu_rows, cols["l_tax"].numel())
    arm = {"rows": m}
    for c in ("l_tax", "l_extendedprice"):
        x = cols[c][:m].cpu().numpy()
        t0 = time.perf_counter()
        td = pc.tdigest(pa.array(x), q=QS, delta=100, buffer_size=500).to_pylist()
        td_s = time.perf_counter() - t0
        sk = ops.QuantileSketch(1, dev)
        sk.update([cols[c][:m].contiguous()])
        ours = sk.quantiles(QS)[0][:, 0].tolist()
        xs = np.sort(x)
        arm[c] = {"tdigest_seconds": td_s, "tdigest": td, "sketch": ours, "exact": [float(xs[nearest_rank(m, q)]) for q in QS],
                  "tdigest_rank_err": [rank_error(xs, v, q) for v, q in zip(td, QS)],
                  "sketch_rank_err": [rank_error(xs, v, q) for v, q in zip(ours, QS)]}
    return arm


def run_wide(args, dev):
    n, k = args.rows, args.cols
    gen = torch.Generator(device=dev)
    gen.manual_seed(1234)
    X = torch.randn(k, n, generator=gen, device=dev, dtype=torch.float32)
    X += torch.arange(k, device=dev, dtype=torch.float32)[:, None] * 0.01
    xs = list(X.unbind(0))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    sk = ops.QuantileSketch(k, dev)
    sk.update(xs)
    torch.cuda.synchronize()
    fresh_s = time.perf_counter() - t0
    kms = event_ms(lambda: sk.update(xs), args.reps)
    ex_ms = event_ms(lambda: sk.quantiles([0.1, 0.9]), args.reps)
    vals = sk.quantiles([0.1, 0.9])[0]
    ranks = [nearest_rank(n, q) + 1 for q in (0.1, 0.9)]

    def kth():
        outs = []
        for lo in range(0, k, 256):
            outs.append(torch.stack([torch.kthvalue(X[lo:lo + 256], r, dim=1).values for r in ranks]))
        return torch.cat(outs, dim=1)
    exact, kth_s = wall(kth, 1)
    rel = float(((vals.to(torch.float64) - exact.to(torch.float64)).abs() / exact.to(torch.float64).abs().clamp_min(1e-300)).max())
    return {"workload": f"{n} rows x {k} f32 columns (seeded normal) at [0.1, 0.9]", "entries": sk.entries()[0].numel(), "capacity": getattr(sk, "capacity", None),
            "fresh_sketch_seconds": fresh_s, "deferral_rounds": sk.rounds, "grows": sk.grows, "kernel_ms_grown": kms,
            "extract_ms": ex_ms, "roofline": roofline(4 * n * k, kms / 1e3, "qk_qsketch_update into a grown sketch: 4 B per value"),
            "torch_kthvalue_seconds": kth_s, "max_rel_err_vs_exact": rel}


def main(argv=None, dev=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--sf", type=float, default=100, help="scale factor of the narrow leg (SF-100: 600 M rows)")
    ap.add_argument("--rows", type=int, default=1_000_000, help="rows of the wide leg")
    ap.add_argument("--cols", type=int, default=4096, help="f32 columns of the wide leg")
    ap.add_argument("--cpu-rows", type=int, default=120_000_000, help="rows of the CPU t-digest arm")
    ap.add_argument("--reps", type=int, default=5, help="timed kernel calls per measurement")
    ap.add_argument("--steps", type=int, default=3, help="timed DataStream runs of the narrow leg")
    args = ap.parse_args(argv)
    dev = dev or torch.device("cuda", torch.cuda.current_device())
    line = {"card": card(), "narrow": run_narrow(args, dev)}
    torch.cuda.empty_cache()
    line["wide"] = run_wide(args, dev)
    print(json.dumps(line), flush=True)
    return line


if __name__ == "__main__":
    main()
