#!/usr/bin/env python
"""Gram-matrix benchmark (DataStream.gramian / qk_gram, csrc/gram.cu) on one GPU; one JSON line on stdout.

  python tools/bench_gram.py [--sf 100] [--rows 1000000] [--cols 4096] [--reps 4]

(a) narrow: lineitem.gramian([l_quantity, l_extendedprice, l_discount, l_tax]) of apps/tpc-h/tpch.py:600-602 on SF-`sf`
    lineitem generated in HBM (SF-100: 600 M rows x 4 fp64 = 19.2 GB), through the DataStream API and as the kernel alone;
(b) wide: an n x k table of seeded f32 columns (the feature-engineering shape of the reference's blog, scaled to one GPU), the
    kernel alone (both MMA shapes) next to torch's fp64 X^T @ X on a pre-stacked matrix -- cuBLAS, for comparison only.
Each roofline is the larger of bytes / HBM peak and flops / FP64 tensor-core peak, both H100 SXM data-sheet figures.  The
card's name and power limit are read in the same run.  Nothing is written to disk."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch

from quokka_b200 import ops

GRAM_COLS = ["l_quantity", "l_extendedprice", "l_discount", "l_tax"]
HBM_PEAK_TBS, FP64_TC_PEAK_TFLOPS = 3.35, 67.0   # H100 SXM data sheet (700 W card): HBM3 bandwidth; FP64 tensor core, dense


def roofline(nbytes, flops, seconds, what):
    t_hbm, t_fp = nbytes / (HBM_PEAK_TBS * 1e12), flops / (FP64_TC_PEAK_TFLOPS * 1e12)
    return {"bound": "hbm" if t_hbm >= t_fp else "fp64_tensor_core", "frac": max(t_hbm, t_fp) / seconds,
            "gb_per_s": nbytes / seconds / 1e9, "tflops": flops / seconds / 1e12, "algorithmic_bytes": nbytes, "algorithmic_flops": flops,
            "peaks": {"hbm_tb_per_s": HBM_PEAK_TBS, "fp64_tensor_core_tflops": FP64_TC_PEAK_TFLOPS,
                      "source": "H100 SXM data sheet (700 W), not measured"}, "what": what}


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
    """(last result, best seconds, all seconds) of fn() after one untimed call, each call ending in a device synchronise."""
    fn()
    times = []
    for _ in range(max(1, steps)):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = fn()
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    return res, min(times), times


def bound_ratio(G, cols):
    """max over i <= j of |G - torch fp64 dot| / (n 2^-53 |x_i| . |x_j|): <= 1 is within the summation bound (torch's own dot
    products carry an error of the same order, so up to 2 is what two correct results can differ by)."""
    worst, n = 0.0, cols[0].numel()
    for i in range(len(cols)):
        xi = cols[i].to(torch.float64)
        for j in range(i, len(cols)):
            xj = xi if j == i else cols[j].to(torch.float64)
            ref = float(torch.dot(xi, xj))
            bound = n * 2.0 ** -53 * float(torch.dot(xi.abs(), xj.abs()))
            worst = max(worst, abs(float(G[i, j]) - ref) / max(bound, 1e-300))
    return worst


def run_narrow(args, dev):
    from quokka_b200 import synth
    from quokka_b200.columns import DeviceColumn, DeviceTable
    from quokka_b200.df import QuokkaContext
    cols = {c: synth.column(c, args.sf, device=dev) for c in GRAM_COLS}
    n, k = cols[GRAM_COLS[0]].numel(), len(GRAM_COLS)
    table = DeviceTable({c: DeviceColumn(v) for c, v in cols.items()})
    res, dt, times = wall(lambda: QuokkaContext().from_device(table).gramian(GRAM_COLS).collect(), args.steps)
    xs = [cols[c] for c in GRAM_COLS]
    st = ops.GramState(k, dev)
    kms = event_ms(lambda: st.update(xs), args.reps)
    G = torch.tensor([[res[c][i].as_py() for c in GRAM_COLS] for i in range(k)], dtype=torch.float64)
    nbytes, flops = 8 * k * n, n * k * (k + 1)
    return {"workload": f"lineitem.gramian({GRAM_COLS}) at SF-{args.sf:g}: {n} rows x {k} fp64 columns resident in HBM",
            "api_seconds": dt, "api_all_seconds": times, "kernel_ms": kms, "plan": ops.gram_last_plan(),
            "roofline": roofline(nbytes, flops, kms / 1e3, "qk_gram alone: every row read once (8 B per value), n k (k + 1) flops"),
            "api_roofline": roofline(nbytes, flops, dt, "the whole DataStream program's wall time"),
            "vs_torch_fp64_bound_ratio": bound_ratio(G, xs)}


def run_wide(args, dev):
    n, k = args.rows, args.cols
    gen = torch.Generator(device=dev)
    gen.manual_seed(1234)
    X = torch.randn(k, n, generator=gen, device=dev, dtype=torch.float32)
    X += torch.arange(k, device=dev, dtype=torch.float32)[:, None] * 0.01           # column means away from zero
    xs = list(X.unbind(0))
    plans = {}
    for variant in (1, 2):                                                           # m8n8k4, m16n8k16
        st = ops.GramState(k, dev)
        st.update(xs, variant=variant)
        plans[variant] = (ops.gram_last_plan(), event_ms(lambda: st.update(xs, variant=variant), args.reps))
    best = min(plans, key=lambda v: plans[v][1])
    st = ops.GramState(k, dev)
    st.update(xs)                                                                    # variant 0: what the library picks
    G = st.gram
    flops = n * k * (k + 1)
    out = {"workload": f"{n} rows x {k} f32 columns (seeded normal), one qk_gram call", "plan": ops.gram_last_plan(),
           "kernel_ms": plans[best][1], "variants_ms": {plans[v][0]: plans[v][1] for v in plans},
           "roofline": roofline(4 * k * n, flops, plans[best][1] / 1e3, "qk_gram alone: n k (k + 1) flops (upper triangle), 4 B per value read once")}
    Xd = torch.empty(n, k, dtype=torch.float64, device=dev)
    Xd.copy_(X.T)
    del X, xs
    torch.matmul(Xd.T, Xd)
    tms = event_ms(lambda: torch.matmul(Xd.T, Xd), max(1, args.reps // 2))
    ref = torch.matmul(Xd.T, Xd)
    Xd.abs_()
    bound = n * 2.0 ** -53 * torch.matmul(Xd.T, Xd)
    out.update(torch_fp64_xtx_ms=tms, torch_fp64_xtx_tflops_2nk2=2 * n * k * k / (tms / 1e3) / 1e12,
               vs_torch_fp64_bound_ratio=float(((G - ref).abs() / bound.clamp_min(1e-300)).max()))
    return out


def main(argv=None, dev=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--sf", type=float, default=100, help="scale factor of the narrow leg (SF-100: 600 M rows x 4 fp64)")
    ap.add_argument("--rows", type=int, default=1_000_000, help="rows of the wide leg")
    ap.add_argument("--cols", type=int, default=4096, help="f32 columns of the wide leg")
    ap.add_argument("--reps", type=int, default=4, help="timed qk_gram calls per measurement")
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
