#!/usr/bin/env python
"""Shift benchmark (OrderedStream.shift / qk_shift_plan + qk_shift_gather, csrc/shift.cu) on one GPU; one JSON line.

  python tools/bench_shift.py [--rows 200000000] [--symbols 8000] [--reps 10] [--steps 2]

Input: device-generated quotes (synth.ticks: time-sorted, `symbols` symbols interleaved), a lag of 1 per symbol of `asize`.
  K  qk_shift_plan (by symbol, on a precomputed code partition) + qk_shift_gather of asize, kernels alone
  N  the same without a key (by=None): one plan launch, no partition
  T  the torch formulation of K: torch.sort(codes, stable=True), index arithmetic, a gather with torch.where; its source rows
     are compared with the kernel's
  D  from_device(quotes, sorted_by="time").shift(1, by="symbol", columns=["asize"], suffix="_prev"), the whole program
  E  the same program with by=None
Bytes are the algorithm's (csrc/shift.cu): by key, the inverse permutation reads dest and writes inv (8 B/row), the plan reads
dest, the code and inv and writes src (16 B/row), the gather reads src and moves the value (4 + 2 x value bytes); without a key
the plan writes src only (4 B/row).  The HBM fraction is against the H100 SXM data sheet's 3.35 TB/s.  The card's name, power
limit and SM clock are read in the same run; without a GPU the script fails.  Nothing is written to disk."""
from __future__ import annotations

import argparse
import functools
import json
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


def model_bytes(n: int, value_bytes: int, keyed: bool) -> int:
    """Algorithmic bytes of one plan + gather: see the module docstring."""
    return n * ((8 + 16) if keyed else 4) + n * (4 + 2 * value_bytes)


def torch_src(codes: torch.Tensor, shift: int) -> torch.Tensor:
    """The lag-by-`shift` source rows per key in torch: a stable sort by key, neighbours in sorted order, scattered back."""
    perm = torch.sort(codes, stable=True).indices
    sc = codes[perm]
    n = codes.numel()
    j = torch.arange(n, device=codes.device) - shift
    ok = (j >= 0) & (j < n)
    jc = j.clamp(0, n - 1)
    ok &= sc[jc] == sc
    src = torch.empty(n, dtype=torch.int64, device=codes.device)
    src[perm] = torch.where(ok, perm[jc], torch.full_like(perm, -1))
    return src


def leg(name, n, nbytes, ms, extra=None):
    out = {"leg": name, "rows": n, "ms": ms, "rows_per_s": n / (ms / 1e3), "algorithmic_bytes": nbytes,
           "gb_per_s": nbytes / (ms / 1e3) / 1e9, "hbm_frac_of_3.35TBs_datasheet": nbytes / (HBM_PEAK_TBS * 1e12) / (ms / 1e3)}
    return out | (extra or {})


def main(argv=None, dev=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--rows", type=int, default=200_000_000, help="quotes")
    ap.add_argument("--symbols", type=int, default=8000)
    ap.add_argument("--reps", type=int, default=10, help="timed calls per kernel measurement")
    ap.add_argument("--steps", type=int, default=2, help="timed runs of each program leg")
    ap.add_argument("--legs", default="KNTDE")
    args = ap.parse_args(argv)
    if dev is None:
        if not torch.cuda.is_available():
            raise SystemExit("bench_shift: no CUDA device (there is no CPU path to measure)")
        dev = torch.device("cuda", torch.cuda.current_device())
    from quokka_b200 import synth
    from quokka_b200.columns import DeviceColumn, DeviceTable
    from quokka_b200.df import QuokkaContext
    q = synth.ticks(synth.T_QUOTES, args.rows, args.symbols, columns=["time", "symbol", "asize"], device=dev)
    n, codes, asize = args.rows, q["symbol"].to(torch.int32).contiguous(), q["asize"]
    vb = asize.element_size()
    line, clock = {"card_name_powerlimit_smclock_maxclock": card(), "workload": f"{n} quotes, {args.symbols} symbols, lag 1 of asize",
                   "legs": []}, []
    dest, seg = ops.partition_plan(codes, args.symbols, L.PART_CODE)
    kernel_src = None
    for name in args.legs:
        if name == "K":
            def run():
                src, _, _ = ops.shift_plan(1, n, codes, args.symbols, dest, seg)
                return src, ops.shift_gather([asize], None, src, [None])
            kernel_src = run()[0]
            line["legs"].append(leg("K plan + gather by symbol", n, model_bytes(n, vb, True), event_ms(run, args.reps)))
            clock.append(card())
        elif name == "N":
            def run():
                src, _, _ = ops.shift_plan(1, n, device=dev)
                return ops.shift_gather([asize], None, src, [None])
            line["legs"].append(leg("N plan + gather, no key", n, model_bytes(n, vb, False), event_ms(run, args.reps)))
            clock.append(card())
        elif name == "T":
            def run():
                s = torch_src(codes, 1)
                return torch.where(s >= 0, asize[s.clamp(min=0)], torch.zeros_like(asize))
            ms = event_ms(run, args.reps)
            if kernel_src is None:
                kernel_src = ops.shift_plan(1, n, codes, args.symbols, dest, seg)[0]
            same = bool(torch.equal(torch_src(codes, 1), kernel_src.to(torch.int64)))
            line["legs"].append({"leg": "T torch.sort(stable) + index arithmetic + gather", "rows": n, "ms": ms, "src_equal": same})
            clock.append(card())
        elif name in "DE":
            table = DeviceTable({c: DeviceColumn(v) for c, v in q.items()})

            def program():
                qc = QuokkaContext()
                s = qc.from_device(table, sorted_by="time").shift(1, by="symbol" if name == "D" else None, columns=["asize"], suffix="_prev")
                return qc.execute_node(s.node, to_arrow=False)
            res, secs, _ = wall(program, args.steps)
            v = res["asize_prev"].valid
            line["legs"].append({"leg": name + (" DataStream shift by symbol" if name == "D" else " DataStream shift, no key"), "rows": n,
                                 "seconds": secs, "rows_per_s": n / secs, "null_rows": int((v == 0).sum().item()) if v is not None else 0})
        torch.cuda.empty_cache()
    line["card_after_each_kernel_leg"] = clock
    print(json.dumps(line), flush=True)
    return line


if __name__ == "__main__":
    main()
