#!/usr/bin/env python
"""Per-event window benchmark (windowed_transform(TumblingWindow | SessionWindow, OnEventTrigger()) / qk_window_running,
csrc/window.cu) on one GPU; one JSON line.

  python tools/bench_window_events.py [--rows 200000000] [--symbols 8000] [--reps 10] [--steps 2]

Input: device-generated quotes (synth.ticks: time-sorted, `symbols` symbols interleaved).  The window lengths follow the data:
with g = the mean time between two quotes of one symbol, tumbling windows are 64 g long (about 64 rows per window and key) and
a session closes after a gap > 2 g.  Legs, each for the tumbling and the session window:
  K  qk_window_running alone on a precomputed key partition: 4 outputs (AVG, MAX, SUM, COUNT) over 2 fp64 value columns
  T  the torch formulation of SUM / COUNT: a cumsum minus the prefix before the run start, read at the peer end (the last row
     with the row's time); its COUNT is compared with the kernel's
  D  from_device(quotes, sorted_by="time").windowed_transform(<window>, OnEventTrigger()), the whole program
  C  the same program with OnCompletionTrigger (one row per window), for scale, on the first --completion-rows quotes: its
     hash aggregate does not fit 200 M rows in 80 GB
Bytes (K): each row's time (8 B), key code (4 B) and value columns (8 B each) are read, each output (8 B) written -- the
minimum; the kernel reads the inputs twice (reduce pass, then apply pass), and the peer pass reads only the tiles whose last
peer group runs past the tile.  The HBM fraction is against the H100 SXM data sheet's 3.35 TB/s.  The card's name, power limit
and SM clock are read in the same run; without a GPU the script fails.  Nothing is written to disk."""
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

AGGS = [(L.WIN_AVG, 0), (L.WIN_MAX, 1), (L.WIN_SUM, 1), (L.WIN_COUNT, 0)]
AGGD = {"avg_bid": "AVG(bid)", "max_ask": "MAX(ask)", "sum_ask": "SUM(ask)", "n": "count(*)"}


def model_bytes(n: int, nvals: int, nout: int) -> tuple:
    """(minimum bytes, bytes the kernel moves): inputs once and outputs once; the kernel reads the inputs twice."""
    inputs = n * (8 + 4 + 8 * nvals)
    return inputs + n * 8 * nout, 2 * inputs + n * 8 * nout


def torch_sum_count(time: torch.Tensor, codes: torch.Tensor, v: torch.Tensor, tumbling: bool, param: int):
    """(SUM, COUNT) of the per-event window in torch, rows in key-segmented order: a global cumsum minus the prefix before the
    row's run start, both read at the row's peer end.  The subtraction cancels: SUM is not within the kernel's error bound."""
    n = time.numel()
    idx = torch.arange(n, device=time.device)
    new = torch.ones(n, dtype=torch.bool, device=time.device)
    end = torch.ones(n, dtype=torch.bool, device=time.device)
    if n > 1:
        key_change = codes[1:] != codes[:-1]
        if tumbling:
            brk = torch.div(time[1:], param, rounding_mode="floor") != torch.div(time[:-1], param, rounding_mode="floor")
        else:
            brk = (time[1:] - time[:-1]) > param
        new[1:] = key_change | brk
        end[:-1] = key_change | (time[1:] != time[:-1])
    start = torch.cummax(torch.where(new, idx, torch.zeros_like(idx)), 0).values
    peer = torch.flip(torch.cummin(torch.flip(torch.where(end, idx, torch.full_like(idx, n)), [0]), 0).values, [0])
    cs = torch.cumsum(v, 0)
    before = torch.where(start > 0, cs[(start - 1).clamp(min=0)], torch.zeros_like(v))
    return cs[peer] - before, peer - start + 1


def leg(name, n, nbytes, ms, extra=None):
    least, moved = nbytes
    out = {"leg": name, "rows": n, "ms": ms, "rows_per_s": n / (ms / 1e3), "min_bytes": least, "kernel_bytes": moved,
           "gb_per_s_kernel_bytes": moved / (ms / 1e3) / 1e9,
           "hbm_frac_of_3.35TBs_datasheet_kernel_bytes": moved / (HBM_PEAK_TBS * 1e12) / (ms / 1e3),
           "hbm_frac_of_3.35TBs_datasheet_min_bytes": least / (HBM_PEAK_TBS * 1e12) / (ms / 1e3)}
    return out | (extra or {})


def main(argv=None, dev=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--rows", type=int, default=200_000_000, help="quotes")
    ap.add_argument("--symbols", type=int, default=8000)
    ap.add_argument("--reps", type=int, default=10, help="timed calls per kernel measurement")
    ap.add_argument("--steps", type=int, default=2, help="timed runs of each program leg")
    ap.add_argument("--legs", default="KTDC")
    ap.add_argument("--completion-rows", type=int, default=50_000_000, help="quotes of the C legs")
    args = ap.parse_args(argv)
    if dev is None:
        if not torch.cuda.is_available():
            raise SystemExit("bench_window_events: no CUDA device (there is no CPU path to measure)")
        dev = torch.device("cuda", torch.cuda.current_device())
    from quokka_b200 import synth
    from quokka_b200.columns import DeviceColumn, DeviceTable
    from quokka_b200.df import QuokkaContext
    from quokka_b200.windowtypes import OnCompletionTrigger, OnEventTrigger, SessionWindow, TumblingWindow
    q = synth.ticks(synth.T_QUOTES, args.rows, args.symbols, columns=["time", "symbol", "bid", "ask"], device=dev)
    n = args.rows
    span = int(q["time"][-1].item() - q["time"][0].item())
    g = max(1, span * args.symbols // max(1, n))
    windows = {"tumbling": (L.WIN_RUN_TUMBLING, 64 * g), "session": (L.WIN_RUN_SESSION, 2 * g)}
    line = {"card_name_powerlimit_smclock_maxclock": card(), "workload": f"{n} quotes, {args.symbols} symbols, tumbling size "
            f"{64 * g}, session timeout {2 * g} (time units; {g} between two quotes of a symbol on average)", "legs": []}
    clock = []
    codes = q["symbol"].to(torch.int32).contiguous()
    dest, seg = ops.partition_plan(codes, args.symbols, L.PART_CODE)
    time, kc, bid, ask = ops.scatter([q["time"], codes, q["bid"].to(torch.float64), q["ask"].to(torch.float64)], dest)
    del codes, dest
    kernel_count = {}
    for name in args.legs:
        if name in "DC" and time is not None:          # the programs need the memory the kernel legs' inputs hold
            time = kc = bid = ask = None
            kernel_count.clear()
            torch.cuda.empty_cache()
        for wname, (kind, param) in windows.items():
            if name == "K":
                run = lambda: ops.window_sliding(time, kc, seg, args.symbols, param, [bid, ask], AGGS, run=kind)
                kernel_count[wname] = run()[3]
                ms = event_ms(run, args.reps)
                line["legs"].append(leg(f"K qk_window_running {wname}", n, model_bytes(n, 2, len(AGGS)), ms))
                clock.append(card())
            elif name == "T":
                run = lambda: torch_sum_count(time, kc, ask, kind == L.WIN_RUN_TUMBLING, param)
                ms = event_ms(run, args.reps)
                cnt = run()[1]
                if wname not in kernel_count:
                    kernel_count[wname] = ops.window_sliding(time, kc, seg, args.symbols, param, [bid, ask], AGGS, run=kind)[3]
                same = bool(torch.equal(cnt.to(torch.float64), kernel_count[wname]))
                line["legs"].append({"leg": f"T torch cumsum - run-start prefix at peer end {wname}", "rows": n, "ms": ms,
                                     "count_equal": same})
                clock.append(card())
            elif name in "DC":
                rows = n if name == "D" else min(n, args.completion_rows)
                table = DeviceTable({c: DeviceColumn(v[:rows]) for c, v in q.items()})
                w = (TumblingWindow if wname == "tumbling" else SessionWindow)("time", "symbol", param, AGGD)
                trig = OnEventTrigger() if name == "D" else OnCompletionTrigger()

                def program():
                    qc = QuokkaContext()
                    s = qc.from_device(table, sorted_by="time").windowed_transform(w, trig)
                    return qc.execute_node(s.node, to_arrow=False)
                res, secs, _ = wall(program, args.steps)
                rows_out = len(res)
                del res
                line["legs"].append({"leg": f"{name} DataStream {wname} " + ("OnEventTrigger" if name == "D" else "OnCompletionTrigger"),
                                     "rows": rows, "seconds": secs, "rows_per_s": rows / secs, "rows_out": rows_out})
            torch.cuda.empty_cache()
    line["card_after_each_kernel_leg"] = clock
    print(json.dumps(line), flush=True)
    return line


if __name__ == "__main__":
    main()
