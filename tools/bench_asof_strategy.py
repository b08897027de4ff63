#!/usr/bin/env python
"""As-of strategy benchmark (OrderedStream.join_asof(strategy=..., tolerance=...) / qk_asof_join, csrc/asof.cu) on one GPU; one
JSON line.

  python tools/bench_asof_strategy.py [--quotes 200000000] [--trades 40000000] [--symbols 8000] [--tolerance 50000] [--reps 10]
                                      [--steps 2] [--legs KD]

Input: device-generated, time-sorted trades and quotes (synth.ticks), `symbols` symbols interleaved.
  K  the kernels alone, CUDA events: backward (qk_asof_merge, today's join) against forward and nearest (qk_asof_join), each
     with and without a tolerance; then forward two other ways: by REVERSAL (both sides flipped, time negated, the backward
     qk_asof_merge, indices mapped back -- the formulation without new CUDA) and by torch.searchsorted over (symbol, time)
     composite keys after a stable sort.  The three forward answers are compared element for element.
  D  the DataStream programs from_device(trades).join_asof(from_device(quotes), strategy=...) for the three strategies.
The card's name, power limit and SM clock are read in the same run; without a GPU the script fails.  Nothing is written to disk."""
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
from benchkit import event_ms, wall
from quokka_b200 import ops

card = functools.partial(benchkit.card, clocks=True)                         # with the SM clock now and at most


def forward_by_reversal(lt, lb, rt, rb, n_by):
    """Forward as-of through the backward kernel: the last right row with -r_time <= -l_time in the reversed streams is the
    first one with r_time >= l_time in the originals (among equal times the earliest)."""
    nl, nr = lt.numel(), rt.numel()
    ridx, _ = ops.asof_merge(-lt.flip(0), lb.flip(0), -rt.flip(0), rb.flip(0), n_by)
    ridx = ridx.flip(0)
    return torch.where(ridx >= 0, nr - 1 - ridx, ridx)


def forward_by_searchsorted(lt, lb, rt, rb):
    """Forward as-of in torch: right rows stably sorted by (symbol, time) as one int64 composite, a lower bound per left row."""
    t0 = torch.minimum(lt.min(), rt.min())
    width = torch.maximum(lt.max(), rt.max()) - t0 + 1
    rc = rb.long() * width + (rt - t0)
    lc = lb.long() * width + (lt - t0)
    rs, order = torch.sort(rc, stable=True)
    pos = torch.searchsorted(rs, lc)
    hit = pos < rs.numel()
    cand = order[pos.clamp(max=max(rs.numel() - 1, 0))]
    hit &= rb[cand] == lb
    return torch.where(hit, cand, torch.full_like(cand, -1)).to(torch.int32)


def _program(trades, quotes, strategy, tolerance):
    from quokka_b200.df import QuokkaContext
    qc = QuokkaContext()
    s = qc.from_device(trades, sorted_by="time").join_asof(qc.from_device(quotes, sorted_by="time"), on="time", by="symbol",
                                                           strategy=strategy, tolerance=tolerance)
    return qc.execute_node(s.node, to_arrow=False)


def main(argv=None, dev=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--quotes", type=int, default=200_000_000)
    ap.add_argument("--trades", type=int, default=40_000_000)
    ap.add_argument("--symbols", type=int, default=8000)
    ap.add_argument("--tolerance", type=int, default=50_000, help="in the time column's unit")
    ap.add_argument("--reps", type=int, default=10, help="timed calls per kernel measurement")
    ap.add_argument("--steps", type=int, default=2, help="timed runs of each program")
    ap.add_argument("--legs", default="KD")
    args = ap.parse_args(argv)
    if dev is None:
        if not torch.cuda.is_available():
            raise SystemExit("bench_asof_strategy: no CUDA device (there is no CPU path to measure)")
        dev = torch.device("cuda", torch.cuda.current_device())
    from quokka_b200 import synth
    from quokka_b200.columns import DeviceColumn, DeviceTable
    nq, nt, nsym, tol = args.quotes, args.trades, args.symbols, args.tolerance
    line = {"card_name_powerlimit_smclock_maxclock": card(),
            "workload": f"{nt} trades, {nq} quotes, {nsym} symbols, tolerance {tol}", "legs": []}
    q = synth.ticks(synth.T_QUOTES, nq, nsym, columns=["time", "symbol", "bid"], device=dev)
    t = synth.ticks(synth.T_TRADES, nt, nsym, columns=["time", "symbol", "size"], device=dev)
    lt, lb, rt, rb = t["time"].contiguous(), t["symbol"].contiguous(), q["time"].contiguous(), q["symbol"].contiguous()
    for name in args.legs:
        if name == "K":
            ms = {}
            for strategy in ("backward", "forward", "nearest"):
                for tl in (None, tol):
                    fn = functools.partial(ops.asof_merge, lt, lb, rt, rb, nsym, strategy=strategy, tolerance=tl)
                    ms[strategy, tl] = event_ms(fn, args.reps)
                    line["legs"].append({"leg": f"K {strategy}" + (f" tolerance {tl}" if tl is not None else ""), "rows": nt + nq,
                                         "ms": ms[strategy, tl], "rows_per_s": (nt + nq) / (ms[strategy, tl] / 1e3)})
            fwd = ops.asof_merge(lt, lb, rt, rb, nsym, strategy="forward")[0]
            ms_rev = event_ms(lambda: forward_by_reversal(lt, lb, rt, rb, nsym), args.reps)
            ms_ss = event_ms(lambda: forward_by_searchsorted(lt, lb, rt, rb), args.reps)
            line["legs"].append({"leg": "K forward by reversal (qk_asof_merge)", "rows": nt + nq, "ms": ms_rev,
                                 "forward_kernel_over_this": ms["forward", None] / ms_rev,
                                 "same_answer": bool(torch.equal(forward_by_reversal(lt, lb, rt, rb, nsym), fwd))})
            line["legs"].append({"leg": "K forward by torch.searchsorted", "rows": nt + nq, "ms": ms_ss,
                                 "forward_kernel_over_this": ms["forward", None] / ms_ss,
                                 "same_answer": bool(torch.equal(forward_by_searchsorted(lt, lb, rt, rb), fwd))})
            line["card_after_kernel_leg"] = card()
        elif name == "D":
            trades = DeviceTable({c: DeviceColumn(v) for c, v in t.items()})
            quotes = DeviceTable({c: DeviceColumn(v) for c, v in q.items()})
            for strategy in ("backward", "forward", "nearest"):
                res, s, _ = wall(lambda: _program(trades, quotes, strategy, None), args.steps)
                line["legs"].append({"leg": f"D join_asof(strategy={strategy!r})", "rows": nt + nq, "seconds": s,
                                     "rows_per_s": (nt + nq) / s, "matched": int(res["bid"].valid.sum().item())
                                     if res["bid"].valid is not None else len(res)})
                del res
        torch.cuda.empty_cache()
    print(json.dumps(line), flush=True)
    return line


if __name__ == "__main__":
    main()
