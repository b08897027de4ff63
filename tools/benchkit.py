"""What the benchmarks under tools/ share: the HBM peak they compare with, the card query and the two timers."""
from __future__ import annotations

import subprocess
import time

import torch

HBM_PEAK_TBS = 3.35                                                           # H100 SXM data sheet (700 W card): HBM3 bandwidth


def card(clocks: bool = False) -> str:
    """Name and power limit of the card, with clocks=True also the SM clock now and at most (a read-only query)."""
    fields = "name,power.limit" + (",clocks.sm,clocks.max.sm" if clocks else "")
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader"], capture_output=True, text=True,
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
