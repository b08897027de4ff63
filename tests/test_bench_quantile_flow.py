"""tools/bench_quantile.py end to end on the numpy shims (tests/cpu_shim.py + tests/quantile_shim.py) with the oracle generator
standing in for the CUDA generator: argument parsing, both legs, the CPU t-digest arm, the roofline and check fields.  The
numbers it prints here mean nothing."""
import importlib.util
import os
import time

import torch

import quantile_shim
import test_bench_flow as TBF

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cpu_ms(fn, reps):
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    return (time.perf_counter() - t0) * 1e3 / reps


def test_bench_quantile_on_the_shim(monkeypatch):
    TBF.install(monkeypatch)
    ops = quantile_shim.install(monkeypatch)
    spec = importlib.util.spec_from_file_location("bench_quantile", os.path.join(ROOT, "tools", "bench_quantile.py"))
    bq = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bq)
    monkeypatch.setattr(bq, "ops", ops)
    monkeypatch.setattr(bq, "event_ms", _cpu_ms)
    monkeypatch.setattr(bq, "card", lambda: "cpu")
    line = bq.main(["--sf", "0.01", "--rows", "3001", "--cols", "37", "--cpu-rows", "20000", "--reps", "1", "--steps", "1"],
                   dev=torch.device("cpu"))
    narrow, wide = line["narrow"], line["wide"]
    assert narrow["roofline"]["algorithmic_bytes"] == 8 * 4 * 60_000                    # SF-0.01 lineitem
    assert narrow["tpch_606_value"] == narrow["tpch_606_exact"]
    assert set(narrow["exact_cols"]) == {"l_quantity", "l_discount", "l_tax"} and narrow["max_rel_err_vs_exact"] <= 2.0 ** -11
    arm = narrow["cpu_arm"]
    assert arm["rows"] == 20_000 and arm["l_tax"]["sketch_rank_err"] == [0.0, 0.0, 0.0] and len(arm["l_extendedprice"]["tdigest"]) == 3
    assert wide["roofline"]["algorithmic_bytes"] == 4 * 3001 * 37 and wide["max_rel_err_vs_exact"] <= 2.0 ** -11
