"""tools/bench_quantile.py end to end on the numpy shim (tests/cpu_shim.py) with the oracle generator
standing in for the CUDA generator: argument parsing, both legs, the CPU t-digest arm, the roofline and check fields.  The
numbers it prints here mean nothing."""
import torch

import cpu_shim
import test_bench_flow as TBF


def test_bench_quantile_on_the_shim(monkeypatch):
    TBF.install(monkeypatch)
    bq = TBF.load_tool("bench_quantile")
    monkeypatch.setattr(bq, "ops", cpu_shim)
    monkeypatch.setattr(bq, "event_ms", TBF.cpu_ms)
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
