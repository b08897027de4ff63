"""tools/bench_gram.py end to end on the numpy shim (tests/cpu_shim.py) with the oracle generator standing in
for the CUDA generator: argument parsing, both legs, the roofline and check fields.  The numbers it prints here mean nothing."""
import torch

import cpu_shim
import test_bench_flow as TBF


def test_bench_gram_on_the_shim(monkeypatch):
    TBF.install(monkeypatch)
    bg = TBF.load_tool("bench_gram")
    monkeypatch.setattr(bg, "ops", cpu_shim)
    monkeypatch.setattr(bg, "event_ms", TBF.cpu_ms)
    monkeypatch.setattr(bg, "card", lambda: "cpu")
    line = bg.main(["--sf", "0.01", "--rows", "3001", "--cols", "37", "--reps", "1", "--steps", "1"], dev=torch.device("cpu"))
    narrow, wide = line["narrow"], line["wide"]
    assert narrow["roofline"]["bound"] == "hbm" and narrow["roofline"]["algorithmic_bytes"] == 8 * 4 * 60_000           # SF-0.01 lineitem
    assert narrow["vs_torch_fp64_bound_ratio"] <= 2
    assert wide["roofline"]["algorithmic_flops"] == 3001 * 37 * 38
    assert len(wide["variants_ms"]) == 1 and wide["vs_torch_fp64_bound_ratio"] <= 2 and wide["torch_fp64_xtx_ms"] > 0
