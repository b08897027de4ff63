"""tools/bench_knn.py end to end on the numpy shim (tests/cpu_shim.py) at a tiny size: argument parsing, both
dtypes, the roofline, the torch baseline and the agreement check.  The numbers it prints here mean nothing."""
import torch

import cpu_shim
import test_bench_flow as TBF


def test_bench_knn_tiny_on_the_shim(monkeypatch):
    cpu_shim.install(monkeypatch)
    bk = TBF.load_tool("bench_knn")
    monkeypatch.setattr(bk, "ops", cpu_shim)
    monkeypatch.setattr(bk, "event_ms", TBF.cpu_ms)
    monkeypatch.setattr(bk, "card", lambda: "cpu")
    out = bk.main(["--rows", "2001", "--dim", "24", "--probes", "1,17", "--k", "10", "--reps", "1"], dev=torch.device("cpu"))
    assert [(c["dtype"], c["q"]) for c in out["cases"]] == [("f32", 1), ("f32", 17), ("f16", 1), ("f16", 17)]
    tiny = bk.main(["--tiny", "--reps", "1", "--dtypes", "f32"], dev=torch.device("cpu"))
    assert (tiny["rows"], tiny["dim"], [c["q"] for c in tiny["cases"]]) == (4096, 64, [1, 17])
    for c in out["cases"]:
        esize = 4 if c["dtype"] == "f32" else 2
        assert c["roofline"]["algorithmic_bytes"] == 2001 * 24 * esize
        assert c["roofline"]["algorithmic_flops"] == 2 * 2001 * 24 * c["q"] * (3 if c["dtype"] == "f32" else 2)
        assert c["agree_outside_tie_band"] == 1.0
