"""tools/bench_knn.py end to end on the numpy shims (tests/cpu_shim.py + tests/knn_shim.py) at a tiny size: argument parsing, both
dtypes, the roofline, the torch baseline and the agreement check.  The numbers it prints here mean nothing."""
import importlib.util
import os
import time

import torch

import knn_shim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cpu_ms(fn, reps):
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    return (time.perf_counter() - t0) * 1e3 / reps


def test_bench_knn_tiny_on_the_shim(monkeypatch):
    ops = knn_shim.install(monkeypatch)
    spec = importlib.util.spec_from_file_location("bench_knn", os.path.join(ROOT, "tools", "bench_knn.py"))
    bk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bk)
    monkeypatch.setattr(bk, "ops", ops)
    monkeypatch.setattr(bk, "event_ms", _cpu_ms)
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
