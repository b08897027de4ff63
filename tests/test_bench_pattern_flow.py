"""tools/bench_pattern.py end to end on the numpy shim (tests/cpu_shim.py) at a tiny size: argument
parsing, the quantile thresholds, both legs, the one-pass bytes and the host arm's agreement checks (restated search, oracle).  The numbers it prints here
mean nothing."""
import numpy as np
import torch

import cpu_shim
import test_bench_flow as TBF


def _quotes(n, n_symbols, dev):
    """Time-sorted quotes from a seeded numpy generator, in synth.ticks' column types."""
    rng = np.random.default_rng(1)
    ask = 100 + rng.standard_normal(n).cumsum() * 0.01
    return {"time": torch.from_numpy(np.sort(rng.integers(0, n * 100, n)).astype(np.int64)),
            "symbol": torch.from_numpy(rng.integers(0, n_symbols, n).astype(np.int32)),
            "bid": torch.from_numpy((ask - 0.05).astype(np.float32)), "ask": torch.from_numpy(ask.astype(np.float32)),
            "asize": torch.from_numpy(rng.integers(1, 100, n).astype(np.float32))}


def test_bench_pattern_tiny_on_the_shim(monkeypatch):
    cpu_shim.install(monkeypatch)
    bp = TBF.load_tool("bench_pattern")
    monkeypatch.setattr(bp, "ops", cpu_shim)
    monkeypatch.setattr(bp, "event_ms", TBF.cpu_ms)
    monkeypatch.setattr(bp, "card", lambda: "cpu")
    monkeypatch.setattr(bp, "quotes", _quotes)
    out = bp.main(["--rows", "3000", "--symbols", "7", "--reps", "1", "--sample", "1200"], dev=torch.device("cpu"))
    assert [leg["leg"] for leg in out["legs"]] == ["A", "B"]
    for leg in out["legs"]:
        assert leg["starts"] > 0 and leg["matches"] == leg["result_rows"] > 0
        assert leg["one_pass_bytes"] == 3000 * sum({"time": 8, "symbol": 4}.get(c, 4) for c in leg["touched_columns"])
        assert leg["host_arm"]["device_equals_host"] and leg["host_arm"]["rows"] == 1200
        assert leg["host_arm"]["device_equals_oracle"] and leg["host_arm"]["oracle_matches"] > 0
    assert out["legs"][0]["touched_columns"] == ["asize", "symbol", "time"]
