"""tools/bench_window_events.py end to end on the numpy shims (tests/cpu_shim.py, tests/window_events_shim.py) with the oracle
generator standing in for the CUDA generator: argument parsing, every leg, the byte model and the check fields.  The numbers it
prints here mean nothing; run as a program without a GPU it fails."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import cpu_shim
import test_bench_flow as TBF
import window_events_shim as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_byte_model():
    bw = TBF.load_tool("bench_window_events")
    assert bw.model_bytes(1000, 2, 4) == (1000 * (8 + 4 + 16 + 32), 1000 * (2 * (8 + 4 + 16) + 32))


@pytest.mark.parametrize("kind,param", [("tumbling", 5), ("session", 2), ("session", 0)])
def test_torch_formulation_matches_the_reference(kind, param):
    bw = TBF.load_tool("bench_window_events")
    rng = np.random.default_rng(4)
    n = 600
    by = np.sort(rng.integers(0, 7, n)).astype(np.int32)
    time = np.zeros(n, np.int64)
    for k in np.unique(by):
        m = by == k
        time[m] = np.sort(rng.integers(-30, 30, m.sum()))
    v = rng.integers(-100, 100, n) / 4.0
    s, c = bw.torch_sum_count(torch.from_numpy(time), torch.from_numpy(by), torch.from_numpy(v), kind == "tumbling", param)
    ref = S.running_window(time, by, kind, param, {"s": ("sum", v), "n": ("count", None)})
    assert np.array_equal(c.numpy(), ref["n"]) and np.array_equal(s.numpy(), ref["s"])


def test_bench_window_events_on_the_shim(monkeypatch):
    TBF.install(monkeypatch)
    bw = TBF.load_tool("bench_window_events")
    monkeypatch.setattr(bw, "ops", cpu_shim)
    monkeypatch.setattr(bw, "event_ms", TBF.cpu_ms)
    monkeypatch.setattr(bw, "card", lambda: "cpu")
    line = bw.main(["--rows", "3000", "--symbols", "17", "--reps", "1", "--steps", "1"], dev=torch.device("cpu"))
    legs = line["legs"]
    assert [x["leg"][0] for x in legs] == list("KKTTDDCC") and line["card_name_powerlimit_smclock_maxclock"] == "cpu"
    assert legs[0]["kernel_bytes"] == bw.model_bytes(3000, 2, 4)[1]
    assert legs[2]["count_equal"] is True and legs[3]["count_equal"] is True
    assert legs[4]["rows_out"] == legs[5]["rows_out"] == 3000
    assert 0 < legs[6]["rows_out"] < 3000 and 0 < legs[7]["rows_out"] < 3000


def test_bench_window_events_fails_without_a_gpu():
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "bench_window_events.py"), "--rows", "10"], capture_output=True, text=True)
    assert r.returncode != 0 and "no CUDA device" in r.stderr + r.stdout
