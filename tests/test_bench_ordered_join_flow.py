"""tools/bench_ordered_join.py end to end on the numpy shim (tests/cpu_shim.py) with the oracle generator standing in for the
CUDA generator: argument parsing, every leg, the byte model and the check fields.  The numbers it prints here mean nothing; run
as a program without a GPU it fails."""
import os
import subprocess
import sys

import pytest
import torch

import cpu_shim
import test_bench_flow as TBF

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_byte_model():
    bj = TBF.load_tool("bench_ordered_join")
    assert bj.model_bytes(1000, 8, 1000, False) == 1000 * (8 + 32) + 1000 * 8
    assert bj.model_bytes(1000, 8, 3000, True) == 1000 * (2 * (8 + 32) + 8 + 16) + 3000 * 8


def test_bench_ordered_join_on_the_shim(monkeypatch):
    TBF.install(monkeypatch)
    bj = TBF.load_tool("bench_ordered_join")
    monkeypatch.setattr(bj, "ops", cpu_shim)
    monkeypatch.setattr(bj, "event_ms", TBF.cpu_ms)
    monkeypatch.setattr(bj, "card", lambda: "cpu")
    line = bj.main(["--rows", "5000", "--symbols", "37", "--sf", "0.002", "--reps", "1", "--steps", "1"], dev=torch.device("cpu"))
    ku, ko, do, ds, lo, ls = line["legs"]
    assert [x["leg"][0] for x in line["legs"]] == list("KKDDLL") and line["card_name_powerlimit_smclock_maxclock"] == "cpu"
    assert ku["pairs"] == ko["pairs"] == 5000 and ko["algorithmic_bytes"] == bj.model_bytes(5000, 4, 5000, True)
    assert ds["same_rows"] is True and ls["same_rows"] is True
    assert do["rows"] == 5000 and lo["build_rows"] > 0


def test_bench_ordered_join_fails_without_a_gpu():
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "bench_ordered_join.py"), "--rows", "10"], capture_output=True, text=True)
    assert r.returncode != 0 and "no CUDA device" in r.stderr + r.stdout
