"""tools/bench_asof_strategy.py end to end on the numpy shims (tests/cpu_shim.py, tests/asof_strategy_shim.py) with the oracle
generator standing in for the CUDA generator: argument parsing, every leg, and the three forward formulations agreeing.  The
numbers it prints here mean nothing; run as a program without a GPU it fails."""
import os
import subprocess
import sys

import pytest
import torch

import cpu_shim
import test_bench_flow as TBF

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_bench_asof_strategy_on_the_shim(monkeypatch):
    TBF.install(monkeypatch)
    bj = TBF.load_tool("bench_asof_strategy")
    monkeypatch.setattr(bj, "ops", cpu_shim)
    monkeypatch.setattr(bj, "event_ms", TBF.cpu_ms)
    monkeypatch.setattr(bj, "card", lambda: "cpu")
    line = bj.main(["--quotes", "4000", "--trades", "900", "--symbols", "37", "--tolerance", "3000", "--reps", "1", "--steps", "1"],
                   dev=torch.device("cpu"))
    legs = line["legs"]
    assert [x["leg"][0] for x in legs] == list("KKKKKKKKDDD") and line["card_name_powerlimit_smclock_maxclock"] == "cpu"
    assert legs[6]["same_answer"] is True and legs[7]["same_answer"] is True
    assert all(x["rows"] == 4900 for x in legs)


def test_bench_asof_strategy_fails_without_a_gpu():
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "bench_asof_strategy.py"), "--quotes", "10"], capture_output=True, text=True)
    assert r.returncode != 0 and "no CUDA device" in r.stderr + r.stdout
