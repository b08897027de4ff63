"""tools/bench_shift.py end to end on the numpy shim (tests/cpu_shim.py) with the oracle generator standing
in for the CUDA generator: argument parsing, every leg, the byte model and the check fields.  The numbers it prints here mean
nothing; run as a program without a GPU it fails."""
import os
import subprocess
import sys

import pytest
import torch

import cpu_shim
import test_bench_flow as TBF

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_byte_model():
    bs = TBF.load_tool("bench_shift")
    assert bs.model_bytes(1000, 4, True) == 1000 * (8 + 16 + 4 + 8)
    assert bs.model_bytes(1000, 8, False) == 1000 * (4 + 4 + 16)


def test_torch_formulation_matches_the_reference():
    import numpy as np
    import shift_cases as SC
    bs = TBF.load_tool("bench_shift")
    codes = np.random.default_rng(2).integers(0, 13, 500).astype(np.int32)
    for n in (1, 2, 4):
        assert np.array_equal(bs.torch_src(torch.from_numpy(codes), n).numpy(), SC.reference_src(codes, n, 500))


def test_bench_shift_on_the_shim(monkeypatch):
    TBF.install(monkeypatch)
    bs = TBF.load_tool("bench_shift")
    monkeypatch.setattr(bs, "ops", cpu_shim)
    monkeypatch.setattr(bs, "event_ms", TBF.cpu_ms)
    monkeypatch.setattr(bs, "card", lambda: "cpu")
    line = bs.main(["--rows", "5000", "--symbols", "37", "--reps", "1", "--steps", "1"], dev=torch.device("cpu"))
    k, nk, t, d, e = line["legs"]
    assert [x["leg"][0] for x in line["legs"]] == list("KNTDE") and line["card_name_powerlimit_smclock_maxclock"] == "cpu"
    assert k["algorithmic_bytes"] == bs.model_bytes(5000, 4, True) and nk["algorithmic_bytes"] == bs.model_bytes(5000, 4, False)
    assert t["src_equal"] is True
    assert d["null_rows"] == 37 and e["null_rows"] == 1 and d["rows"] == e["rows"] == 5000


def test_bench_shift_fails_without_a_gpu():
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "bench_shift.py"), "--rows", "10"], capture_output=True, text=True)
    assert r.returncode != 0 and "no CUDA device" in r.stderr + r.stdout
