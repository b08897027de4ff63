"""tools/bench_shift.py end to end on the numpy shims (tests/cpu_shim.py + tests/shift_shim.py) with the oracle generator standing
in for the CUDA generator: argument parsing, every leg, the byte model and the check fields.  The numbers it prints here mean
nothing; run as a program without a GPU it fails."""
import importlib.util
import os
import subprocess
import sys
import time

import pytest
import torch

import shift_shim
import test_bench_flow as TBF

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cpu_ms(fn, reps):
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    return max((time.perf_counter() - t0) * 1e3 / reps, 1e-6)


def _load():
    spec = importlib.util.spec_from_file_location("bench_shift", os.path.join(ROOT, "tools", "bench_shift.py"))
    bs = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bs)
    return bs


def test_byte_model():
    bs = _load()
    assert bs.model_bytes(1000, 4, True) == 1000 * (8 + 16 + 4 + 8)
    assert bs.model_bytes(1000, 8, False) == 1000 * (4 + 4 + 16)


def test_torch_formulation_matches_the_reference():
    import numpy as np
    import shift_cases as SC
    bs = _load()
    codes = np.random.default_rng(2).integers(0, 13, 500).astype(np.int32)
    for n in (1, 2, 4):
        assert np.array_equal(bs.torch_src(torch.from_numpy(codes), n).numpy(), SC.reference_src(codes, n, 500))


def test_bench_shift_on_the_shim(monkeypatch):
    TBF.install(monkeypatch)
    ops = shift_shim.install(monkeypatch)
    bs = _load()
    monkeypatch.setattr(bs, "ops", ops)
    monkeypatch.setattr(bs, "event_ms", _cpu_ms)
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
