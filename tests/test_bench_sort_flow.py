"""tools/bench_sort.py end to end on the numpy shim (tests/cpu_shim.py) with the oracle generator standing in
for the CUDA generator: argument parsing, every leg, the byte model and the check fields.  The numbers it prints here mean
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
    bs = TBF.load_tool("bench_sort")
    n = 1000
    assert bs.model_bytes(n, 4, 2) == n * (4 + 12) + n * 8 * 2 + n * 24 + n * 16          # pass 0, two counts, one full scatter, the last one
    assert bs.model_bytes(n, 8, 8) == n * 20 + n * 64 + n * 24 * 7 + n * 16
    assert bs.model_bytes(n, 8, 1, null_pass=True) == n * 20 + n * 8 + n * 4 + n * 24 + n * 16
    assert bs.model_bytes(n, 8, 0) == n * (8 + 12 + 12 + 4)


def test_bench_sort_on_the_shim(monkeypatch):
    TBF.install(monkeypatch)
    bs = TBF.load_tool("bench_sort")
    plans = []

    class Ops:
        @staticmethod
        def sort_perm(key, valid, descending, perm_in=None, want_image=False):
            distinct_bytes = sum(len(set(((int(v) >> (8 * d)) & 0xff) for v in key.view(torch.int64 if key.element_size() == 8 else torch.int32).tolist())) > 1 for d in range(key.element_size()))
            plans.append(f"d8 passes={distinct_bytes}/8 nulls=0")
            return cpu_shim.sort_perm(key, valid, descending, perm_in, want_image)

        @staticmethod
        def sort_last_plan():
            return plans[-1]
    monkeypatch.setattr(bs, "ops", Ops)
    monkeypatch.setattr(bs, "event_ms", TBF.cpu_ms)
    monkeypatch.setattr(bs, "card", lambda: "cpu")
    line = bs.main(["--sf", "0.01", "--rows", "3001", "--api-sf", "0.01", "--asof-quotes", "5000", "--reps", "1", "--steps", "1"],
                   dev=torch.device("cpu"))
    a, b, c, d, e = line["legs"]
    assert [x["leg"][0] for x in line["legs"]] == list("ABCDE") and line["card_name_powerlimit_smclock_maxclock"] == "cpu"
    for leg, kb in ((a, 4), (b, 8), (c, 8)):
        assert leg["equals_torch_indices"] is True and leg["timed_calls"] == 1
        assert leg["algorithmic_bytes"] == bs.model_bytes(leg["rows"], kb, leg["live_passes"])
    assert a["rows"] == c["rows"] == d["rows"] and b["rows"] == 3001 and b["live_passes"] == 8 and a["live_passes"] <= 2
    assert d["sorted"] is True
    assert e["same_matches"] is True and e["sort_then_join_seconds"] > 0


def test_bench_sort_fails_without_a_gpu():
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "bench_sort.py"), "--sf", "0.001", "--rows", "10"], capture_output=True, text=True)
    assert r.returncode != 0 and "no CUDA device" in r.stderr + r.stdout
