"""tests/ranks.py spawn on a rank that outlives its timeout: the run fails naming that rank, and no rank process is left."""
import os
import time

import pytest

import ranks


def _sleeper(rank, world, port, out_dir):
    open(os.path.join(out_dir, f"pid{rank}"), "w").write(str(os.getpid()))
    if rank == 1:
        time.sleep(600)
    open(os.path.join(out_dir, f"ok{rank}"), "w").write("ok")


def test_spawn_terminates_a_hung_rank(tmp_path):
    with pytest.raises(AssertionError, match=r"rank\(s\) \[1\] still running"):
        ranks.spawn(tmp_path, 2, _sleeper, timeout=10)
    pids = [int(open(tmp_path / f"pid{r}").read()) for r in range(2)]
    assert not [p for p in pids if os.path.exists(f"/proc/{p}")]
