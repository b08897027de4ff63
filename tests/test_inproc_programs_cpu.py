"""DataStream programs on two in-process ranks without a GPU: tests/inproc_link.py run_program_ranks over tests/cpu_shim.py,
with the link protocol restated by tests/xchg_shim.py, once with mailboxes that hold every exchange and once with 1 MB
mailboxes, so that the larger exchanges go in rounds.  The same runner drives the kernels on one GPU in
tests/test_gpu_inproc_programs.py.  Also: the device-resident readers serve the channel of the rank that reads them."""
import numpy as np
import pytest
import torch

import inproc_link as IL
import ranks

MB = 1 << 20


@pytest.mark.parametrize("mailbox_mb", [64, 1], ids=lambda m: f"{m}MB")
@pytest.mark.parametrize("suite", ["api", "sort", "shift", "ordered_join", "asof_strategy"])
def test_suite_on_two_inproc_ranks(suite, mailbox_mb):
    counts = IL.run_program_ranks(2, ranks.SUITES[suite], "cpu", mailbox_mb * MB)
    print(f"{suite} mailbox {mailbox_mb} MB: {dict(counts)}")
    missing = [k for k in IL.REACHES.get(suite, ()) if counts[k] == 0]
    assert not missing, (suite, dict(counts))
    if mailbox_mb == 1 and suite in IL.IN_ROUNDS_AT_1MB:
        assert counts["exchange_rounds"] > 0, dict(counts)


def case_left_join_rank_without_build_rows(qc):
    """A left join with the build side hash-partitioned, where no build key hashes to one rank at three ranks (k % 3 == 0):
    that rank's probe rows must keep their place with NULL build columns -- a string, an fp64 and an int32 column."""
    import pandas as pd
    import pyarrow as pa
    qc.set_config("broadcast_rows", 0)
    qc.set_config("broadcast_cost_based", False)
    rng = np.random.default_rng(5)
    lk = rng.integers(0, 600, 2_000)
    rk = np.array([k for k in range(600) if k % 3 != 0 and k % 7 != 1] * 2, dtype=np.int64)
    left = pd.DataFrame({"k": lk, "a": rng.random(len(lk))})
    right = pd.DataFrame({"rk": rk, "s": rng.choice(["x", "yy", "zzz"], len(rk)), "f": rng.random(len(rk)),
                          "i": rng.integers(-9, 9, len(rk)).astype(np.int32)})
    got = qc.from_arrow(pa.Table.from_pandas(left, preserve_index=False)).join(
        qc.from_arrow(pa.Table.from_pandas(right, preserve_index=False)), left_on="k", right_on="rk", how="left").collect().to_pandas()
    exp = left.merge(right, left_on="k", right_on="rk", how="left").drop(columns=["rk"])
    assert len(got) == len(exp) and (exp.s.isna()).sum() > 0, (len(got), len(exp))
    key = ["k", "a", "f"]
    g = got[key + ["s", "i"]].sort_values(key, na_position="first").reset_index(drop=True)
    e = exp[key + ["s", "i"]].sort_values(key, na_position="first").reset_index(drop=True)
    for c in key:
        assert np.array_equal(g[c].to_numpy(dtype=np.float64), e[c].to_numpy(dtype=np.float64), equal_nan=True), c
    assert g.s.isna().tolist() == e.s.isna().tolist() and g.s.dropna().tolist() == e.s.dropna().tolist()
    assert g.i.isna().tolist() == e.i.isna().tolist() and g.i.dropna().astype(np.int64).tolist() == e.i.dropna().astype(np.int64).tolist()


@pytest.mark.parametrize("world", [2, 3])
def test_left_join_on_a_rank_without_build_rows(world):
    IL.run_program_ranks(world, ["test_inproc_programs_cpu:case_left_join_rank_without_build_rows"], "cpu", 64 * MB)


def test_device_readers_serve_the_rank_that_reads_them(monkeypatch):
    """Without RANK in the environment (a launcher that passes rank and world to init_process_group), rank 1 still reads
    channel 1."""
    import cpu_shim
    from quokka_b200.columns import DeviceColumn, DeviceTable
    from quokka_b200.dataset import InputDeviceDataset, InputPinnedDataset
    monkeypatch.delenv("RANK", raising=False)
    cpu_shim.install(monkeypatch)
    IL.install(monkeypatch)

    def body(r):
        dev = InputDeviceDataset(DeviceTable({"x": DeviceColumn(torch.arange(10))}), batch_rows=4)
        pinned = InputPinnedDataset.__new__(InputPinnedDataset)      # pinned host memory needs CUDA; the channel does not
        pinned.n, pinned.chunk_rows = 10, 4
        return sorted(dev.get_own_state(2)), sorted(pinned.get_own_state(2))

    assert IL.run_ranks(IL.InprocLink(2, 1 << 16, "cpu", cpu_shim), body) == [([0], [0]), ([1], [1])]


def test_left_join_executor_without_build_rows(monkeypatch):
    """BuildProbeJoinExecutor on a rank without build rows: a left join emits nothing until it has a template row, then its
    probe rows with NULL build columns of the template's types, the build key dropped."""
    import cpu_shim
    from quokka_b200.columns import DeviceColumn, DeviceTable
    from quokka_b200.executors import BuildProbeJoinExecutor
    cpu_shim.install(monkeypatch)
    ex = BuildProbeJoinExecutor(left_on="k", right_on="rk", how="left")
    probe = DeviceTable({"k": DeviceColumn(torch.tensor([4, 1, 7])), "a": DeviceColumn(torch.tensor([0.5, 1.5, 2.5], dtype=torch.float64))})
    assert ex.execute([probe], 0, 0) is None
    ex.set_left_template(DeviceTable({"rk": DeviceColumn(torch.tensor([9])), "v": DeviceColumn(torch.tensor([3], dtype=torch.int32)),
                                      "s": DeviceColumn(torch.tensor([0], dtype=torch.int32), ["x"])}))
    out = ex.execute([probe], 0, 0)
    assert out.column_names == ["k", "a", "v", "s"]
    assert out["k"].data.tolist() == [4, 1, 7] and out["a"].data.tolist() == [0.5, 1.5, 2.5]
    assert out["v"].data.dtype == torch.int32 and out["v"].valid.tolist() == [0, 0, 0]
    assert out["s"].dictionary == ["x"] and out["s"].valid.tolist() == [0, 0, 0]
