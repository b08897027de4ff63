"""OrderedStream.shift without a GPU: the pandas reference against pandas' own fills, the numpy stand-ins of the shift kernels
(tests/shift_shim.py) against the reference for every key, n and size case, the edge flags, the order-check count, both gather
sources, and the API cases through the planner and the executors on the shims."""
import numpy as np
import pytest
import torch

import cpu_shim
import shift_api_cases as A
import shift_cases as SC
import shift_shim
from quokka_b200 import _lib as L


def _plan(keys, n, nrows, **kw):
    """shift_shim.shift_plan over `keys` (None = one key), with the stable code partition the executor feeds it."""
    if keys is None:
        return shift_shim.shift_plan(n, nrows, **kw)
    codes = torch.from_numpy(keys)
    n_by = int(keys.max()) + 1 if len(keys) else 1
    dest, seg = cpu_shim.partition_plan(codes, n_by, L.PART_CODE)
    return shift_shim.shift_plan(n, nrows, codes, n_by, dest, seg, **kw)


def test_reference_matches_pandas_fill():
    rng = np.random.default_rng(0)
    keys, v = rng.integers(0, 5, 300), rng.standard_normal(300)
    for n in (1, -2, 7, 0):
        got = SC.reference_shift(keys, n, {"v": (v, None)}, fill=9.5)["v"][0]
        assert np.array_equal(got, SC.pandas_shift(keys, n, v, 9.5)), n
    assert SC.reference_src(None, 2, 5).tolist() == [-1, -1, 0, 1, 2]
    assert SC.reference_src(np.array([0, 1, 0, 0, 1]), -1, 5).tolist() == [2, 4, 3, -1, -1]


@pytest.mark.parametrize("nrows", SC.SIZES)
def test_shim_plan_matches_the_reference(nrows):
    for name, keys in SC.key_cases(nrows):
        for n in SC.n_cases(nrows):
            src, _, _ = _plan(keys, n, nrows)
            assert np.array_equal(src.numpy().astype(np.int64), SC.reference_src(keys, n, nrows)), (name, n)


def test_plan_numbers_sources_from_lo():
    """[B | A] with lo = len(B): A's rows come first in the numbering, B's after them -- the gather's two tables."""
    keys = np.array([0, 1, 0, 1, 0, 0, 1], np.int32)          # B = the first three rows
    src, _, _ = _plan(keys, 1, 7, lo=3, hi=7)
    ref = SC.reference_src(keys, 1, 7)[3:]                     # rows 1, 2, 4, 3 of the whole
    exp = np.where(ref >= 3, ref - 3, np.where(ref >= 0, ref + 4, -1))
    assert src.numpy().tolist() == exp.tolist() == [5, 6, 1, 0]


def test_edge_flags():
    keys = np.array([0, 1, 0, 0, 2, 1, 0], np.int32)
    _, lag2, _ = _plan(keys, 2, 7, lo=0, hi=0, want_edge=True)
    assert lag2.numpy().tolist() == [0, 1, 0, 1, 1, 1, 1]       # the last two rows of every key
    _, lead1, _ = _plan(keys, -1, 7, lo=0, hi=0, want_edge=True)
    assert lead1.numpy().tolist() == [1, 1, 0, 0, 1, 0, 0]      # the first row of every key
    _, none, _ = _plan(None, 3, 7, lo=0, hi=0, want_edge=True)
    assert none.numpy().tolist() == [0, 0, 0, 0, 1, 1, 1]
    _, huge, _ = _plan(keys, SC.HUGE, 7, lo=0, hi=0, want_edge=True)
    assert huge.numpy().tolist() == [1] * 7
    _, zero, _ = _plan(keys, 0, 7, lo=0, hi=0, want_edge=True)
    assert zero.numpy().tolist() == [0] * 7


def test_order_check_counts_rows_below_their_predecessor():
    keys = np.array([0, 1, 0, 1, 0], np.int32)
    time = torch.tensor([5, 1, 4, 2, 4], dtype=torch.int64)    # key 0: 5, 4, 4 (one drop); key 1: 1, 2
    assert _plan(keys, 1, 5, time=time)[2] == 1
    assert _plan(None, 1, 5, time=time)[2] == 2                # 5 > 1 and 4 > 2
    assert _plan(keys, 1, 5, time=torch.tensor([1, 1, 2, 3, 2], dtype=torch.int64))[2] == 0


def test_gather_reads_both_tables_and_fills():
    a = [torch.tensor([10, 11, 12], dtype=torch.int64), torch.tensor([1.5, 2.5, 3.5])]
    b = [torch.tensor([20, 21], dtype=torch.int64), torch.tensor([-1.0, -2.0])]
    src = torch.tensor([4, -1, 0, 3, 2], dtype=torch.int32)
    av = [torch.tensor([1, 0, 1], dtype=torch.uint8), None]
    outs, valid = shift_shim.shift_gather(a, b, src, [7, None], av, [None, None])
    assert outs[0].tolist() == [21, 7, 10, 20, 12] and valid[0].tolist() == [1, 1, 1, 1, 1]
    assert outs[1].tolist() == [-2.0, 0.0, 1.5, -1.0, 3.5] and valid[1].tolist() == [1, 0, 1, 1, 1]
    outs, valid = shift_shim.shift_gather(a, None, torch.tensor([1, -1], dtype=torch.int32), [7, 0.5], av, None)
    assert outs[0].tolist() == [11, 7] and valid[0].tolist() == [0, 1] and valid[1] is None


def test_shim_enforces_the_limits():
    with pytest.raises(L.QkError):
        shift_shim.shift_gather([torch.zeros(4, 2)], None, torch.zeros(4, dtype=torch.int32), [None])
    with pytest.raises(L.QkError):
        shift_shim.shift_plan(1, 4, by=torch.zeros(4, dtype=torch.int32))
    with pytest.raises(L.QkError, match="2\\^31"):
        shift_shim.shift_plan(1, 1 << 31)


def test_no_cpu_fallback():
    from quokka_b200 import ops
    with pytest.raises(L.QkError, match="CUDA tensor"):
        ops.shift_plan(1, 4, by=torch.zeros(4, dtype=torch.int32), n_by=1, dest=torch.zeros(4, dtype=torch.int32),
                       seg=torch.zeros(2, dtype=torch.int64))
    with pytest.raises(L.QkError, match="CUDA tensor"):
        ops.shift_gather([torch.zeros(4)], None, torch.zeros(4, dtype=torch.int32), [None])


def test_fill_conversion():
    import datetime
    import pyarrow as pa
    from quokka_b200.columns import DeviceColumn
    from quokka_b200.executors import shift_fill
    i32, f64 = DeviceColumn(torch.zeros(1, dtype=torch.int32)), DeviceColumn(torch.zeros(1, dtype=torch.float64))
    assert shift_fill(i32, "a", -7) == (-7, None) and shift_fill(f64, "b", 3) == (3.0, None)
    for col, bad in ((i32, 1.5), (i32, 1 << 31), (i32, "x"), (i32, True), (f64, "1")):
        with pytest.raises(L.QkError, match="column 'c'"):
            shift_fill(col, "c", bad)
    s = DeviceColumn(torch.zeros(1, dtype=torch.uint8), ["a", "b"])
    assert shift_fill(s, "s", "b") == (1, ["a", "b"]) and shift_fill(s, "s", "z") == (2, ["a", "b", "z"]) and s.dictionary == ["a", "b"]
    d = DeviceColumn(torch.zeros(1, dtype=torch.int32), None, pa.date32())
    assert shift_fill(d, "d", datetime.date(1970, 1, 11))[0] == 10
    with pytest.raises(L.QkError):
        shift_fill(d, "d", datetime.datetime(1970, 1, 11))
    ts = DeviceColumn(torch.zeros(1, dtype=torch.int64), None, pa.timestamp("ms"))
    assert shift_fill(ts, "t", datetime.datetime(1970, 1, 1, 0, 0, 2))[0] == 2000 and shift_fill(ts, "t", 5)[0] == 5
    b = DeviceColumn(torch.zeros(1, dtype=torch.uint8), None, pa.bool_())
    assert shift_fill(b, "f", True)[0] == 1
    with pytest.raises(L.QkError):
        shift_fill(b, "f", 1)
    assert shift_fill(i32, "a", None) == (None, None)


@pytest.fixture
def qc(monkeypatch):
    cpu_shim.install(monkeypatch)
    from quokka_b200.df import QuokkaContext
    return QuokkaContext()


def test_shift_lag_lead(qc): A.case_shift_lag_lead(qc)
def test_shift_in_place(qc): A.case_shift_in_place(qc)
def test_shift_fills(qc): A.case_shift_fills(qc)
def test_shift_nulls_from_left_join(qc): A.case_shift_nulls_from_left_join(qc)
def test_sort_then_shift(qc): A.case_sort_then_shift(qc)
def test_shift_then_asof(qc, golden_dir): A.case_shift_then_asof(qc, golden_dir)
def test_shift_out_of_order(qc): A.case_shift_out_of_order(qc)
def test_shift_errors(qc): A.case_shift_errors(qc)


def test_explain_prints_the_shift(qc, capsys):
    import pyarrow as pa
    s = qc.from_arrow_sorted(pa.table({"t": [1, 2, 3], "k": [0, 1, 0], "v": [1.0, 2.0, 3.0]}), "t").shift(1, "k", columns=["v"], suffix="_p")
    s.explain()
    assert "shift n=1 by=k columns=['v'] suffix=_p" in capsys.readouterr().out
    s.explain("physical")
    assert "ShiftExecutor [ordered]" in capsys.readouterr().out
