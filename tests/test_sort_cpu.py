"""DataStream.sort without a GPU: the Python-comparison reference against the image reference and hand-worked orders, the numpy
stand-in of the sort kernel against the reference, SortExecutor's batching invariance, and the API cases through the planner and
the executors on the shims."""
import numpy as np
import pytest
import torch

import cpu_shim
import sort_api_cases as A
import sort_cases as SC
import sort_shim
from quokka_b200 import _lib as L


def test_reference_hand_worked():
    nan, inf = float("nan"), float("inf")
    k = np.array([1.0, nan, -0.0, 0.0, -inf, inf, -nan, -1.0])
    assert SC.reference_perm_small([k], [None], [False]).tolist() == [4, 7, 2, 3, 0, 5, 1, 6]        # -0.0 = 0.0 and NaNs tie, in input order
    assert SC.reference_perm_small([k], [None], [True]).tolist() == [1, 6, 5, 0, 2, 3, 7, 4]
    v = np.array([1, 1, 0, 1, 1, 0, 1, 1], np.uint8)
    assert SC.reference_perm_small([k], [v], [False]).tolist() == [4, 7, 3, 0, 1, 6, 2, 5]           # NULLs last, tied
    assert SC.reference_perm_small([k], [v], [True]).tolist() == [1, 6, 0, 3, 7, 4, 2, 5]            # ... in both directions
    i = np.array([np.iinfo(np.int64).max, -1, np.iinfo(np.int64).min, 0], np.int64)
    assert SC.reference_perm_small([i], [None], [False]).tolist() == [2, 1, 3, 0]
    assert SC.reference_perm_small([i], [None], [True]).tolist() == [0, 3, 1, 2]
    codes, words = np.array([0, 1, 2, 1], np.int32), ["pear", "apple", "Zebra"]
    assert SC.reference_perm_small([codes], [None], [False], [words]).tolist() == [2, 1, 3, 0]       # by the string, not the code


@pytest.mark.parametrize("n", [0, 1, 33, 700])
def test_references_agree(n):
    for name, key in SC.key_cases(n):
        for vname, valid in SC.valid_cases(n):
            for desc in (False, True):
                a, b = SC.reference_perm_small([key], [valid], [desc]), SC.reference_perm([key], [valid], [desc])
                assert np.array_equal(a, b), (name, vname, desc)
    for ncols in (1, 2, 3, 4):
        for seed in (0, 1):
            keys, valids, desc, dicts = SC.multi_column_case(n, ncols, seed)
            assert np.array_equal(SC.reference_perm_small(keys, valids, desc, dicts), SC.reference_perm(keys, valids, desc, dicts)), (ncols, seed)


@pytest.mark.parametrize("n", SC.SIZES)
def test_shim_matches_the_reference(n):
    for name, key in SC.key_cases(n):
        for vname, valid in SC.valid_cases(n)[:2]:
            for desc in (False, True):
                v = None if valid is None else torch.from_numpy(valid)
                perm, image = sort_shim.sort_perm(torch.from_numpy(key), v, desc, want_image=True)
                assert np.array_equal(perm.numpy(), SC.reference_perm([key], [valid], [desc])), (name, vname, desc)
                assert np.array_equal(image.numpy().view(np.uint64), SC.sorted_image(key, valid, desc)), (name, vname, desc)


def test_shim_chains_and_enforces_the_limits():
    keys, valids, desc, _ = SC.multi_column_case(999, 4, 0)
    perm = None
    for k, v, d in list(zip(keys, valids, desc))[::-1]:
        perm = sort_shim.sort_perm(torch.from_numpy(k), None if v is None else torch.from_numpy(v), d, perm)
    assert np.array_equal(perm.numpy(), SC.reference_perm(keys, valids, desc))
    with pytest.raises(L.QkError):
        sort_shim.sort_perm(torch.zeros(4, dtype=torch.int16), None, False)
    with pytest.raises(L.QkError):
        sort_shim.sort_perm(torch.zeros(4, 2), None, False)
    with pytest.raises(L.QkError):
        sort_shim.sort_perm(torch.zeros(4), torch.ones(3, dtype=torch.uint8), False)
    with pytest.raises(L.QkError, match="2\\^31"):
        sort_shim.sort_perm(torch.zeros(1, dtype=torch.uint8).expand(1 << 31), None, False)


def test_no_cpu_fallback():
    from quokka_b200 import ops
    with pytest.raises(L.QkError, match="CUDA tensor"):
        ops.sort_perm(torch.zeros(4), None, False)


def test_sort_executor_batching_invariance(monkeypatch):
    cpu_shim.install(monkeypatch)
    from quokka_b200.columns import DeviceTable
    from quokka_b200.executors import SortExecutor
    keys, valids, desc, dicts = SC.multi_column_case(3000, 4, 1)
    names = ["c0", "c1", "c2", "c3"]
    cols = dict(zip(names, keys)) | {"rowid": np.arange(3000, dtype=np.int64)}
    full = DeviceTable.from_numpy(cols, dictionaries={"c2": dicts[2]})
    full.columns["c1"].valid = torch.from_numpy(valids[1])
    expect = SC.reference_perm(keys, valids, desc, dicts)
    for cuts in ([0, 3000], [0, 1, 2, 1500, 2999, 3000], list(range(0, 3001, 250)), [0, 0, 3000]):
        ex = SortExecutor(names, desc)
        for lo, hi in zip(cuts, cuts[1:]):
            assert ex.execute([full.slice(lo, hi)], 0, 0) is None
        out = ex.done(0)
        assert np.array_equal(out["rowid"].data.numpy(), expect), cuts
    assert SortExecutor(names, desc).done(0) is None


@pytest.fixture
def qc(monkeypatch):
    cpu_shim.install(monkeypatch)
    from quokka_b200.df import QuokkaContext
    return QuokkaContext()


def test_sort_collect(qc): A.case_sort_collect(qc)
def test_sort_select_filter_keep_order(qc): A.case_sort_select_filter_keep_order(qc)
def test_sort_nulls_from_left_join(qc): A.case_sort_nulls_from_left_join(qc)
def test_sort_then_asof(qc, golden_dir): A.case_sort_then_asof(qc, golden_dir)
def test_sort_then_window(qc, golden_dir): A.case_sort_then_window(qc, golden_dir)
def test_sort_then_pattern(qc, golden_dir): A.case_sort_then_pattern(qc, golden_dir)
def test_sort_then_quantile_and_gram(qc): A.case_sort_then_quantile_and_gram(qc)
def test_sort_ranges(qc): A.case_sort_ranges(qc)
def test_sort_errors(qc): A.case_sort_errors(qc)


def test_explain_prints_the_sort(qc, capsys):
    import pyarrow as pa
    s = qc.from_arrow(pa.table({"a": [3, 1, 2], "b": [1.0, 2.0, 3.0]})).sort(["a", "b"], [True, False])
    s.explain()
    assert "sort a desc, b" in capsys.readouterr().out
    s.explain("physical")
    assert "SortExecutor [ordered]" in capsys.readouterr().out
