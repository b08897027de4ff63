"""The sort kernel (csrc/sort.cu) on the GPU against the exact reference of tests/sort_cases.py -- permutation equality, which
stability makes unique -- and DataStream.sort through the API on the device."""
import ctypes as C

import numpy as np
import pytest
import torch

import ranks
import sort_api_cases as A
import sort_cases as SC

pytestmark = pytest.mark.gpu


def _dev(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _check(key, valid, desc, what):
    from quokka_b200 import ops
    perm, image = ops.sort_perm(_dev(key), _dev(valid), desc, want_image=True)
    assert np.array_equal(perm.cpu().numpy(), SC.reference_perm([key], [valid], [desc])), what
    got, exp = image.cpu().numpy().view(np.uint64), SC.sorted_image(key, valid, desc)
    if key.dtype.itemsize == 8:
        assert np.array_equal(got, exp), what
    else:       # a narrow key sits in the image's top bytes: other bits than the host image's, the same order and the same ties
        nv = len(key) if valid is None else int(valid.sum())           # valid rows first; every NULL row holds 0 (~0 when descending)
        assert np.array_equal(np.unique(got[:nv], return_inverse=True)[1], np.unique(exp[:nv], return_inverse=True)[1]), what
        assert np.array_equal(got[nv:], exp[nv:]), what


@pytest.mark.parametrize("n", SC.SIZES + SC.CHUNK_SIZES[1:2])
def test_every_generator_bit_for_bit(n):
    for name, key in SC.key_cases(n):
        for vname, valid in SC.valid_cases(n):
            for desc in (False, True):
                _check(key, valid, desc, (n, name, vname, desc))


@pytest.mark.parametrize("n", [1_000_003, SC.CHUNK_SIZES[0], SC.CHUNK_SIZES[2]])
def test_large_inputs(n):
    cases = dict(SC.key_cases(n))
    valid = SC.valid_cases(n)[1][1]
    for name, v, desc in (("int64-full-range", None, False), ("float64-special", valid, True), ("int32-dates", None, False),
                          ("float32-random", valid, False), ("uint8-full-range", None, True), ("int64-two-values", None, False)):
        _check(cases[name], v, desc, (n, name, desc))


def test_forty_million_rows():
    n = 40_000_003
    rng = np.random.default_rng(40)
    _check(rng.integers(-(1 << 62), 1 << 62, n, dtype=np.int64), None, False, "int64")
    _check(rng.integers(8035, 10561, n).astype(np.int32), None, True, "dates desc")


@pytest.mark.parametrize("ncols", [1, 2, 3, 4])
def test_perm_in_chaining(ncols):
    from quokka_b200 import ops
    for n in (33, 5000, 70_001):
        for seed in (0, 1):
            keys, valids, desc, _ = SC.multi_column_case(n, ncols, seed)
            perm = None
            for k, v, d in list(zip(keys, valids, desc))[::-1]:
                perm = ops.sort_perm(_dev(k), _dev(v), d, perm)
            assert np.array_equal(perm.cpu().numpy(), SC.reference_perm(keys, valids, desc)), (n, ncols, seed)


def test_table_sort_with_strings():
    from quokka_b200.columns import DeviceTable
    from quokka_b200.executors import sort_perm_table
    keys, valids, desc, dicts = SC.multi_column_case(20_000, 4, 1)
    t = DeviceTable.from_numpy({f"c{i}": k for i, k in enumerate(keys)}, dictionaries={"c2": dicts[2]})
    t.columns["c1"].valid = _dev(valids[1])
    perm = sort_perm_table(t, ["c0", "c1", "c2", "c3"], desc)
    assert np.array_equal(perm.cpu().numpy(), SC.reference_perm(keys, valids, desc, dicts))


def test_sliced_and_misaligned_views():
    from quokka_b200 import ops
    rng = np.random.default_rng(5)
    for dt in SC.DTYPES:
        base = (rng.standard_normal(10_007) * 100).astype(dt)
        for off in (1, 3, 5):
            key = base[off:off + 9001]
            got = ops.sort_perm(_dev(base)[off:off + 9001], None, False)
            assert np.array_equal(got.cpu().numpy(), SC.reference_perm([key], [None], [False])), (dt, off)


def test_last_plan_reports_skipped_passes():
    from quokka_b200 import ops
    rng = np.random.default_rng(6)
    n = 300_000
    ops.sort_perm(_dev(rng.integers(8035, 10561, n).astype(np.int32)), None, False)
    assert ops.sort_last_plan() == "d8 passes=2/8 nulls=0"
    ops.sort_perm(_dev(rng.integers(-(1 << 63), (1 << 63) - 1, n, dtype=np.int64)), None, False)
    assert ops.sort_last_plan() == "d8 passes=8/8 nulls=0"
    ops.sort_perm(_dev(rng.integers(0, 200, n).astype(np.int64)), _dev((rng.random(n) < 0.5).astype(np.uint8)), True)
    assert ops.sort_last_plan() == "d8 passes=1/8 nulls=1"
    ops.sort_perm(_dev(np.full(n, 3.5)), _dev(np.ones(n, np.uint8)), False)
    assert ops.sort_last_plan() == "d8 passes=0/8 nulls=0"


def test_two_runs_are_identical():
    from quokka_b200 import ops
    rng = np.random.default_rng(7)
    key, valid = _dev(rng.integers(0, 1000, 2_000_003).astype(np.int64)), _dev((rng.random(2_000_003) < 0.9).astype(np.uint8))
    a, ia = ops.sort_perm(key, valid, True, want_image=True)
    b, ib = ops.sort_perm(key, valid, True, want_image=True)
    assert torch.equal(a, b) and torch.equal(ia, ib)


def test_argument_errors():
    from quokka_b200 import _lib as L, ops
    lib = L.lib()
    key = torch.arange(100, dtype=torch.int64, device="cuda")
    out = torch.empty(100, dtype=torch.int32, device="cuda")
    ws = torch.empty(lib.qk_sort_workspace_bytes(100), dtype=torch.uint8, device="cuda")
    kc = ops.col(key)
    args = lambda **kw: (C.byref(kw.get("key", kc)), None, 0, None, kw.get("out", out.data_ptr()), None, kw.get("n", 100),
                         kw.get("ws", ws.data_ptr()), kw.get("ws_bytes", ws.numel()), None)
    assert lib.qk_sort_perm(*args(ws_bytes=64)) == L.ERR_CAPACITY and b"workspace" in lib.qk_last_error()
    assert lib.qk_sort_perm(*args(ws=None)) == L.ERR_CAPACITY
    assert lib.qk_sort_perm(*args(out=None)) == L.ERR_INVALID
    assert lib.qk_sort_perm(*args(n=99)) == L.ERR_INVALID
    assert lib.qk_sort_perm(None, None, 0, None, out.data_ptr(), None, 100, ws.data_ptr(), ws.numel(), None) == L.ERR_INVALID
    assert lib.qk_sort_perm(*args(n=1 << 31)) == L.ERR_UNSUPPORTED
    bad = L.qk_column(key.data_ptr(), None, 100, 99, 0)
    assert lib.qk_sort_perm(*args(key=bad)) == L.ERR_INVALID and b"dtype" in lib.qk_last_error()
    vec = L.qk_column(key.data_ptr(), None, 100, L.QK_F32, 2)
    assert lib.qk_sort_perm(*args(key=vec)) == L.ERR_UNSUPPORTED
    empty = L.qk_column(None, None, 0, L.QK_I64, 0)
    assert lib.qk_sort_perm(*args(key=empty, n=0, out=None, ws=None, ws_bytes=0)) == 0
    assert lib.qk_sort_workspace_bytes(-1) == 0
    torch.cuda.synchronize()


@pytest.fixture
def qc():
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


def test_sort_two_ranks_nccl():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    ranks.nccl_suites("sort")
