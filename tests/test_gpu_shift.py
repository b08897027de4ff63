"""The shift kernels (csrc/shift.cu) on the GPU against the numpy stand-ins of tests/shift_shim.py, bit for bit -- source rows,
edge flags, order-check counts, every dtype with and without validity, both gather sources, up to 2^24 + 3 rows -- and
OrderedStream.shift through the API on the device."""
import ctypes as C

import numpy as np
import pytest
import torch

import ranks
import shift_api_cases as A
import shift_cases as SC
import shift_shim
from quokka_b200 import _lib as L

pytestmark = pytest.mark.gpu


def _dev(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _both(keys, n, nrows, lo=0, hi=None, time=None):
    """(device answer, shim answer) of shift_plan with edge flags, on the device's partition (checked against the shim's)."""
    from quokka_b200 import ops
    import cpu_shim
    hi = nrows if hi is None else hi
    t = None if time is None else torch.from_numpy(time)
    if keys is None:
        got = ops.shift_plan(n, nrows, lo=lo, hi=hi, want_edge=True, time=None if t is None else t.cuda(), device=torch.device("cuda"))
        exp = shift_shim.shift_plan(n, nrows, lo=lo, hi=hi, want_edge=True, time=t)
        return got, exp
    n_by = int(keys.max()) + 1 if len(keys) else 1
    codes = _dev(keys)
    dest, seg = ops.partition_plan(codes, n_by, L.PART_CODE)
    hdest, hseg = cpu_shim.partition_plan(torch.from_numpy(keys), n_by, L.PART_CODE)
    assert torch.equal(dest.cpu(), hdest) and torch.equal(seg.cpu(), hseg)
    got = ops.shift_plan(n, nrows, codes, n_by, dest, seg, lo=lo, hi=hi, want_edge=True, time=None if t is None else t.cuda())
    exp = shift_shim.shift_plan(n, nrows, torch.from_numpy(keys), n_by, hdest, hseg, lo=lo, hi=hi, want_edge=True, time=t)
    return got, exp


def _same(got, exp, what):
    assert torch.equal(got[0].cpu(), exp[0]), what
    assert torch.equal(got[1].cpu(), exp[1]), what
    assert got[2] == exp[2], what


@pytest.mark.parametrize("nrows", SC.SIZES)
def test_plan_every_case_bit_for_bit(nrows):
    rng = np.random.default_rng(nrows)
    time = np.sort(rng.integers(0, 1000, nrows)).astype(np.int64)
    time[rng.random(nrows) < 0.01] = -1                                        # a few rows out of order
    for name, keys in SC.key_cases(nrows):
        for n in SC.n_cases(nrows):
            _same(*_both(keys, n, nrows, time=time), (nrows, name, n))
            if keys is not None:
                assert np.array_equal(_both(keys, n, nrows)[0][0].cpu().numpy().astype(np.int64), SC.reference_src(keys, n, nrows))
        lo = nrows // 3
        for n in (1, -2):
            _same(*_both(keys, n, nrows, lo=lo, hi=nrows), (nrows, name, n, "lo"))
            _same(*_both(keys, n, nrows, lo=0, hi=nrows - lo), (nrows, name, n, "hi"))


@pytest.mark.parametrize("nrows", [(1 << 24) + 3])
def test_plan_large(nrows):
    rng = np.random.default_rng(24)
    keys = rng.integers(0, 8000, nrows).astype(np.int32)
    time = np.arange(nrows, dtype=np.int64)
    for n in (1, -1, 5):
        _same(*_both(keys, n, nrows, time=time), n)
    _same(*_both(None, 3, nrows, lo=17, hi=nrows), "no key")


def _gather_case(nrows, nb, seed, with_valid):
    rng = np.random.default_rng(seed)
    vals = SC.value_cases(nrows + nb, seed)
    names = list(vals)
    a = [_dev(vals[c][0][:nrows]) for c in names]
    b = [_dev(vals[c][0][nrows:]) for c in names]
    av = [_dev(vals[c][1][:nrows]) if with_valid and vals[c][1] is not None else None for c in names]
    bv = [_dev(vals[c][1][nrows:]) if with_valid and vals[c][1] is not None else None for c in names]
    fills = [SC.FILLS[c] if i % 2 == 0 else None for i, c in enumerate(names)]
    src = rng.integers(-1, nrows + nb, nrows).astype(np.int32)
    return a, b, av, bv, fills, _dev(src)


@pytest.mark.parametrize("nrows", [1, 1000, 65_537, (1 << 24) + 1])
@pytest.mark.parametrize("with_valid", [False, True])
def test_gather_every_dtype_bit_for_bit(nrows, with_valid):
    from quokka_b200 import ops
    for nb in (0, 5, 3000):
        a, b, av, bv, fills, src = _gather_case(nrows, nb, nrows + nb, with_valid)
        if nb == 0:
            src = torch.where(src >= nrows, torch.full_like(src, -1), src)
        got = ops.shift_gather(a, b if nb else None, src, fills, av, bv)
        cpu = lambda xs: None if xs is None else [None if x is None else x.cpu() for x in xs]
        exp = shift_shim.shift_gather(cpu(a), cpu(b) if nb else None, src.cpu(), fills, cpu(av), cpu(bv))
        for c in range(len(a)):
            assert torch.equal(got[0][c].cpu().view(torch.uint8), exp[0][c].view(torch.uint8)), (nrows, nb, c)
            assert (got[1][c] is None) == (exp[1][c] is None), (nrows, nb, c)
            if got[1][c] is not None:
                assert torch.equal(got[1][c].cpu(), exp[1][c]), (nrows, nb, c)


def test_gather_more_columns_than_one_launch_takes():
    from quokka_b200 import ops
    n = 5000
    rng = np.random.default_rng(3)
    a = [_dev(rng.integers(0, 1 << 40, n)) for _ in range(L.MAX_COLS + 3)]
    src = _dev(rng.integers(-1, n, n).astype(np.int32))
    outs, valid = ops.shift_gather(a, None, src, [9] * len(a))
    s = src.long()
    for x, o in zip(a, outs):
        assert torch.equal(o, torch.where(s >= 0, x[s.clamp(min=0)], torch.full_like(x, 9)))
    assert all(v is None for v in valid)


def test_argument_errors():
    from quokka_b200 import ops
    lib = L.lib()
    n = 100
    codes = torch.zeros(n, dtype=torch.int32, device="cuda")
    dest, seg = ops.partition_plan(codes, 1, L.PART_CODE)
    src = torch.empty(n, dtype=torch.int32, device="cuda")
    ws = torch.empty(lib.qk_shift_workspace_bytes(n), dtype=torch.uint8, device="cuda")
    status = torch.zeros(1, dtype=torch.int64, device="cuda")
    t = torch.zeros(n, dtype=torch.int64, device="cuda")

    def plan(**kw):
        return lib.qk_shift_plan(kw.get("by", codes.data_ptr()), 1, kw.get("dest", dest.data_ptr()), seg.data_ptr(), kw.get("n", n), 1,
                                 kw.get("lo", 0), kw.get("hi", n), kw.get("src", src.data_ptr()), None, kw.get("time", None),
                                 kw.get("status", None), kw.get("ws", ws.data_ptr()), kw.get("ws_bytes", ws.numel()), None)
    assert plan() == 0
    assert plan(ws_bytes=16) == L.ERR_CAPACITY and b"workspace" in lib.qk_last_error()
    assert plan(dest=None) == L.ERR_INVALID
    assert plan(hi=n + 1) == L.ERR_INVALID and plan(lo=5, hi=4) == L.ERR_INVALID
    assert plan(src=None) == L.ERR_INVALID
    assert plan(time=t.data_ptr()) == L.ERR_INVALID and plan(time=t.data_ptr(), status=status.data_ptr()) == 0
    assert plan(n=1 << 31) == L.ERR_UNSUPPORTED
    assert lib.qk_shift_plan(None, 0, None, None, 0, 1, 0, 0, None, None, None, None, None, 0, None) == 0
    assert lib.qk_shift_workspace_bytes(-1) == 0
    vec = torch.zeros(n, 2, device="cuda")
    with pytest.raises(L.QkError, match="vector"):
        ops.shift_gather([vec], None, src, [None])
    with pytest.raises(L.QkError, match="dtype"):
        ops.shift_gather([t], [torch.zeros(3, dtype=torch.int32, device="cuda")], src, [None])
    torch.cuda.synchronize()


@pytest.fixture
def qc():
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


def test_shift_two_ranks_nccl():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    ranks.nccl_suites("shift")
