"""Per-event tumbling and session windows on the device: qk_window_running (csrc/window.cu) through the C ABI against the
vectorised reference (window_events_shim.running_window_ranges) with the value columns and error bounds of
tests/test_gpu_windows.py, the linear-work case, determinism, argument checks, and the API cases on one GPU and on in-process
ranks.

The kernel works in tiles of 2048 rows and its carry scan in chunks of 1024 tiles, so the sizes straddle both."""
import ctypes as C
import types

import numpy as np
import pytest
import torch

import inproc_link as IL
import ranks
import window_events_cases as A
import window_events_shim as S
from test_gpu_windows import _win_specs, check_agg, dev, draw_keys, draw_times, exact_col, general_col, host, segmented

pytestmark = pytest.mark.gpu

TILE, CHUNK = 2048, 2048 * 1024


@pytest.fixture(scope="module")
def qb():
    from quokka_b200 import _lib, ops
    _lib.lib()
    return types.SimpleNamespace(L=_lib, ops=ops)


def _times(rng, n, nkeys, kind):
    if kind == "distinct":                                # strictly increasing: with timeout 0 every row is its own session
        return (np.arange(n, dtype=np.int64) * 3 - n).astype(np.int64)
    return draw_times(rng, n, nkeys, kind)


def _inputs(n, nkeys, tkind, seed):
    rng = np.random.default_rng(seed)
    time, by = _times(rng, n, nkeys, tkind), draw_keys(rng, n, nkeys)
    order, seg = segmented(time, by, nkeys)
    vals = [(exact_col if c % 2 == 0 else general_col)(rng, n) for c in range(8)]
    return time[order], by[order], seg, vals


def _code(qb, kind):
    return qb.L.WIN_RUN_TUMBLING if kind == "tumbling" else qb.L.WIN_RUN_SESSION


@pytest.mark.parametrize("n,nkeys,tkind,kind,param", [
    (0, 1, "neg", "tumbling", 10), (1, 1, "tiny", "session", 0),
    (TILE - 1, 3, "tiny", "tumbling", 3), (TILE, 3, "neg", "session", 5), (TILE + 1, 1, "huge", "session", 2 ** 62),
    (CHUNK - 1, 8000, "tiny", "tumbling", 2), (CHUNK, 3, "neg", "session", 0), (CHUNK + 1, 1, "neg", "tumbling", 10 ** 12),
    (100_003, 1, "distinct", "session", 0), (100_003, 8000, "huge", "tumbling", 2 ** 61),
    (5_000_003, 8000, "neg", "session", 40), (5_000_003, 3, "tiny", "tumbling", 7)])
def test_window_running_kernel(qb, n, nkeys, tkind, kind, param):
    """16 outputs over 8 columns against the ranges: heavy ties, keys without rows, one run across every tile (size 10^12 over
    one key), every row its own run (distinct times, timeout 0), gaps of 2^63 between -2^62 and +2^62 (timeout 2^62)."""
    ts, bs, seg, vals = _inputs(n, nkeys, tkind, n + nkeys + len(kind))
    names, specs = _win_specs(qb)
    outs = qb.ops.window_sliding(dev(ts), dev(bs), dev(seg), nkeys, param, [dev(v) for v in vals], specs, run=_code(qb, kind))
    ro, lo, hi = S.running_window_ranges(ts, bs, kind, param)
    assert np.array_equal(ro, np.arange(n))                          # the inputs are already in the reference's order
    for (op, src), o in zip(names, outs):
        check_agg(op, host(o), S.padded(vals[src]), src % 2 == 0, lo, hi, (op, src))


def _timed(fn, reps=5):
    fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def test_one_time_ten_million_rows(qb):
    """One key, 10 M rows at one time: every row gets the whole column's aggregate, at about the cost of 10 M distinct times
    (one peer-end search per tile, not a walk per row)."""
    L, ops = qb.L, qb.ops
    n = 10_000_000
    rng = np.random.default_rng(10)
    ve, vg = exact_col(rng, n), general_col(rng, n)
    by, seg = torch.zeros(n, dtype=torch.int32, device="cuda"), dev(np.array([0, n], np.int64))
    specs = [(L.WIN_SUM, 0), (L.WIN_MIN, 0), (L.WIN_MAX, 1), (L.WIN_COUNT, 0), (L.WIN_AVG, 0), (L.WIN_SUM, 1)]
    dv = [dev(ve), dev(vg)]
    same = torch.zeros(n, dtype=torch.int64, device="cuda")
    outs = [host(o) for o in ops.window_sliding(same, by, seg, 1, 0, dv, specs, run=L.WIN_RUN_SESSION)]
    exp_sum = float(np.sum(ve))                                          # exact: every partial sum of the column is
    assert np.all(outs[0] == exp_sum) and np.all(outs[1] == ve.min()) and np.all(outs[2] == vg.max())
    assert np.all(outs[3] == n) and np.all(outs[4] == exp_sum / n)
    assert np.all(outs[5].view(np.int64) == outs[5][0].view(np.int64))
    exact = S.R.range_sum_exact(vg, np.array([0]), np.array([n]))[0]
    assert abs(np.longdouble(outs[5][0]) - exact) <= (n - 1) * np.longdouble(2.0 ** -53) * np.sum(np.abs(vg), dtype=np.longdouble)
    distinct = torch.arange(n, dtype=torch.int64, device="cuda")
    t_same = _timed(lambda: ops.window_sliding(same, by, seg, 1, 0, dv, specs, run=L.WIN_RUN_SESSION))
    t_distinct = _timed(lambda: ops.window_sliding(distinct, by, seg, 1, 0, dv, specs, run=L.WIN_RUN_SESSION))
    print(f"10 M rows: one time {t_same:.3f} ms, distinct times {t_distinct:.3f} ms")
    assert t_same < 4 * t_distinct, (t_same, t_distinct)


def test_window_running_is_deterministic(qb):
    ts, bs, seg, vals = _inputs(CHUNK + 4097, 8000, "tiny", 77)
    names, specs = _win_specs(qb)
    args = (dev(ts), dev(bs), dev(seg), 8000, 3, [dev(v) for v in vals], specs)
    a = [host(o) for o in qb.ops.window_sliding(*args, run=qb.L.WIN_RUN_SESSION)]
    b = [host(o) for o in qb.ops.window_sliding(*args, run=qb.L.WIN_RUN_SESSION)]
    for x, y in zip(a, b):
        assert np.array_equal(x.view(np.int64), y.view(np.int64))


def test_window_running_bad_arguments(qb):
    L, ops = qb.L, qb.ops
    n = 100
    t, b = torch.arange(n, dtype=torch.int64, device="cuda"), torch.zeros(n, dtype=torch.int32, device="cuda")
    seg, v = dev(np.array([0, n], np.int64)), torch.ones(n, dtype=torch.float64, device="cuda")
    ok = dict(run=L.WIN_RUN_TUMBLING, size=10, vals=[v], aggs=[(L.WIN_SUM, 0)])
    ops.window_sliding(t, b, seg, 1, **ok)
    for bad in (dict(size=0), dict(run=L.WIN_RUN_SESSION, size=-1), dict(run=3), dict(aggs=[(6, 0)]), dict(aggs=[(L.WIN_MIN, 1)]),
                dict(vals=[v.float()]), dict(vals=[v[:-1]]), dict(aggs=[(L.WIN_COUNT, 0)] * 17)):
        with pytest.raises(L.QkError):
            ops.window_sliding(t, b, seg, 1, **{**ok, **bad})
    with pytest.raises(L.QkError):
        ops.window_sliding(t, b.to(torch.int64), seg, 1, **ok)
    # a workspace one byte short
    need = L.lib().qk_window_running_workspace_bytes(n)
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    out = torch.empty(n, dtype=torch.float64, device="cuda")
    one = (C.c_int32 * 1)
    rc = L.lib().qk_window_running(C.byref(ops.col(t)), C.byref(ops.col(b)), seg.data_ptr(), 1, L.WIN_RUN_TUMBLING, 10, ops.cols([v]), 1,
                                   one(L.WIN_SUM), one(0), 1, ops.cols([out]), ws.data_ptr(), need - 1, 0)
    assert rc == L.ERR_CAPACITY


@pytest.mark.parametrize("case", A.API_CASES, ids=lambda f: f.__name__)
def test_window_events_api_on_device(case):
    import inspect
    from quokka_b200.df import QuokkaContext
    args = {"qc": QuokkaContext(), "golden_dir": ranks.GOLDEN}
    case(*[args[p] for p in inspect.signature(case).parameters])


@pytest.mark.parametrize("world", [2, 3])
def test_window_events_on_inproc_ranks(world):
    counts = IL.run_program_ranks(world, A.SUITE, "cuda", 64 << 20)
    print(f"world {world}: {dict(sorted(counts.items()))}")
