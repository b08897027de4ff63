"""Per-event tumbling and session windows without a GPU: the vectorised ranges against the one-row-at-a-time reference on
random inputs, and the API cases through the planner and the executors on the shims."""
import numpy as np
import pytest

import cpu_shim
import window_events_cases as A
import window_events_shim as S
from oracle import relops as R


@pytest.fixture
def qc(monkeypatch):
    cpu_shim.install(monkeypatch)
    from quokka_b200.df import QuokkaContext
    return QuokkaContext()


def _inputs(seed):
    """Heavy ties, keys without rows between keys with rows, negative times, and times near -2^62 and +2^62 in one key."""
    rng = np.random.default_rng(seed)
    n, nk = int(rng.integers(0, 120)), int(rng.integers(1, 7))
    span = int(rng.integers(1, 40))
    time = np.sort(rng.integers(-span, span, n)).astype(np.int64)
    if seed % 4 == 0:
        big = np.int64(2 ** 62)
        time = np.sort(np.where(rng.random(n) < 0.5, -big + rng.integers(0, 30, n), big - rng.integers(0, 30, n))).astype(np.int64)
    by = (rng.integers(0, nk, n) * 2).astype(np.int32)
    return time, by, rng.integers(-64, 64, n) / 4.0


@pytest.mark.parametrize("kind,param", [("tumbling", 1), ("tumbling", 7), ("tumbling", 2 ** 62), ("session", 0), ("session", 3),
                                        ("session", 2 ** 62), ("session", 2 ** 63 - 1)])
def test_ranges_are_the_row_loop(kind, param):
    for seed in range(60):
        time, by, v = _inputs(seed)
        ref = S.running_window(time, by, kind, param, {"s": ("sum", v), "mn": ("min", v), "mx": ("max", v), "n": ("count", None)})
        order, lo, hi = S.running_window_ranges(time, by, kind, param)
        assert np.all(lo <= np.arange(len(order))) and np.all(hi > np.arange(len(order)))
        for name, op in (("s", "sum"), ("mn", "min"), ("mx", "max"), ("n", "count")):
            got = np.empty(len(order))
            got[order] = R.range_aggregate(op, None if op == "count" else S.padded(v[order]), lo, hi)
            assert np.array_equal(got, ref[name]), (seed, name)


def test_session_gap_does_not_overflow():
    """From -2^62 to +2^62 the gap is 2^63, beyond int64; as an unsigned difference it is exact."""
    t = np.array([-2 ** 62, 2 ** 62], dtype=np.int64)
    assert S.run_breaks(t[:1], t[1:], "session", 2 ** 63 - 1)[0]
    assert not S.run_breaks(t[:1], t[1:], "session", 2 ** 63)[0]
    order, lo, hi = S.running_window_ranges(t, np.zeros(2, np.int32), "session", 2 ** 62)
    assert list(lo) == [0, 1] and list(hi) == [1, 2]


def test_shim_matches_the_row_loop():
    """cpu_shim.window_sliding(run=...) against the row loop."""
    import torch
    from quokka_b200 import _lib as L
    for seed in range(30):
        time, by, v = _inputs(seed)
        o = np.lexsort((time, by))
        time, by, v = time[o], by[o], v[o]
        for kind, code, param in (("tumbling", L.WIN_RUN_TUMBLING, 5), ("session", L.WIN_RUN_SESSION, 2)):
            outs = cpu_shim.window_sliding(torch.from_numpy(time), torch.from_numpy(by), None, 0, param, [torch.from_numpy(v)],
                                           [(L.WIN_SUM, 0), (L.WIN_AVG, 0), (L.WIN_COUNT, 0), (L.WIN_MIN, 0), (L.WIN_MAX, 0)], run=code)
            ref = S.running_window(time, by, kind, param, {"s": ("sum", v), "a": ("avg", v), "n": ("count", None), "mn": ("min", v),
                                                           "mx": ("max", v)})
            for got, name in zip(outs, "s a n mn mx".split()):
                np.testing.assert_allclose(got.numpy(), ref[name], rtol=1e-15, atol=0, err_msg=name)


@pytest.mark.parametrize("case", A.API_CASES, ids=lambda f: f.__name__)
def test_window_events_api(qc, case):
    import inspect
    import ranks
    args = {"qc": qc, "golden_dir": ranks.GOLDEN}
    case(*[args[p] for p in inspect.signature(case).parameters])
