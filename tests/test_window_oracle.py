"""The vectorised window references of oracle/relops.py against the per-row ones, and the kernel limits the CPU shim mirrors.
No GPU: the GPU window tests (tests/test_gpu_windows.py) trust the vectorised references, so they are pinned here first."""
import math

import numpy as np
import pytest
import torch

from oracle import relops as R
from quokka_b200 import _lib as L
import cpu_shim


def _case(seed, n, nkeys, span, tmin):
    rng = np.random.default_rng(seed)
    time = np.sort(rng.integers(tmin, tmin + span, n)).astype(np.int64)          # span << n: many ties
    by = rng.integers(0, nkeys, n).astype(np.int32)
    v = rng.integers(-2 ** 24, 2 ** 24, n).astype(np.float64) / 16.0              # exact: multiples of 2^-4
    aggs = {"s": ("sum", v), "mn": ("min", v), "mx": ("max", v), "n": ("count", None), "a": ("avg", v)}
    return time, by, aggs


CASES = [(1, 1, 1, 1, 0), (2, 40, 3, 5, -3), (3, 200, 4, 1000, -500), (4, 300, 7, 40, -10 ** 12), (5, 500, 2, 5000, 10 ** 15),
         (6, 64, 1, 3, -2)]


@pytest.mark.parametrize("seed,n,nkeys,span,tmin", CASES)
@pytest.mark.parametrize("size", [1, 2, 7, 100, 10 ** 6])
def test_sliding_fast_equals_slow(seed, n, nkeys, span, tmin, size):
    time, by, aggs = _case(seed, n, nkeys, span, tmin)
    slow, fast = R.sliding_window(time, by, size, aggs), R.sliding_window_fast(time, by, size, aggs)
    for k in aggs:
        assert np.array_equal(slow[k], fast[k]), k


@pytest.mark.parametrize("seed,n,nkeys,span,tmin", CASES)
@pytest.mark.parametrize("size,hop", [(3, 1), (25, 10), (3000, 1000), (2500, 1000), (300, 1000), (7, 7), (1, 5), (10, 3)])
def test_hopping_fast_equals_slow(seed, n, nkeys, span, tmin, size, hop):
    """size % hop != 0 and hop > size (rows that fall in no window, empty windows skipped) included."""
    time, by, aggs = _case(seed, n, nkeys, span, tmin)
    slow, fast = R.hopping_window(time, by, size, hop, aggs), R.hopping_window_fast(time, by, size, hop, aggs)
    assert len(slow["start"]) == len(fast["start"])
    for k in slow:
        assert np.array_equal(slow[k], fast[k]), k


@pytest.mark.parametrize("seed,n,nkeys,span,tmin", CASES)
@pytest.mark.parametrize("timeout", [0, 1, 5, 10 ** 9])
def test_session_fast_equals_slow(seed, n, nkeys, span, tmin, timeout):
    time, by, aggs = _case(seed, n, nkeys, span, tmin)
    slow, fast = R.session_window(time, by, timeout, aggs), R.session_window_fast(time, by, timeout, aggs)
    assert len(slow["start"]) == len(fast["start"])
    for k in slow:
        assert np.array_equal(slow[k], fast[k]), k


def test_hopping_rows_in_no_window():
    """hop > size: rows between windows belong to none; the key's first window starts at its first time truncated to hop."""
    time = np.array([-7, -6, 0, 2, 3, 9, 10, 14], dtype=np.int64)
    by = np.zeros(len(time), dtype=np.int32)
    out = R.hopping_window_fast(time, by, 2, 5, {"n": ("count", None)})
    assert out["start"].tolist() == [0, 10] and out["n"].tolist() == [1, 1]      # -7, -6, 2, 3, 9 and 14 are in no window
    slow = R.hopping_window(time, by, 2, 5, {"n": ("count", None)})
    assert slow["start"].tolist() == [0, 10] and slow["n"].tolist() == [1, 1]


@pytest.mark.parametrize("nt,nq,nkeys", [(0, 10, 3), (10, 0, 3), (500, 2000, 1), (3000, 1000, 50), (2000, 5000, 700)])
def test_asof_fast_equals_slow(nt, nq, nkeys):
    rng = np.random.default_rng(nt + nq + nkeys)
    lt, rt = np.sort(rng.integers(0, 3000, nt)), np.sort(rng.integers(0, 3000, nq))     # ties on both sides
    lb, rb = rng.integers(0, nkeys, nt), rng.integers(0, nkeys + 2, nq)                # right keys no left row has
    assert np.array_equal(R.asof_backward_fast(lt, lb, rt, rb), R.asof_backward(lt, lb, rt, rb))


def test_range_sum_exact_is_exact():
    rng = np.random.default_rng(7)
    n = 5000
    mag = 10.0 ** rng.uniform(-3, 8, n)
    v = mag * np.where(rng.random(n) < 0.5, -1.0, 1.0)
    lo = rng.integers(0, n, 300)
    hi = np.minimum(lo + rng.integers(1, 2000, 300), n)
    got = R.range_sum_exact(v, lo, hi)
    for a, b, g in zip(lo, hi, got):
        exact = math.fsum(v[a:b])
        assert abs(float(g) - exact) <= 2.0 ** -52 * abs(exact)
    m = R.range_minmax(v, lo, hi, np.minimum)
    assert np.array_equal(m, np.array([v[a:b].min() for a, b in zip(lo, hi)]))


# ------------------------------------------------------------------ the CPU shim refuses what the kernels refuse
def test_shim_merge_cutoff_matches_kernel():
    """qk_asof_merge takes tables of up to 160 KB of int32: 40 960 keys.  Above that the caller falls back to asof_backward."""
    t = torch.zeros(4, dtype=torch.int64)
    b = torch.zeros(4, dtype=torch.int32)
    out, _ = cpu_shim.asof_merge(t, b, t, b, 40_960)
    assert out is not None and out.tolist() == [3, 3, 3, 3]
    assert cpu_shim.asof_merge(t, b, t, b, 40_961) == (None, None)


def test_shim_partition_limits_match_kernel():
    key = torch.arange(10, dtype=torch.int64)
    cpu_shim.partition_plan(key, 16_384, L.PART_MOD)
    with pytest.raises(L.QkError, match="nparts"):
        cpu_shim.partition_plan(key, 16_385, L.PART_MOD)
    dest, offs = cpu_shim.partition_plan(key * 50_000 - 7, 100_000, L.PART_CODE)    # CODE mode: any nparts, codes clamped
    assert offs.numel() == 100_001 and int(offs[-1]) == 10
    assert dest.tolist() == list(range(10))
