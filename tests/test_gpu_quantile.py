"""qk_qsketch_update / qk_qsketch_merge (csrc/quantile.cu) and DataStream.approximate_quantile on the real sm_90a kernels.

The sketch is exact bookkeeping (counts, min and max images per bucket), so the kernel's compacted entries must equal
tests/quantile_cases.py's numpy sketch as a set, bit for bit, whatever the dtype, length, alignment, mask or growth path."""
import numpy as np
import pytest
import torch

import quantile_cases as QC

pytestmark = pytest.mark.gpu


def _entries(sk):
    k, c, lo, hi = (t.cpu().numpy().view(np.uint64) for t in sk.entries())
    o = np.argsort(k)
    return k[o], c[o], lo[o], hi[o]


def _assert_same(sk, ref, what=""):
    got = _entries(sk)
    assert len(got[0]) == len(ref[0]), f"{what}: {len(got[0])} entries, expected {len(ref[0])}"
    for name, a, b in zip(("key", "count", "min", "max"), got, ref):
        assert np.array_equal(a, b), f"{what}: {name} differs"


def _device(cols, misalign=False):
    out = []
    for x in cols:
        t = torch.from_numpy(np.concatenate([x[:1], x]) if misalign and len(x) else x.copy()).cuda()
        out.append(t[1:] if misalign and len(x) else t)
    return out


@pytest.mark.parametrize("n", [0, 1, 31, 33, 4097, 100_003, 5_000_011])
def test_entries_equal_numpy_sketch_all_dtypes(n):
    from quokka_b200 import ops
    cols = list(QC.special_columns(n, n + 1).values()) if n else [np.zeros(0, dt) for dt in (np.float64, np.float32, np.int64, np.int32, np.uint8)]
    sk = ops.QuantileSketch(len(cols), "cuda")
    sk.update(_device(cols))
    torch.cuda.synchronize()
    ref = QC.sketch_entries(cols)
    _assert_same(sk, ref, f"n={n}")
    qs = [0.0, 0.1, 0.5, 0.9, 1.0]
    got, valid = sk.quantiles(qs)
    want, wvalid = QC.sketch_quantiles(ref, len(cols), qs)
    assert np.array_equal(valid.cpu().numpy(), wvalid)
    assert np.array_equal(got.cpu().numpy()[wvalid].view(np.uint64), want[wvalid].view(np.uint64))


@pytest.mark.parametrize("n", [4097, 100_003])
def test_misaligned_views_and_masks(n):
    """Column views that start one element into their buffer (never 16-byte aligned), and per-column row masks."""
    from quokka_b200 import ops
    cols = list(QC.special_columns(n, 3).values())
    dev = _device(cols, misalign=True)
    assert all(t.data_ptr() % 16 for t in dev if t.element_size() > 1)
    sk = ops.QuantileSketch(len(cols), "cuda")
    sk.update(dev)
    _assert_same(sk, QC.sketch_entries(cols), "misaligned")
    rng = np.random.default_rng(n)
    masks = [rng.random(n) < 0.3, None, np.ones(n, bool), np.zeros(n, bool), rng.random(n) < 0.9]
    sk = ops.QuantileSketch(len(cols), "cuda")
    sk.update(_device(cols), [None if m is None else torch.from_numpy(m.astype(np.uint8)).cuda() for m in masks])
    _assert_same(sk, QC.sketch_entries(cols, masks), "masked")
    _, valid = sk.quantiles([0.5])
    assert valid.cpu().numpy().tolist() == [[True, True, True, False, True]]


def test_forced_growth_path_counts_every_tile_once():
    """Start at the minimum capacity with millions of distinct buckets: the kernel defers tiles, the host grows the table
    several times and re-runs exactly the deferred tiles.  The result still equals the numpy sketch."""
    from quokka_b200 import ops
    rng = np.random.default_rng(99)
    n = 3_000_017
    cols = [rng.lognormal(0, s, n) * rng.choice([-1.0, 1.0], n) for s in (60, 50, 40)]
    cols.append(rng.uniform(-1e300, 1e300, n) * 10.0 ** -rng.integers(0, 600, n))
    ref = QC.sketch_entries(cols)
    assert len(ref[0]) > 2_500_000
    sk = ops.QuantileSketch(4, "cuda", capacity=ops.QSKETCH_MIN_CAPACITY)
    assert sk.capacity == ops.QSKETCH_MIN_CAPACITY
    sk.update(_device(cols))
    assert sk.rounds >= 2 and sk.grows >= 2, (sk.rounds, sk.grows)
    assert int(sk.ctrl[0]) == len(ref[0]) and 2 * len(ref[0]) <= sk.capacity
    _assert_same(sk, ref, "grown")
    half = n // 2                                          # a second batch into the grown table, then a merged copy
    sk2 = ops.QuantileSketch(4, "cuda", capacity=ops.QSKETCH_MIN_CAPACITY)
    dev = _device(cols)
    sk2.update([t[:half] for t in dev])
    sk2.update([t[half:] for t in dev])
    _assert_same(sk2, ref, "two batches")
    sk3 = ops.QuantileSketch(4, "cuda", capacity=ops.QSKETCH_MIN_CAPACITY)
    sk3.merge(*sk.entries())
    sk3.merge(*ops.QuantileSketch(4, "cuda").entries())
    _assert_same(sk3, ref, "merged")


def test_deterministic_and_split_invariant():
    from quokka_b200 import ops
    cols = list(QC.special_columns(1_000_003, 11).values())
    dev = _device(cols)
    runs = []
    for cuts in ((0, len(cols[0])), (0, 2048, 2049, 500_000, len(cols[0]))):
        sk = ops.QuantileSketch(len(cols), "cuda")
        for lo, hi in zip(cuts[:-1], cuts[1:]):
            sk.update([t[lo:hi] for t in dev])
        runs.append(sk.quantiles([0.0, 0.05, 0.5, 0.95, 1.0])[0].cpu().numpy())
        _assert_same(sk, QC.sketch_entries(cols), f"cuts {cuts}")
    sk = ops.QuantileSketch(len(cols), "cuda")
    sk.update(dev)
    runs.append(sk.quantiles([0.0, 0.05, 0.5, 0.95, 1.0])[0].cpu().numpy())
    assert all(np.array_equal(r.view(np.uint64), runs[0].view(np.uint64)) for r in runs)


@pytest.fixture
def qc():
    from quokka_b200.df import QuokkaContext
    return QuokkaContext()


def test_quantile_lineitem(qc): QC.case_quantile_lineitem(qc)
def test_quantile_tpch_606(qc): QC.case_quantile_tpch_606(qc)
def test_quantile_ragged_batches(qc): QC.case_quantile_ragged_batches(qc)
def test_quantile_left_join_nulls(qc): QC.case_quantile_left_join_nulls(qc)
def test_quantile_empty(qc): QC.case_quantile_empty(qc)
def test_quantile_rejects(qc): QC.case_quantile_rejects(qc)
def test_quantile_winsorised_covariance(qc): QC.case_quantile_winsorised_covariance(qc)
