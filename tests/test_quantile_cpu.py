"""DataStream.approximate_quantile / approximate_median without a GPU: the planner and the executors on tests/cpu_shim.py +
tests/quantile_shim.py, the answer step (ops.qsketch_quantiles) against the numpy restatement, and the argument checks of
qk_qsketch_update / qk_qsketch_merge."""
import ctypes as C

import numpy as np
import pytest
import torch

import quantile_cases as QC
import quantile_shim


@pytest.fixture
def qc(monkeypatch):
    quantile_shim.install(monkeypatch)
    from quokka_b200.df import QuokkaContext
    return QuokkaContext()


def test_quantile_lineitem(qc): QC.case_quantile_lineitem(qc)
def test_quantile_tpch_606(qc): QC.case_quantile_tpch_606(qc)
def test_quantile_ragged_batches(qc): QC.case_quantile_ragged_batches(qc)
def test_quantile_left_join_nulls(qc): QC.case_quantile_left_join_nulls(qc)
def test_quantile_empty(qc): QC.case_quantile_empty(qc)
def test_quantile_rejects(qc): QC.case_quantile_rejects(qc)
def test_quantile_winsorised_covariance(qc): QC.case_quantile_winsorised_covariance(qc)


def test_quantile_plan_shape(qc):
    """Per-rank partial on PassThrough + CustomChannels(1), final on Broadcast + a single channel, both silent until done()."""
    from quokka_b200.executors import QuantileFinalExecutor, QuantilePartialExecutor
    import api_cases as A
    s = qc.from_arrow(A.tables()[0]).approximate_quantile(QC.QUANT_COLS, [0.1, 0.9])
    fin = s.node
    part = fin.parents[0]
    assert isinstance(fin.executor, QuantileFinalExecutor) and isinstance(part.executor, QuantilePartialExecutor)
    assert type(fin.partitioners[0]).__name__ == "BroadcastPartitioner" and type(fin.placement).__name__ == "SingleChannelStrategy"
    assert type(part.partitioners[0]).__name__ == "PassThroughPartitioner" and type(part.placement).__name__ == "CustomChannelsStrategy"
    assert fin.executor.silent_streams == "all" and part.executor.silent_streams == "all"
    assert s.schema == QC.QUANT_COLS
    assert qc.from_arrow(A.tables()[0]).approximate_median(["l_tax"]).node.executor.quantiles == [0.5]


def test_answer_step_matches_the_numpy_restatement():
    """ops.qsketch_quantiles (torch, the product's answer step) == sketch_quantiles (numpy, one bucket at a time), bit for
    bit, on entries of every dtype and special value, in shuffled order; and the rank rule is round half away from zero."""
    from quokka_b200 import ops
    cols = QC.special_columns(20_011, 5)
    xs = list(cols.values()) + [np.zeros(0)]                      # an empty column: NULL
    e = QC.sketch_entries(xs)
    perm = np.random.default_rng(1).permutation(len(e[0]))
    qs = [0.0, 1e-9, 0.1, 0.25, 0.5, 0.5 + 1e-12, 0.9, 0.999999, 1.0]
    got, valid = ops.qsketch_quantiles(*(torch.from_numpy(a[perm].view(np.int64).copy()) for a in e), len(xs), qs)
    ref, rvalid = QC.sketch_quantiles(e, len(xs), qs)
    assert np.array_equal(valid.numpy(), rvalid) and not rvalid[:, -1].any()
    assert np.array_equal(got.numpy()[rvalid].view(np.uint64), ref[rvalid].view(np.uint64))
    for j, x in enumerate(xs[:-1]):
        for i, q in enumerate(qs):
            QC.check_guarantee(ref[i, j], x, q, f"column {j}")
    assert [QC.round_half_away(v) for v in (0.5, 1.5, 2.5, 2.4999999999999996, 0.49999999999999994)] == [1, 2, 3, 2, 0]
    assert QC.quantile_nearest(np.array([3.0, 1.0, np.nan, 2.0]), 1.0) != QC.quantile_nearest(np.array([3.0, 1.0, 2.0]), 1.0)


def test_bucket_rule_guarantee_on_split_and_merged_inputs():
    """The numpy sketch of a split input, merged, equals the sketch of the whole; its answers meet the guarantee on normal,
    price-like and mixed +-0 / +-inf / log-normal data."""
    rng = np.random.default_rng(23)
    n = 50_000
    datasets = [rng.normal(3.0, 2.0, n), np.round(rng.uniform(900, 105_000, n), 2),
                np.concatenate([rng.lognormal(0, 30, n // 2) * rng.choice([-1, 1], n // 2), np.repeat([0.0, -0.0, np.inf, -np.inf], 50)])]
    for x in datasets:
        whole = QC.sketch_entries([x])
        sh = quantile_shim.QuantileSketch(1, None)
        for lo, hi in ((0, 7), (7, 7), (7, n // 3), (n // 3, len(x))):
            sh.update([torch.from_numpy(x[lo:hi].copy())])
        merged = tuple(t.numpy().view(np.uint64) for t in sh.entries())
        assert all(np.array_equal(a, b) for a, b in zip(whole, merged))
        qs = list(np.linspace(0, 1, 41))
        ref, _ = QC.sketch_quantiles(whole, 1, qs)
        for i, q in enumerate(qs):
            QC.check_guarantee(ref[i, 0], x, q)


def test_qsketch_argument_errors_are_reported_without_a_gpu():
    from quokka_b200 import _lib as L
    lib = L.lib()
    ws = (C.c_uint8 * 256)()
    buf = (C.c_double * 8)()
    p = C.cast(buf, C.c_void_p)
    tab = C.cast((C.c_uint64 * 16)(), C.c_void_p)
    ctrl = C.cast((C.c_uint64 * 4)(), C.c_void_p)
    dfr = C.cast((C.c_int32 * 4)(), C.c_void_p)

    def cols(*specs):
        arr = (L.qk_column * len(specs))()
        for i, (data, valid, length, dt) in enumerate(specs):
            arr[i] = L.qk_column(data, valid, length, dt, 0)
        return arr

    ok = cols((p, None, 8, L.QK_F64), (p, None, 8, L.QK_I32))

    def upd(c, k=2, n=8, cap=4096, table=tab, tiles=None, ntiles=2, wsb=256):
        return lib.qk_qsketch_update(c, None, k, n, table, cap, ctrl, tiles, ntiles, dfr, ws, wsb, None)

    assert upd(ok, k=0) == L.ERR_INVALID and b"k must be" in lib.qk_last_error()
    assert upd(cols((None, None, 8, L.QK_F64), (p, None, 8, L.QK_F64))) == L.ERR_INVALID
    assert b"null data" in lib.qk_last_error()
    assert upd(cols((p, None, 8, L.QK_F64), (p, None, 7, L.QK_F64))) == L.ERR_INVALID and b"rows" in lib.qk_last_error()
    assert upd(cols((p, None, 8, 9), (p, None, 8, L.QK_F64))) == L.ERR_INVALID and b"dtype" in lib.qk_last_error()
    assert upd(cols((p, p, 8, L.QK_F64), (p, None, 8, L.QK_F64))) == L.ERR_UNSUPPORTED and b"validity" in lib.qk_last_error()
    for cap in (1000, 2048, 1 << 32):
        assert upd(ok, cap=cap) == L.ERR_INVALID and b"capacity" in lib.qk_last_error()
    assert upd(ok, table=None) == L.ERR_INVALID and b"null table" in lib.qk_last_error()
    assert upd(ok, ntiles=3) == L.ERR_INVALID and b"ntiles" in lib.qk_last_error()
    assert upd(ok, wsb=8) == L.ERR_CAPACITY and b"workspace" in lib.qk_last_error()
    assert lib.qk_qsketch_workspace_bytes(0) == 0 and lib.qk_qsketch_workspace_bytes(4096) >= 4096 * 24
    m = C.cast((C.c_uint64 * 4)(), C.c_void_p)
    assert lib.qk_qsketch_merge(m, m, m, m, -1, tab, 4096, ctrl, None) == L.ERR_INVALID
    assert lib.qk_qsketch_merge(None, m, m, m, 4, tab, 4096, ctrl, None) == L.ERR_INVALID and b"null entry" in lib.qk_last_error()
    assert lib.qk_qsketch_merge(m, m, m, m, 4, tab, 4097, ctrl, None) == L.ERR_INVALID and b"capacity" in lib.qk_last_error()
    assert lib.qk_qsketch_merge(m, m, m, m, 2049, tab, 4096, ctrl, None) == L.ERR_CAPACITY
    assert lib.qk_qsketch_merge(m, m, m, m, 0, tab, 4096, None, None) == L.ERR_INVALID


def test_sass_has_warp_match_and_reduce():
    """The update kernel aggregates lanes of a bucket with match.any and redux.sync, as its comment says."""
    import subprocess
    from quokka_b200 import _lib, build
    build.build()
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True).stdout
    fun = [f for f in sass.split("Function : ") if f.split("\n", 1)[0].find("k_qsketch_update") >= 0]
    assert len(fun) == 1 and "MATCH.ANY" in fun[0] and "REDUX" in fun[0]
