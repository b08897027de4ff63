"""DataStream.gramian / covariance without a GPU: the planner and the executors on tests/cpu_shim.py + tests/gram_shim.py, the C-ABI argument checks
of qk_gram, the DMMA instructions in libqk.so, and the reference computation of tests/gram_cases.py against exact arithmetic."""
import ctypes as C
import subprocess
from fractions import Fraction

import numpy as np
import pytest

import gram_cases as GC
import gram_shim


@pytest.fixture
def qc(monkeypatch):
    gram_shim.install(monkeypatch)
    from quokka_b200.df import QuokkaContext
    return QuokkaContext()


def test_gram_lineitem(qc): GC.case_gram_lineitem(qc)
def test_gram_filtered_ints(qc): GC.case_gram_filtered_ints(qc)
def test_gram_ragged_batches(qc): GC.case_gram_ragged_batches(qc)
def test_gram_left_join_nulls(qc): GC.case_gram_left_join_nulls(qc)
def test_gram_empty(qc): GC.case_gram_empty(qc)
def test_gram_rejects_strings_and_dates(qc): GC.case_gram_rejects_strings_and_dates(qc)


def test_gram_plan_shape(qc):
    """Per-rank partial on PassThrough + CustomChannels(1), final on Broadcast + a single channel, both silent until done()."""
    from quokka_b200.executors import GramFinalExecutor, GramPartialExecutor
    import api_cases as A
    s = qc.from_arrow(A.tables()[0]).gramian(GC.LINEITEM_COLS)
    fin = s.node
    part = fin.parents[0]
    assert isinstance(fin.executor, GramFinalExecutor) and isinstance(part.executor, GramPartialExecutor)
    assert type(fin.partitioners[0]).__name__ == "BroadcastPartitioner" and type(fin.placement).__name__ == "SingleChannelStrategy"
    assert type(part.partitioners[0]).__name__ == "PassThroughPartitioner" and type(part.placement).__name__ == "CustomChannelsStrategy"
    assert fin.executor.silent_streams == "all" and part.executor.silent_streams == "all"
    assert s.schema == GC.LINEITEM_COLS


def test_reference_error_is_far_below_the_bound():
    """gram_ref's own error, against exact rational arithmetic, on mixed magnitudes and a mean far from zero."""
    rng = np.random.default_rng(11)
    n, k = 400, 3
    x = np.stack([rng.normal(1e6, 1.0, n), rng.normal(0, 1e-8, n) * 10.0 ** rng.integers(-3, 4, n), rng.normal(-3e3, 50, n)], axis=1)
    shift = np.array([1e6 + 0.25, 0.0, -3e3])
    g, bound = GC.gram_ref(x, shift)
    y = x - shift
    for i in range(k):
        for j in range(k):
            exact = sum(Fraction(float(a)) * Fraction(float(b)) for a, b in zip(y[:, i], y[:, j]))
            err = abs(Fraction(float(g[i, j])) - exact)
            assert err <= Fraction(float(bound[i, j])) / 64, (i, j)            # one final rounding + 2^-64 per term


def test_sass_has_fp64_tensor_core_mma():
    from quokka_b200 import _lib, build
    build.build()
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True).stdout
    assert "DMMA" in sass


def test_gram_argument_errors_are_reported_without_a_gpu():
    from quokka_b200 import _lib as L
    lib = L.lib()
    ws = (C.c_uint8 * 64)()
    g = (C.c_double * 4)()

    def cols(*specs):
        arr = (L.qk_column * len(specs))()
        for i, (data, valid, length, dt) in enumerate(specs):
            arr[i] = L.qk_column(data, valid, length, dt, 0)
        return arr

    buf = (C.c_double * 8)()
    p = C.cast(buf, C.c_void_p)
    ok = cols((p, None, 8, L.QK_F64), (p, None, 8, L.QK_F64))
    assert lib.qk_gram(ok, 0, 8, None, g, None, 0, ws, 64, None) == L.ERR_INVALID                   # k < 1
    assert b"k must be" in lib.qk_last_error()
    assert lib.qk_gram(cols((None, None, 8, L.QK_F64), (p, None, 8, L.QK_F64)), 2, 8, None, g, None, 0, ws, 64, None) == L.ERR_INVALID
    assert b"null data" in lib.qk_last_error()
    assert lib.qk_gram(cols((p, None, 8, L.QK_F64), (p, None, 7, L.QK_F64)), 2, 8, None, g, None, 0, ws, 64, None) == L.ERR_INVALID
    assert b"rows" in lib.qk_last_error()
    assert lib.qk_gram(cols((p, None, 8, L.QK_U8), (p, None, 8, L.QK_F64)), 2, 8, None, g, None, 0, ws, 64, None) == L.ERR_INVALID
    assert b"dtype" in lib.qk_last_error()
    assert lib.qk_gram(cols((p, p, 8, L.QK_F64), (p, None, 8, L.QK_F64)), 2, 8, None, g, None, 0, ws, 64, None) == L.ERR_UNSUPPORTED
    assert b"validity" in lib.qk_last_error()
    assert lib.qk_gram(ok, 2, 8, None, g, None, 0, ws, 64, None) == L.ERR_CAPACITY                  # 64 bytes of workspace
    assert b"workspace" in lib.qk_last_error()
    assert lib.qk_gram(ok, 2, 8, None, None, None, 0, ws, 64, None) == L.ERR_INVALID                # no output
    assert lib.qk_gram(cols((p, None, 0, L.QK_F64), (p, None, 0, L.QK_F64)), 2, 0, None, g, None, 0, None, 0, None) == 0   # no-op
    assert lib.qk_gram_workspace_bytes(8, 0) == 0
    assert lib.qk_gram_workspace_bytes(1 << 20, 1031) > 1031 * 16


def test_gram_state_shim_matches_numpy():
    import torch
    rng = np.random.default_rng(5)
    st = gram_shim.GramState(3, None)
    x = rng.normal(size=(50, 3))
    c = np.array([0.5, -1.0, 2.0])
    for lo, hi in ((0, 17), (17, 17), (17, 50)):
        st.update([torch.from_numpy(x[lo:hi, i].copy()) for i in range(3)], torch.from_numpy(c))
    y = x - c
    np.testing.assert_allclose(st.gram.numpy(), y.T @ y, rtol=1e-12)
    np.testing.assert_allclose(st.sums.numpy(), y.sum(axis=0), rtol=1e-12)
    assert st.n == 50
