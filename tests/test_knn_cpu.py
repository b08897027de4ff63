"""Vector columns and DataStream.vector_nn_join without a GPU: the planner, the edges and the executors on tests/cpu_shim.py +
tests/knn_shim.py (numpy stand-ins for qk_knn_topk / qk_knn_merge), the reference of tests/knn_cases.py, and the C-ABI argument
checks of the new entry points."""
import ctypes as C

import numpy as np
import pytest

import cpu_shim
import knn_cases as K
import knn_shim


@pytest.fixture
def qc(monkeypatch):
    cpu_shim.install(monkeypatch)
    from quokka_b200.df import QuokkaContext
    return QuokkaContext()


def test_vector_roundtrip(qc): K.case_vector_roundtrip(qc)
def test_vector_rejects(qc): K.case_vector_rejects(qc)
def test_vector_ops(qc): K.case_vector_ops(qc)
def test_vector_plan_errors(qc): K.case_vector_plan_errors(qc)
def test_knn_api(qc): K.case_knn_api(qc)
def test_knn_api_one_batch(qc): K.case_knn_api(qc, chunk_rows=1 << 20)
def test_knn_fewer_rows(qc): K.case_knn_fewer_rows(qc)
def test_knn_args(qc): K.case_knn_args(qc)
def test_vector_parquet(qc, tmp_path): K.case_vector_parquet(qc, tmp_path)


def test_vector_empty_chunk(monkeypatch):
    import torch
    cpu_shim.install(monkeypatch)
    K.case_vector_empty_chunk(torch.device("cpu"))


def test_knn_plan_shape(qc):
    """Per-rank partial on PassThrough + CustomChannels(1), final on Broadcast + a single channel, both silent until done()."""
    from quokka_b200.executors import KnnFinalExecutor, KnnPartialExecutor
    tbl, _ = K.api_stream(n=20, d=12)
    probes, _ = K.api_probes()
    s = qc.from_arrow(tbl).vector_nn_join(probes, vec_column="vec", k=2)
    fin, part = s.node, s.node.parents[0]
    assert isinstance(fin.executor, KnnFinalExecutor) and isinstance(part.executor, KnnPartialExecutor)
    assert type(fin.partitioners[0]).__name__ == "BroadcastPartitioner" and type(fin.placement).__name__ == "SingleChannelStrategy"
    assert type(part.partitioners[0]).__name__ == "PassThroughPartitioner" and type(part.placement).__name__ == "CustomChannelsStrategy"
    assert fin.executor.silent_streams == "all" and part.executor.silent_streams == "all"
    assert fin.vectors == {"vec", "vec_probe"}


def test_reference_check_catches_wrong_answers():
    """The contract check of tests/knn_cases.py rejects a wrong row, a wrong score and a wrong order."""
    X = K.gaussian(200, 8, 3)
    phat = K.normalise(K.gaussian(3, 8, 4))
    rows, sc = K.exact_topk(X, phat, 5)
    K.check_topk(X, phat, 5, sc.astype(np.float32), rows)
    for mutate in (lambda r, s: r.__setitem__((0, 4), 199 if r[0, 4] != 199 else 198),
                   lambda r, s: s.__setitem__((1, 0), s[1, 0] + 1e-3),
                   lambda r, s: (r.__setitem__((2, slice(0, 2)), r[2, [1, 0]]), s.__setitem__((2, slice(0, 2)), s[2, [1, 0]]))):
        r, s = rows.copy(), sc.copy()
        mutate(r, s)
        with pytest.raises(AssertionError):
            K.check_topk(X, phat, 5, s, r)


def test_knn_shim_merge_order():
    """The merge rule the kernel documents: score desc, key asc, a before b on a full tie; -1 keys end a list."""
    import torch
    a_s = torch.tensor([[3.0, 1.0, -np.inf]], dtype=torch.float32)
    a_k = torch.tensor([[5, 2, -1]])
    b_s = torch.tensor([[3.0, 2.0]], dtype=torch.float32)
    b_k = torch.tensor([[4, 9]])
    s, k, src = knn_shim.knn_merge(a_s, a_k, b_s, b_k, 4)
    assert k.tolist() == [[4, 5, 9, 2]] and src.tolist() == [[3, 0, 4, 1]]


def test_knn_cabi_argument_errors():
    """qk_knn_topk / qk_knn_merge reject bad arguments before touching the device; scalar kernels reject vector columns."""
    from quokka_b200 import _lib as L
    lib = L.lib()
    x = L.qk_column(16, None, 10, L.QK_F32, 8)
    out = (C.c_float * 4)()
    rows = (C.c_int64 * 4)()
    assert lib.qk_knn_topk(C.byref(x), 16, 1, 0, out, rows, 16, 1 << 20, None) == L.ERR_INVALID            # k = 0
    assert lib.qk_knn_topk(C.byref(x), 16, 1, 257, out, rows, 16, 1 << 20, None) == L.ERR_INVALID          # k > 256
    assert lib.qk_knn_topk(C.byref(x), 16, 0, 1, out, rows, 16, 1 << 20, None) == L.ERR_INVALID            # q = 0
    bad = L.qk_column(16, None, 10, L.QK_I32, 8)
    assert lib.qk_knn_topk(C.byref(bad), 16, 1, 1, out, rows, 16, 1 << 20, None) == L.ERR_INVALID          # integer vectors
    wide = L.qk_column(16, None, 10, L.QK_F32, 4097)
    assert lib.qk_knn_topk(C.byref(wide), 16, 1, 1, out, rows, 16, 1 << 20, None) == L.ERR_INVALID         # d > 4096
    assert lib.qk_knn_topk(C.byref(x), None, 1, 1, out, rows, 16, 1 << 20, None) == L.ERR_INVALID          # no probes
    assert lib.qk_knn_merge(-1, None, None, 1, None, None, 1, 1, None, None, None, None) == L.ERR_INVALID
    assert lib.qk_knn_workspace_bytes(10, 8, 1, 0) == 0
    ws = (C.c_uint8 * 64)()
    assert lib.qk_topk_candidates(C.byref(x), 1, 1, rows, rows, ws, 64, None) == L.ERR_UNSUPPORTED         # a vector column
    h = L.qk_column(16, None, 10, L.QK_F16, 0)
    assert lib.qk_topk_candidates(C.byref(h), 1, 1, rows, rows, ws, 64, None) == L.ERR_UNSUPPORTED         # a scalar f16 column


def test_knn_no_spills():
    """`-Xptxas -v` of csrc/knn.cu: no local-memory spills in the kernels."""
    import os
    import subprocess
    from quokka_b200 import build
    r = subprocess.run([build._nvcc(), *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", os.path.join(build.CSRC, "knn.cu"), "-o", os.devnull],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    assert "spill" in r.stdout
    assert all(" 0 bytes spill stores" in line for line in r.stdout.splitlines() if "spill stores" in line), r.stdout
