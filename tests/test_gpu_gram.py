"""qk_gram (csrc/gram.cu) and DataStream.gramian / covariance on the real sm_90a kernels.

Exact cases use integer values with |v|^2 n < 2^53, so every summation order gives the exact result: the kernel must match
the reference bit for bit.  General data is checked against the sequential-summation bound of tests/gram_cases.py."""
import numpy as np
import pytest
import torch

import gram_cases as GC

pytestmark = pytest.mark.gpu

DTYPES = [torch.float64, torch.float32, torch.int32, torch.int64]


def _gram(columns, shift=None, sums=True, variant=0, state=None):
    from quokka_b200 import ops
    st = state or ops.GramState(len(columns), columns[0].device)
    st.update(columns, None if shift is None else torch.as_tensor(shift, dtype=torch.float64, device="cuda"), variant=variant)
    torch.cuda.synchronize()
    return st


def _int_columns(n, k, vmax, seed, misalign=False):
    """k integer-valued columns of mixed dtypes (host int64 matrix + device columns); misalign: every column is a view that
    starts one element into its buffer (4- or 8-byte offsets, never 16-byte aligned)."""
    rng = np.random.default_rng(seed)
    x = rng.integers(-vmax, vmax + 1, size=(n, k), dtype=np.int64)
    cols = []
    for j in range(k):
        dt = DTYPES[j % 4]
        t = torch.from_numpy(np.concatenate([[7], x[:, j]]) if misalign else x[:, j].copy()).to(dt).cuda()
        cols.append(t[1:] if misalign else t)
    return x, cols


def _exact_ref(x, shift=None):
    y = x if shift is None else x - np.asarray(shift, dtype=np.int64)
    if y.shape[0] * y.shape[1] ** 2 <= 2e8:
        return (y.T @ y).astype(np.float64), y.sum(axis=0).astype(np.float64)        # int64 products
    yf = y.astype(np.float64)                                                         # BLAS: exact too (every partial < 2^53)
    return yf.T @ yf, yf.sum(axis=0)


@pytest.mark.parametrize("variant", [1, 2])
@pytest.mark.parametrize("n", [0, 1, 15, 16, 17, 1000, 100_003, 5_000_011])
def test_exact_rows(n, variant):
    x, cols = _int_columns(n, 7, 1000, seed=n)
    st = _gram(cols, variant=variant)
    g, s = _exact_ref(x)
    assert np.array_equal(st.gram.cpu().numpy(), g) and np.array_equal(st.sums.cpu().numpy(), s)


@pytest.mark.parametrize("variant", [1, 2])
@pytest.mark.parametrize("k", [1, 2, 3, 4, 7, 8, 16, 17, 63, 64, 65, 129, 300, 1031])
def test_exact_columns(k, variant):
    n = 1000 if k > 300 else 4099
    x, cols = _int_columns(n, k, 1000, seed=k)
    shift = np.arange(k) % 5 - 2
    st = _gram(cols, shift=shift, variant=variant)
    g, s = _exact_ref(x, shift)
    assert np.array_equal(st.gram.cpu().numpy(), g)
    assert np.array_equal(st.sums.cpu().numpy(), s)


@pytest.mark.parametrize("k,n", [(4, 100_003), (17, 4099), (65, 2050), (300, 3001)])
def test_exact_misaligned_columns_and_no_sums(k, n):
    x, cols = _int_columns(n, k, 3000, seed=k + 1, misalign=True)
    assert any(c.data_ptr() % 16 for c in cols)
    from quokka_b200 import ops
    st = ops.GramState(k, "cuda")
    sums_before = st.sums.clone()
    from quokka_b200 import _lib as L
    import ctypes as C
    ws = ops._ws(L.lib().qk_gram_workspace_bytes(n, k), "cuda")
    L.check(L.lib().qk_gram(ops.cols(cols), k, n, None, st.gram.data_ptr(), None, 0, ws.data_ptr(), ws.numel(), ops._stream()))
    torch.cuda.synchronize()
    g, _ = _exact_ref(x)
    assert np.array_equal(st.gram.cpu().numpy(), g)
    assert torch.equal(st.sums, sums_before)


def _general(n, k, seed):
    """Mixed magnitudes and means far from zero."""
    rng = np.random.default_rng(seed)
    scale = 10.0 ** rng.integers(-6, 7, k)
    mean = 10.0 ** rng.integers(-2, 9, k) * rng.choice([-1, 1], k)
    x = rng.normal(size=(n, k)) * scale + mean
    return x, [torch.from_numpy(x[:, j].copy()).cuda() for j in range(k)]


@pytest.mark.parametrize("variant", [1, 2])
@pytest.mark.parametrize("n,k", [(300_007, 5), (20_011, 70), (4_099, 257)])
def test_general_data_within_bound(n, k, variant):
    x, cols = _general(n, k, seed=n + k)
    shift = x[0]
    st = _gram(cols, shift=shift, variant=variant)
    g, b = GC.gram_ref(x, shift)
    GC.assert_within(st.gram.cpu().numpy(), g, b, "gram")
    s_ref = (x - shift).astype(np.longdouble).sum(axis=0).astype(np.float64)
    assert np.all(np.abs(st.sums.cpu().numpy() - s_ref) <= n * 2.0 ** -53 * np.abs(x - shift).sum(axis=0))
    g2 = _gram(cols, shift=shift, variant=variant).gram
    assert torch.equal(st.gram, g2), "two runs on the same inputs must be bit-identical"


def test_accumulation_across_calls():
    x, cols = _general(200_003, 33, seed=9)
    half = 77_777
    st = _gram([c[:half] for c in cols])
    _gram([c[half:] for c in cols], state=st)
    whole = _gram(cols)
    g, b = GC.gram_ref(x)
    GC.assert_within(st.gram.cpu().numpy(), g, b, "two halves")
    GC.assert_within(whole.gram.cpu().numpy(), g, b, "whole")
    assert st.n == whole.n == len(x)


def test_symmetric_output():
    x, cols = _general(10_001, 150, seed=4)
    G = _gram(cols).gram
    assert torch.equal(G, G.T)


@pytest.fixture
def qc():
    from quokka_b200.df import QuokkaContext
    return QuokkaContext()


def test_gram_lineitem(qc): GC.case_gram_lineitem(qc)
def test_gram_filtered_ints(qc): GC.case_gram_filtered_ints(qc)
def test_gram_ragged_batches(qc): GC.case_gram_ragged_batches(qc)
def test_gram_left_join_nulls(qc): GC.case_gram_left_join_nulls(qc)
def test_gram_empty(qc): GC.case_gram_empty(qc)
def test_gram_rejects_strings_and_dates(qc): GC.case_gram_rejects_strings_and_dates(qc)


def test_covariance_wide_matches_numpy(qc):
    from quokka_b200.columns import DeviceTable
    x, _ = _general(30_011, 40, seed=21)
    names = [f"c{j}" for j in range(40)]
    d = qc.from_device(DeviceTable.from_numpy({n: x[:, j].copy() for j, n in enumerate(names)}), batch_rows=4096)
    c, b = GC.cov_ref(x)
    GC.assert_within(GC.table_matrix(d.covariance(names), names), c, b, "covariance")
