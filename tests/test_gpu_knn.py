"""qk_knn_topk / qk_knn_merge through the C-ABI against the fp64 reference of tests/knn_cases.py, vector rows through qk_gather and
the contiguous exchange, and the vector_nn_join API cases on the real kernels."""
import numpy as np
import pytest
import torch

import knn_cases as K
import ranks

pytestmark = pytest.mark.gpu


def _ops():
    from quokka_b200 import ops
    return ops


def _run(X, P, k, dtype=torch.float32):
    ops = _ops()
    x = torch.from_numpy(np.ascontiguousarray(X)).to(dtype).cuda()
    phat = K.normalise(P)
    s, r = ops.knn_topk(x, torch.from_numpy(phat).cuda(), k)
    return phat, s.cpu().numpy(), r.cpu().numpy()


@pytest.mark.parametrize("d", [1, 3, 8, 100, 768, 4096])
@pytest.mark.parametrize("k", [1, 10, 256])
def test_exact_integer_ranking(d, k):
    """Signed permutations of one base vector: one exact norm, exact dots, real ties; rows must equal the exact ranking with
    ties in row order, for both tile shapes (q = 3 and q = 40)."""
    n = 700 if d < 4096 else 300
    X = K.signed_permutations(n, d, seed=d)
    for q in (3, 40):
        P = K.exact_probes(q, d, seed=q + d)
        phat, s, r = _run(X, P, k)
        er, es = K.exact_topk(X, phat, k)
        assert (r == er).all()
        K.check_topk(X, phat, k, s, r)


@pytest.mark.parametrize("gen", ["gaussian", "clustered"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_general_data(gen, dtype):
    X = getattr(K, gen)(20_011, 96, seed=4)
    if dtype == torch.float16:
        X = X.astype(np.float16).astype(np.float32)
    for q, k in ((1, 10), (16, 10), (17, 32), (200, 5)):
        P = K.gaussian(q, 96, seed=q)
        phat, s, r = _run(X, P, k, dtype)
        K.check_topk(X, phat, k, s, r)


@pytest.mark.parametrize("n", [0, 1, 5, 63, 64, 65, 127, 128, 129, 1000])
def test_tile_edges_and_short_batches(n):
    X = K.gaussian(n, 19, seed=n)
    for q in (1, 17):
        P = K.gaussian(q, 19, seed=7)
        phat, s, r = _run(X, P, 10)
        K.check_topk(X, phat, 10, s, r)


def test_zero_and_nan_rows():
    X = K.gaussian(300, 8, seed=1)
    X[[3, 50, 299]] = 0.0
    X[10, 2] = np.nan
    X[11, 0] = np.inf
    phat, s, r = _run(X, K.gaussian(4, 8, seed=2), 256)
    assert not set(r.reshape(-1).tolist()) & {3, 50, 299, 10, 11}
    K.check_topk(X, phat, 256, s, r)


def test_probe_chunking_is_invisible(monkeypatch):
    ops = _ops()
    X = K.clustered(5000, 33, seed=3)
    P = K.gaussian(300, 33, seed=5)
    phat, s, r = _run(X, P, 7)
    monkeypatch.setattr(ops, "KNN_WS_BUDGET", 1)          # every call takes the smallest chunk
    _, s2, r2 = _run(X, P, 7)
    assert (r == r2).all() and (s.view(np.uint32) == s2.view(np.uint32)).all()
    K.check_topk(X, phat, 7, s, r)


def test_misaligned_view():
    ops = _ops()
    n, d = 513, 7
    X = K.gaussian(n, d, seed=8)
    buf = torch.empty(n * d + 1, dtype=torch.float32, device="cuda")
    buf[1:] = torch.from_numpy(X.reshape(-1)).cuda()
    view = buf[1:].view(n, d)
    phat = torch.from_numpy(K.normalise(K.gaussian(3, d, seed=9))).cuda()
    s1, r1 = ops.knn_topk(view, phat, 12)
    s2, r2 = ops.knn_topk(view.clone(), phat, 12)
    assert torch.equal(r1, r2) and torch.equal(s1.view(torch.int32), s2.view(torch.int32))


def test_scores_bit_identical_across_batchings_shapes_and_runs():
    """k >= n returns every row's score: a row's score must not depend on its position, the batch, q or the call."""
    ops = _ops()
    X = K.gaussian(250, 130, seed=11)
    x = torch.from_numpy(X).cuda()
    P = torch.from_numpy(K.normalise(K.gaussian(40, 130, seed=12))).cuda()

    def by_row(xs, base, q):
        s, r = ops.knn_topk(xs, P[:q], 256)
        out = {}
        for p in range(q):
            for sc, row in zip(s[p].cpu().numpy(), r[p].cpu().numpy()):
                if row >= 0:
                    out[(p, int(row) + base)] = np.float32(sc).view(np.uint32)
        return out
    whole = by_row(x, 0, 40)
    parts = by_row(x[:97], 0, 40) | by_row(x[97:], 97, 40)
    assert whole == parts
    one = by_row(x, 0, 1)                                  # the 64 x 16 tile shape
    assert all(whole[key] == v for key, v in one.items())
    assert by_row(x, 0, 40) == whole


def test_merge_matches_reference():
    import knn_shim
    ops = _ops()
    rng = np.random.default_rng(3)
    q, ka, kb, k = 9, 6, 4, 7
    def lists(kk, base):
        s = -np.sort(-rng.integers(0, 5, size=(q, kk)).astype(np.float32), axis=1)
        key = np.tile(np.arange(kk, dtype=np.int64), (q, 1)) + base
        key[2, kk // 2:] = -1
        s[2, kk // 2:] = -np.inf
        return torch.from_numpy(s), torch.from_numpy(key)
    a, b = lists(ka, 0), lists(kb, 100)
    want = knn_shim.knn_merge(*a, *b, k)
    got = ops.knn_merge(a[0].cuda(), a[1].cuda(), b[0].cuda(), b[1].cuda(), k)
    for g, w in zip(got, want):
        assert torch.equal(g.cpu(), w)


def test_gather_vector_rows():
    ops = _ops()
    for dt in (torch.float32, torch.float16):
        x = torch.randn(1000, 37, device="cuda").to(dt)
        s = torch.arange(1000, device="cuda", dtype=torch.int64)
        idx = torch.tensor([5, -1, 999, 0, 5], dtype=torch.int32, device="cuda")
        gx, gs = ops.gather([x, s], idx)
        want = x[idx.clamp(min=0).long()].clone()
        want[1] = 0
        assert torch.equal(gx, want) and gs.tolist() == [5, 0, 999, 0, 5]


def test_xchg_push_recv_vector_rows():
    """One-rank channel: contiguous rows of a vector column and a scalar column through qk_xchg_push / qk_xchg_recv."""
    from quokka_b200 import _lib as L
    ops = _ops()
    ctrl = torch.zeros(L.XCHG_CTRL_BYTES, dtype=torch.uint8, device="cuda")
    mb_bytes = 1 << 22
    mailbox = torch.zeros(mb_bytes, dtype=torch.uint8, device="cuda")
    ch = ops.XchgChannel(1, 0, [ctrl.data_ptr()], [mailbox.data_ptr()], mb_bytes, torch.device("cuda"))
    x = torch.randn(3000, 300, device="cuda").to(torch.float16)
    ids = torch.arange(3000, dtype=torch.int64, device="cuda")
    ch.meta([2000])
    base1 = (1000 * 600 + 255) // 256 * 256
    ch.push([x, ids], [500], [1500], [[0, base1]])
    ox = torch.empty(1000, 300, dtype=torch.float16, device="cuda")
    oi = torch.empty(1000, dtype=torch.int64, device="cuda")
    ch.recv([0, base1], [ox, oi])
    torch.cuda.synchronize()
    assert torch.equal(ox, x[500:1500]) and torch.equal(oi, ids[500:1500])


@pytest.fixture
def qc():
    from quokka_b200.df import QuokkaContext
    return QuokkaContext()


def test_api_vector_roundtrip(qc): K.case_vector_roundtrip(qc)
def test_api_vector_rejects(qc): K.case_vector_rejects(qc)
def test_api_vector_ops(qc): K.case_vector_ops(qc)
def test_api_vector_plan_errors(qc): K.case_vector_plan_errors(qc)
def test_api_knn(qc): K.case_knn_api(qc)
def test_api_knn_fewer_rows(qc): K.case_knn_fewer_rows(qc)
def test_api_knn_args(qc): K.case_knn_args(qc)
def test_api_vector_parquet(qc, tmp_path): K.case_vector_parquet(qc, tmp_path)
def test_vector_empty_chunk(): K.case_vector_empty_chunk(torch.device("cuda"))


def test_api_two_nccl_ranks():
    """When the box shows >= 2 GPUs: the vector and vector_nn_join API cases on 2 NCCL ranks (tests/dist_nccl_check.py knn)."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    ranks.nccl_suites("knn")
