"""The ordered probe and the placement kernels (csrc/join.cu) on the GPU against the numpy stand-ins of
tests/ordered_join_shim.py, bit for bit -- 0 to 2^20 + 3 probe rows, all four joins, uint8 / int32 / int64 keys, probes that
match nothing, one key with 10^5 build rows -- and DataStream.join(maintain_sort_order=...) through the API on the device."""
import re

import numpy as np
import pytest
import torch

import ordered_join_api_cases as A
import ordered_join_shim as S
import ranks
from quokka_b200 import _lib as L

pytestmark = pytest.mark.gpu

SIZES = (0, 1, 255, 256, 257, (1 << 20) + 3)
HOWS = (L.JOIN_INNER, L.JOIN_LEFT, L.JOIN_SEMI, L.JOIN_ANTI)
DTYPES = (np.uint8, np.int32, np.int64)


def _table(build_batches):
    """An ops.JoinTable over the build key batches, in order (build rows numbered across batches)."""
    from quokka_b200 import ops
    t = ops.JoinTable(sum(len(b) for b in build_batches), torch.device("cuda"))
    for b in build_batches:
        t.build(torch.from_numpy(b).cuda())
    t.check_flags()
    return t


def _same_probe(table, build_batches, probe: np.ndarray, how, what):
    pi, bi = table.probe_ordered(torch.from_numpy(probe).cuda(), how)
    ei, eb = S.ordered_pairs(probe, np.concatenate(build_batches) if build_batches else np.zeros(0, np.int64), how)
    assert np.array_equal(pi.cpu().numpy(), ei), what
    assert (bi is None) == (eb is None) and (bi is None or np.array_equal(bi.cpu().numpy(), eb)), what
    return pi, bi


def _keys(rng, n, dtype, hi):
    return rng.integers(0, hi, n).astype(dtype)


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: d.__name__)
@pytest.mark.parametrize("n", SIZES)
def test_probe_ordered_matches_the_shim(n, dtype):
    rng = np.random.default_rng(n + 7)
    hi = 200 if dtype == np.uint8 else max(4, n // 3)
    # duplicate build keys over two batches (several matches per row, more than a thread orders for a few), and some keys absent
    build = [_keys(rng, max(1, min(n // 2, 2000 if dtype == np.uint8 else n)), dtype, hi), np.repeat(_keys(rng, 3, dtype, hi), 20).astype(dtype)]
    t = _table(build)
    probe = _keys(rng, n, dtype, hi + hi // 4 if dtype != np.uint8 else 255)
    for how in HOWS:
        _same_probe(t, build, probe, how, (n, dtype.__name__, how))


@pytest.mark.parametrize("how", HOWS)
def test_probe_ordered_when_nothing_matches(how):
    build = [np.arange(1000, dtype=np.int64)]
    t = _table(build)
    probe = np.arange(5000, 5000 + 257, dtype=np.int64)
    pi, _ = _same_probe(t, build, probe, how, how)
    assert len(pi) == {L.JOIN_INNER: 0, L.JOIN_LEFT: 257, L.JOIN_SEMI: 0, L.JOIN_ANTI: 257}[how]


def test_one_key_with_1e5_build_rows_is_ordered_and_repeatable():
    """A key with 10^5 build rows (a CTA sorts them) next to keys with a few; a second call returns the same pairs."""
    rng = np.random.default_rng(3)
    b = np.concatenate([np.full(100_000, 7, np.int64), rng.integers(0, 50, 3000).astype(np.int64)])
    build = [rng.permutation(b)]
    t = _table(build)
    probe = rng.integers(0, 60, 301).astype(np.int64)
    probe[:3] = 7
    for how in HOWS:
        first = _same_probe(t, build, probe, how, how)
        again = t.probe_ordered(torch.from_numpy(probe).cuda(), how)
        assert torch.equal(first[0], again[0]) and (first[1] is None or torch.equal(first[1], again[1])), how


@pytest.mark.parametrize("n", SIZES)
def test_place_matches_the_shim(n):
    """Runs from three senders: each sends ascending positions of a disjoint share of the left rows, 0 to 3 rows for each."""
    from quokka_b200 import ops
    rng = np.random.default_rng(n + 11)
    owner, reps = rng.integers(0, 3, n), rng.integers(0, 4, n)
    pos = np.concatenate([np.repeat(np.nonzero(owner == s)[0], reps[owner == s]) for s in range(3)]).astype(np.int32)
    src, left = ops.JoinTable.place(torch.from_numpy(pos).cuda(), n)
    es, el = S.join_place(torch.from_numpy(pos), n)
    assert torch.equal(src.cpu(), es) and torch.equal(left.cpu(), el)
    again = ops.JoinTable.place(torch.from_numpy(pos).cuda(), n)
    assert torch.equal(again[0], src) and torch.equal(again[1], left)


def test_workspace_one_byte_short_is_refused():
    import ctypes as C
    from quokka_b200 import ops
    t = _table([np.arange(10, dtype=np.int64)])
    key = torch.arange(300, dtype=torch.int64, device="cuda")
    need = L.lib().qk_join_probe_ordered_workspace_bytes(300)
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    out = torch.empty(300, dtype=torch.int32, device="cuda")
    cnt = torch.zeros(1, dtype=torch.int64, device="cuda")
    kc = ops.col(key)
    rc = L.lib().qk_join_probe_ordered(t.table.data_ptr(), t.capacity, C.byref(kc), L.JOIN_INNER, out.data_ptr(), out.data_ptr(), 300,
                                       cnt.data_ptr(), ws.data_ptr(), need - 1, None)
    assert rc == L.ERR_CAPACITY
    need = L.lib().qk_join_place_workspace_bytes(300)
    pos = torch.arange(300, dtype=torch.int32, device="cuda")
    rc = L.lib().qk_join_place(pos.data_ptr(), 300, 300, out.data_ptr(), None, ws.data_ptr(), need - 1, None)
    assert rc == L.ERR_CAPACITY


@pytest.fixture
def qc():
    from quokka_b200.df import QuokkaContext
    return QuokkaContext()


@pytest.mark.parametrize("case", A.API_CASES, ids=lambda c: c.__name__)
def test_api_case_on_the_device(qc, case):
    case(qc)


def test_ordered_join_two_ranks_nccl():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    rc, out = ranks.torchrun("dist_nccl_ordered_join_check.py", 2)
    assert rc == 0 and ranks.NCCL_MARKER in out, out[-4000:]
    missing = [n for n in ranks.expand(ranks.SUITES["ordered_join"]) if not re.search(f"^{re.escape(n)}: ok", out, re.M)]
    assert not missing, f"no ok line for {missing}\n{out[-4000:]}"
