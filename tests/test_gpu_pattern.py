"""qk_pattern_search through the C-ABI against the brute-force oracle of tests/pattern_cases.py (bound times are integers and
the link decisions fp64, so the answers must be equal), the pruning rule and the step budget, the entry point's argument errors,
and the pattern_recognize API cases on the real kernels."""
import numpy as np
import pyarrow as pa
import pytest
import torch

import pattern_cases as P
import pattern_shim
import ranks

pytestmark = pytest.mark.gpu


def _ops():
    from quokka_b200 import ops
    return ops


def _kernel(*a, **k):
    return P.search(_ops().pattern_search, *a, device="cuda", **k)


def _stream(seed, n, keys, tmax):
    rng = np.random.default_rng(seed)
    return pa.table({"time": np.sort(rng.integers(0, tmax, n)).astype(np.int64), "sym": rng.integers(0, keys, n).astype(np.int64),
                     "px": rng.integers(0, 10, n).astype(np.float64), "sz": rng.integers(0, 5, n).astype(np.int64)})


@pytest.mark.parametrize("m", [2, 3, 4, 5])
@pytest.mark.parametrize("keys", [1, 7])
@pytest.mark.parametrize("seed", range(4))
def test_kernel_against_oracle(m, keys, seed):
    """Generated streams with dense ties and generated link programs; spans from 0 to past every segment's end."""
    tab = P.random_stream(seed * 31 + m + keys, n=(40 if m == 2 else 25 if m == 3 else 12) * keys, keys=keys, tmax=12 * keys, nulls=seed == 1)
    ev = P.random_events(seed * 17 + m * 3 + keys, m)
    for span in (0, 2, 9, 10 ** 6):
        assert _kernel(tab, "time", ev, span, "sym") == P.pattern_recognize(tab, "time", ev, span, "sym"), (ev, span)


def test_kernel_lexicographic_rule():
    """The two hand-worked tie cases in both row orders: tied rows that lead to different completions, and the cap path (a level
    that binds earlier than the best match lifts the caps below it)."""
    t = pa.table({"t": np.array([1, 1, 2, 2, 5, 9], np.int64), "k": np.zeros(6, np.int64),
                  "v": np.array([1.0, 2.0, 10.0, 20.0, 15.0, 25.0])})
    ev = [("a", "v = 1"), ("b", "v >= 2"), ("c", "c.v > b.v")]
    for tab in (t, t.take(pa.array([0, 1, 3, 2, 4, 5]))):
        assert _kernel(tab, "t", ev, 100, "k") == [(0, 1, 2, 5)]
    t = pa.table({"t": np.array(P.CAP_TABLE["t"], np.int64), "k": np.zeros(7, np.int64), "v": np.array(P.CAP_TABLE["v"])})
    for tab in (t, t.take(pa.array([0, 2, 1, 3, 4, 5, 6]))):
        assert _kernel(tab, "t", P.CAP_EVENTS, 20, "k") == [(0, 1, 2, 3, 12)]


@pytest.mark.parametrize("m", [3, 4, 5])
def test_kernel_against_oracle_dense_ties(m):
    """Many rows per timestamp and chained link programs: the caps of the best match, and when they are lifted, decide."""
    for seed in range(100):
        tab = P.tie_stream(seed * 5 + m)
        ev = P.tie_events(seed * 11 + m, m)
        for span in (3, 10):
            assert _kernel(tab, "time", ev, span, "sym") == P.pattern_recognize(tab, "time", ev, span, "sym"), (seed, ev, span)


@pytest.mark.parametrize("m", [6, 7, 8])
def test_long_patterns_against_oracle(m):
    tab = P.random_stream(m, n=16, keys=1, tmax=30)
    ev = [("a", None)] + [(chr(97 + i), f"px >= {chr(96 + i)}.px - 4" if i % 2 else "sz != 4") for i in range(1, m)]
    for span in (8, 30):
        assert _kernel(tab, "time", ev, span, "sym") == P.pattern_recognize(tab, "time", ev, span, "sym")


@pytest.mark.parametrize("m", [2, 4, 8])
def test_many_keys_against_the_search_restated(m):
    """5 000 keys, 150 000 rows: the kernel against the host restatement of its search (itself checked against the oracle)."""
    tab = _stream(m, 150_000, 5000, 1000)
    ev = [("a", "px >= 5")] + [(chr(97 + i), "px < b.px" if i == 2 else "sz >= 2") for i in range(1, m)]
    got = _kernel(tab, "time", ev, 200, "sym")
    assert got == P.search(pattern_shim.pattern_search, tab, "time", ev, 200, "sym")
    assert len(got) > 100


def test_million_rows_row_local():
    """~10^6 rows, a two-event row-local pattern: the answer per start is the first row of its key after it (strictly later) that
    satisfies event 1 and lies in the span -- a searchsorted per key."""
    n = 1_000_000
    tab = _stream(5, n, 300, 10 ** 7)
    ev = [("a", "px >= 8"), ("b", "px = 0 and sz > 2")]
    span = 20_000
    got = _kernel(tab, "time", ev, span, "sym")
    t, k, px, sz = (tab[c].to_numpy() for c in ("time", "sym", "px", "sz"))
    want = []
    for key in np.unique(k):
        sel = k == key
        tt, pp, ss = t[sel], px[sel], sz[sel]
        bt = tt[(pp == 0) & (ss > 2)]
        for t0 in tt[pp >= 8]:
            j = np.searchsorted(bt, t0, side="right")
            if j < len(bt) and bt[j] <= t0 + span:
                want.append((int(key), int(t0), int(bt[j])))
    assert got == sorted(want, key=lambda x: (str(x[0]), *x[1:])) and len(want) > 10_000


def test_pruning_rule_and_budget():
    """A row-local pattern over a long span finishes within a budget a little above the span (each level ends with its first
    binding), and the rows-tested counter says so exactly: a start at t tests t + 1 (b), t + 2 (c) and every row of (t + 2, t + 1000]
    for d.  The same pattern with link programs chained through every level must search the span at every level and runs into
    the same budget: an ordinary QkError return naming the start."""
    from quokka_b200 import _lib as L
    n, span = 4000, 1000
    tab = pa.table({"t": np.arange(n, dtype=np.int64), "k": np.zeros(n, np.int64), "v": np.ones(n)})
    tested = torch.zeros(1, dtype=torch.int64, device="cuda")
    local = [("a", "v = 1"), ("b", "v = 1"), ("c", "v = 1"), ("d", "v = 2")]
    assert _kernel(tab, "t", local, span, "k", budget=3 * (span + 1) + 64, rows_tested=tested) == []
    want = sum(min(s + span, n - 1) - s for s in range(n))          # rows s + 1 .. min(s + span, n - 1), each tested once
    assert int(tested.item()) == want
    host = torch.zeros(1, dtype=torch.int64)
    P.search(pattern_shim.pattern_search, tab, "t", local, span, "k", rows_tested=host)
    assert int(host.item()) == want
    linked = [("a", "v = 1"), ("b", "v = 1"), ("c", "c.v >= b.v"), ("d", "d.v = 2 + 0 * c.v")]
    with pytest.raises(L.QkError, match="tested more than"):
        _kernel(tab, "t", linked, span, "k", budget=3 * (span + 1) + 64)


def test_argument_errors():
    from quokka_b200 import _lib as L
    ops = _ops()
    dev = "cuda"
    t = torch.arange(4, dtype=torch.int64, device=dev)
    by = torch.zeros(4, dtype=torch.int32, device=dev)
    seg = torch.tensor([0, 4], dtype=torch.int64, device=dev)
    cand = torch.full((4,), 3, dtype=torch.uint8, device=dev)
    starts = torch.arange(4, dtype=torch.int32, device=dev)
    ok = dict(maxspan=10, link_cols=[], link_valid=[], links=[[], []], budget=100)

    def call(**kw):
        a = dict(ok, **kw)
        return ops.pattern_search(a.pop("time", t), a.pop("by", by), seg, 1, cand, starts, a.pop("m", 2), a["maxspan"], a["link_cols"],
                                  a["link_valid"], a["links"], a["budget"])
    assert call().cpu().tolist() == [[0, 1], [1, 2], [2, 3], [-1, -1]]
    # a segment that ends before the start's row, and one past the columns: no match, nothing read outside them
    for bad in ([0, 2], [0, 1 << 40]):
        out = ops.pattern_search(t, by, torch.tensor(bad, dtype=torch.int64, device=dev), 1, cand, starts, 2, 10, [], [], [[], []], 100)
        assert out.cpu().tolist()[2:] == [[-1, -1], [-1, -1]]
    for kw, msg in [(dict(seg_n=3), "segment offsets"), (dict(cand_n=3), "candidate mask")]:
        with pytest.raises(L.QkError, match=msg):
            ops.pattern_search(t, by, seg if "seg_n" not in kw else torch.zeros(3, dtype=torch.int64, device=dev), 1,
                               cand if "cand_n" not in kw else cand[:3], starts, 2, 10, [], [], [[], []], 100)
    for kw, msg in [(dict(m=1, links=[[]]), "events"), (dict(m=9, links=[[]] * 9), "events"), (dict(maxspan=-1), "maxspan"),
                    (dict(budget=0), "budget"), (dict(time=t.to(torch.int32)), "int64"), (dict(by=by.to(torch.int64)), "int32"),
                    (dict(links=[[(L.OP_CONST, 0, 0, 1.0, 0)], []]), "event 0"),
                    (dict(links=[[], [(L.OP_COL, 0, 0, 0.0, 0)]]), "column slot"),
                    (dict(link_cols=[t.double()], link_valid=[None], links=[[], [(L.OP_COL, 0, 2, 0.0, 0)]]), "reads event"),
                    (dict(link_cols=[t.double()], link_valid=[None], links=[[], [(L.OP_COL, 0, 1, 0.0, 0), (L.OP_IN_SET, 0, 8, 0.0, 1)]]), "not supported"),
                    (dict(link_cols=[t.double()], link_valid=[None], links=[[], [(L.OP_ADD, 0, 0, 0.0, 0)]]), "underflow"),
                    (dict(link_cols=[t.double().reshape(2, 2)], link_valid=[None]), "scalar")]:
        with pytest.raises(L.QkError, match=msg):
            call(**kw)


@pytest.fixture
def qc():
    from quokka_b200.df import QuokkaContext
    return QuokkaContext()


@pytest.mark.parametrize("case", P.API_CASES + P.SINGLE_RANK_CASES, ids=lambda c: c.__name__)
def test_api_case(qc, case):
    case(qc)


def test_api_two_nccl_ranks():
    """When the box shows >= 2 GPUs: the pattern_recognize API cases on 2 NCCL ranks (tests/dist_nccl_check.py pattern)."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    ranks.nccl_suites("pattern")
