"""The cross-rank steps the done-time executors share, on gloo ranks (kernels replaced by tests/cpu_shim.py):

  * runtime.Exchange.to_ranks / hand_off at worlds 1, 2 and 3: tables in source-rank order, `src_rank` on every one, None and
    empty inputs, a subset of the ranks, empty slices, and the own slice of a hand-off kept in place;
  * a traffic guard: the Exchange.__call__ and allgather_words calls and the bytes each rank sends for a multi-column sort on
    a string column, shift with and without a key, a left ordered join with a hash-partitioned build side (and one whose
    build rows sit on one rank) and as-of joins over time ranges for every strategy.  The numbers are what these programs
    moved before the executors shared these steps; moving code between the executors and the runtime must not change them."""
import numpy as np
import pytest
import torch

import ranks


def _table(**cols):
    from quokka_b200.columns import DeviceColumn, DeviceTable
    return DeviceTable({n: DeviceColumn(torch.as_tensor(v)) for n, v in cols.items()})


def _x(g):
    return g["x"].data.tolist()


def case_to_ranks():
    from quokka_b200 import runtime as RT
    w, me = RT.world_size(), RT.rank()
    ex = RT.Exchange(torch.device("cpu"))
    mine = _table(x=np.full(me + 1, me, np.int64))
    got = ex.to_ranks(mine, "all")
    assert [g.src_rank for g in got] == list(range(w)), got
    assert [_x(g) for g in got] == [[s] * (s + 1) for s in range(w)]
    # None on rank 1, an empty table on rank 2: those ranks send nothing, and still receive
    silent = {1: None, 2: _table(x=np.zeros(0, np.int64))}
    got = ex.to_ranks(silent.get(me, mine), "some silent")
    assert [g.src_rank for g in got] == [s for s in range(w) if s not in silent]
    assert all(_x(g) == [g.src_rank] * (g.src_rank + 1) for g in got)
    # to the later ranks only: rank r hears from the ranks before it
    got = ex.to_ranks(mine, "later", ranks=range(me + 1, w))
    assert [g.src_rank for g in got] == list(range(me)), got
    assert ex.to_ranks(mine, "nobody", ranks=[]) == []
    assert ex.to_ranks(None, "none anywhere") == []
    assert ex.max_over_ranks([me, w - me, 7]) == [w - 1, w, 7]


def _cuts(s, w):
    """Rank s's bounds: 1 + r + s rows to rank r, none where (r + s) % 3 == 2 (its own slice on rank 1, a later rank's on
    rank 0, an earlier rank's on rank 2)."""
    cut = [0]
    for r in range(w):
        cut.append(cut[-1] + (0 if (r + s) % 3 == 2 else 1 + r + s))
    return cut


def case_hand_off():
    from quokka_b200 import runtime as RT
    w, me = RT.world_size(), RT.rank()
    ex = RT.Exchange(torch.device("cpu"))
    cut = _cuts(me, w)
    n = cut[-1]
    t = _table(x=np.arange(n, dtype=np.int64) + 1000 * me)
    sent0 = ex.bytes_sent
    got = ex.hand_off(t, cut, "slices")
    assert ex.bytes_sent - sent0 == 8 * (n - (cut[me + 1] - cut[me])), ex.bytes_sent - sent0
    assert [g.src_rank for g in got] == [s for s in range(w) if (me + s) % 3 != 2], [g.src_rank for g in got]
    for g in got:
        c = _cuts(g.src_rank, w)
        assert _x(g) == list(range(1000 * g.src_rank + c[me], 1000 * g.src_rank + c[me + 1])), (g.src_rank, _x(g))
    own = next((g for g in got if g.src_rank == me), None)
    if own is not None:
        assert own["x"].data.data_ptr() == t["x"].data[cut[me]:].data_ptr()     # the own slice never left this rank
    # rank 0 has no table, rank 1 keeps all its rows, the others cut evenly
    if me == 0:
        got = ex.hand_off(None, None, "sparse")
    else:
        got = ex.hand_off(t, [0] * (me + 1) + [n] * (w - me) if me == 1 else [n * r // w for r in range(w + 1)], "sparse")
    assert [g.src_rank for g in got] == [s for s in range(1, w) if s > 1 or me == 1], [g.src_rank for g in got]


@pytest.mark.parametrize("world", [1, 2, 3])
def test_to_ranks_and_hand_off_gloo(tmp_path, world):
    ranks.spawn(tmp_path, world, ranks.gloo_rank, ["test_cross_rank_steps:case_to_ranks", "test_cross_rank_steps:case_hand_off"])


# ------------------------------------------------------------------ the traffic guard
def _sort(qc):
    import sort_api_cases as SA
    cols, _ = SA._mixed_table(3001, 7)
    res = qc.from_arrow(SA._arrow(cols)).sort(["s", "d", "rowid"], [False, True, False]).collect()
    assert res.num_rows == 3001


def _shift(qc, by, n):
    import shift_api_cases as SH
    res = qc.from_arrow_sorted(SH._quotes(2501, 23, 4), "time").shift(n, by=by, columns=["px", "q" if by else "sym"], suffix="_s").collect()
    assert res.num_rows == 2501


def _ordered_left_join(qc, build_rows=None):
    import ordered_join_api_cases as OJ
    s = OJ._symbols()
    if build_rows is not None:
        s = s.slice(0, build_rows)
    saved = dict(qc.exec_config)
    qc.exec_config.update(broadcast_rows=0, broadcast_cost_based=False)      # the build side hash-partitioned across ranks
    try:
        res = qc.from_arrow_sorted(OJ._quotes(), "time").join(qc.from_arrow(s), on="symbol", how="left", maintain_sort_order="left")
        assert res.collect().num_rows >= 2400
    finally:
        qc.exec_config.clear()
        qc.exec_config.update(saved)


def _asof(qc, strategy):
    import asof_strategy_api_cases as AS
    trades, quotes = AS._tables(700, 900, 6, 120, 0)
    AS.check(qc, trades, quotes, strategy, None)


PROGRAMS = {
    "sort string first": _sort,
    "shift by key": lambda qc: _shift(qc, "sym", 2),
    "shift lead no key": lambda qc: _shift(qc, None, -3),
    "ordered left join": _ordered_left_join,
    "ordered left join one build row": lambda qc: _ordered_left_join(qc, 1),
    "asof backward": lambda qc: _asof(qc, "backward"),
    "asof forward": lambda qc: _asof(qc, "forward"),
    "asof nearest": lambda qc: _asof(qc, "nearest"),
}

# world -> program -> per rank: [Exchange.__call__ calls, allgather_words calls, bytes sent to other ranks]
TRAFFIC = {
    2: {
        "sort string first": [[4, 2, 68700], [4, 2, 77948]],
        "shift by key": [[2, 1, 68604], [2, 1, 67554]],
        "shift lead no key": [[2, 1, 67500], [2, 1, 67614]],
        "ordered left join": [[5, 1, 89330], [5, 1, 83056]],
        "ordered left join one build row": [[5, 1, 65474], [5, 1, 65536]],
        "asof backward": [[3, 1, 17188], [3, 1, 19092]],
        "asof forward": [[3, 1, 17332], [3, 1, 18692]],
        "asof nearest": [[4, 1, 17380], [4, 1, 19284]],
    },
    3: {
        "sort string first": [[4, 2, 78744], [4, 2, 80344], [4, 2, 107960]],
        "shift by key": [[2, 1, 92172], [2, 1, 91176], [2, 1, 90072]],
        "shift lead no key": [[2, 1, 89964], [2, 1, 90132], [2, 1, 90192]],
        "ordered left join": [[5, 1, 109248], [5, 1, 108362], [5, 1, 103778]],
        "ordered left join one build row": [[5, 1, 81200], [5, 1, 80778], [5, 1, 80890]],
        "asof backward": [[3, 1, 23616], [3, 1, 22220], [3, 1, 26084]],
        "asof forward": [[3, 1, 24384], [3, 1, 21916], [3, 1, 25684]],
        "asof nearest": [[4, 1, 24000], [4, 1, 22604], [4, 1, 26468]],
    },
}


def _traffic(fn, qc):
    """[Exchange.__call__ calls, allgather_words calls, bytes sent] of this rank while fn(qc) runs, over every Exchange."""
    from quokka_b200 import runtime as RT
    tally = [0, 0, 0]
    call, words = RT.Exchange.__call__, RT.Exchange.allgather_words

    def counted_call(self, *a, **kw):
        before = self.bytes_sent
        out = call(self, *a, **kw)
        tally[0] += 1
        tally[2] += self.bytes_sent - before
        return out

    def counted_words(self, *a, **kw):
        tally[1] += 1
        return words(self, *a, **kw)

    RT.Exchange.__call__, RT.Exchange.allgather_words = counted_call, counted_words
    try:
        fn(qc)
    finally:
        RT.Exchange.__call__, RT.Exchange.allgather_words = call, words
    return tally


def case_traffic(qc):
    from quokka_b200 import runtime as RT
    w, me = RT.world_size(), RT.rank()
    got = {name: _traffic(fn, qc) for name, fn in PROGRAMS.items()}
    want = {name: per_rank[me] for name, per_rank in TRAFFIC[w].items()}
    assert got == want, (w, me, got)


@pytest.mark.parametrize("world", [2, 3])
def test_traffic_gloo(tmp_path, world):
    ranks.spawn(tmp_path, world, ranks.gloo_rank, ["test_cross_rank_steps:case_traffic"])


def test_one_rank_shift_has_no_boundary_pass(monkeypatch):
    """At one rank no rank receives boundary rows, so a shift runs no edge pass: one code partition (with a key), one plan
    and one gather."""
    import cpu_shim
    import shift_api_cases as SH
    from quokka_b200.df import QuokkaContext
    cpu_shim.install(monkeypatch)
    calls = []
    for name in ("partition_plan", "shift_plan", "shift_gather"):
        fn = getattr(cpu_shim, name)
        monkeypatch.setattr(cpu_shim, name, lambda *a, _fn=fn, _name=name, **kw: calls.append((_name, kw.get("want_edge", False))) or _fn(*a, **kw))
    qc = QuokkaContext()
    for by, n in (("sym", 2), (None, -1)):
        calls.clear()
        res = qc.from_arrow_sorted(SH._quotes(501, 7, 1), "time").shift(n, by=by, columns=["px"], suffix="_s").collect()
        assert res.num_rows == 501
        assert calls == [("partition_plan", False)] * (by is not None) + [("shift_plan", False), ("shift_gather", False)], (by, calls)
