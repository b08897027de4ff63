"""DataStream.join(maintain_sort_order=...) without a GPU: the plan (an OrderedStream with its sort column mapped, sides never
swapped, a stable pass-through edge for the ordered side, the build edge by the unordered join's rule, no Bloom filter), the
refusals, the unordered join's plan left as it was, the numpy stand-ins of the two kernels, and the API cases through the
planner and the executors on the shims."""
import numpy as np
import pyarrow as pa
import pytest
import torch

import cpu_shim
import ordered_join_api_cases as A
import ordered_join_shim as S
from quokka_b200 import _lib as L
from quokka_b200.datastream import OrderedStream
from quokka_b200.target_info import BroadcastPartitioner, HashPartitioner, PassThroughPartitioner


@pytest.fixture
def qc(monkeypatch):
    cpu_shim.install(monkeypatch)
    from quokka_b200.df import QuokkaContext
    return QuokkaContext()


def _join_actor(qc, stream):
    g = qc.plan(stream.node)
    joins = [a for a in g.actors.values() if a.kind == "exec" and "Join" in type(a.obj).__name__]
    assert len(joins) == 1
    j = joins[0]
    edges = {sid: next(ti for tgt, s, ti in g.actors[src].targets if tgt == j.id and s == sid) for sid, src in j.sources.items()}
    return g, j, edges


def _small(qc):
    big = pa.table({"time": np.arange(50, dtype=np.int64), "k": np.arange(50, dtype=np.int64) % 7, "v": np.arange(50.0)})
    dim = pa.table({"k": np.arange(7, dtype=np.int64), "w": np.arange(7, dtype=np.int32)})
    return qc.from_arrow_sorted(big, "time"), qc.from_arrow(dim), qc.from_arrow_sorted(dim, "k")


@pytest.mark.parametrize("broadcast_rows", [1 << 40, 0])
def test_plan_keeps_the_left_side_in_place(qc, broadcast_rows):
    qc.set_config("broadcast_rows", broadcast_rows)
    q, d, _ = _small(qc)
    # the build side is far larger than the ordered side: the unordered join would swap them
    s = q.select(["time", "k"]).join(qc.from_arrow(pa.table({"k": np.arange(500, dtype=np.int64) % 7, "z": np.arange(500)})),
                                      on="k", maintain_sort_order="left")
    assert isinstance(s, OrderedStream) and s.sorted_by == "time"
    g, j, edges = _join_actor(qc, s)
    assert type(j.obj).__name__ == "OrderedJoinExecutor" and j.obj.probe_is_left and j.obj.probe_on == "k" and j.ordered
    assert isinstance(edges[0].partitioner, PassThroughPartitioner) and edges[0].stable and edges[0].bloom_key is None
    assert isinstance(edges[1].partitioner, BroadcastPartitioner if broadcast_rows else HashPartitioner) and edges[1].stable


def test_plan_keeps_the_right_side_in_place(qc):
    q, _, d_sorted = _small(qc)
    s = q.join(d_sorted, on="k", maintain_sort_order="right")
    assert isinstance(s, OrderedStream) and s.sorted_by == "k"
    _, j, edges = _join_actor(qc, s)
    assert not j.obj.probe_is_left and isinstance(edges[0].partitioner, PassThroughPartitioner) and edges[0].stable
    q2 = q.rename({"time": "t"})
    s2 = qc.from_arrow(pa.table({"k": [1, 2], "time": [5, 6]})).join(q2.rename({"t": "time"}), on="k", maintain_sort_order="right")
    assert s2.sorted_by == "time_2" and s2.schema == ["k", "time", "time_2", "v"]


def test_schema_is_the_unordered_joins(qc):
    q, d, d_sorted = _small(qc)
    for how in ("inner", "left", "semi", "anti"):
        assert q.join(d, on="k", how=how, maintain_sort_order="left").schema == q.join(d, on="k", how=how).schema
    assert q.join(d_sorted, on="k", maintain_sort_order="right").schema == q.join(d_sorted, on="k").schema


def test_refusals(qc):
    q, d, d_sorted = _small(qc)
    unordered = qc.from_arrow(pa.table({"time": [1, 2], "k": [1, 2]}))
    with pytest.raises(AssertionError):
        unordered.join(d, on="k", maintain_sort_order="left")
    with pytest.raises(AssertionError):
        q.join(d, on="k", maintain_sort_order="right")                  # the right side is not ordered
    with pytest.raises(NotImplementedError):
        q.join(d_sorted, on="k", how="left", maintain_sort_order="right")
    for how in ("semi", "anti"):
        with pytest.raises(AssertionError):
            q.join(d_sorted, on="k", how=how, maintain_sort_order="right")
    with pytest.raises(ValueError):
        q.join(d, on="k", maintain_sort_order="both")


def test_without_an_order_nothing_changes(qc):
    q, d, _ = _small(qc)
    s = q.join(d, on="k")
    assert type(s).__name__ == "DataStream" and s.node.maintain_sort_order is None
    _, j, _ = _join_actor(qc, s)
    assert type(j.obj).__name__ == "BuildProbeJoinExecutor"


def test_filters_pushed_below_keep_the_order(qc):
    q, d, _ = _small(qc)
    s = q.join(d, on="k", maintain_sort_order="left").filter_sql("v > 10")
    from quokka_b200.datastream import push_filters
    node = push_filters(s.node, [])
    assert node.kind == "join" and node.maintain_sort_order == "left" and node.parents[0].kind == "filter"


def test_explain_shows_the_order(qc, capsys):
    q, d, _ = _small(qc)
    s = q.join(d, on="k", maintain_sort_order="left")
    s.explain()
    assert "inner k=k keeps left order" in capsys.readouterr().out
    s.explain("physical")
    assert "OrderedJoinExecutor [ordered]" in capsys.readouterr().out


def test_shim_probe_orders_by_probe_row_then_build_row():
    t = cpu_shim.JoinTable(8, torch.device("cpu"))
    t.build(torch.tensor([5, 3, 5, 9], dtype=torch.int64))
    t.build(torch.tensor([5, 1], dtype=torch.int64))
    key = torch.tensor([5, 2, 9, 5], dtype=torch.int64)
    pi, bi = t.probe_ordered(key, L.JOIN_INNER)
    assert pi.tolist() == [0, 0, 0, 2, 3, 3, 3] and bi.tolist() == [0, 2, 4, 3, 0, 2, 4]
    pi, bi = t.probe_ordered(key, L.JOIN_LEFT)
    assert pi.tolist() == [0, 0, 0, 1, 2, 3, 3, 3] and bi.tolist() == [0, 2, 4, -1, 3, 0, 2, 4]
    assert t.probe_ordered(key, L.JOIN_SEMI)[0].tolist() == [0, 2, 3] and t.probe_ordered(key, L.JOIN_ANTI)[0].tolist() == [1]


def test_shim_place_puts_runs_into_left_order():
    # two senders: positions {1, 4, 4} and {0, 2, 2, 2}; one position's rows stay in arrival order
    pos = torch.tensor([1, 4, 4, 0, 2, 2, 2], dtype=torch.int32)
    src, left = cpu_shim.JoinTable.place(pos, 6)
    assert src.tolist() == [3, 0, 4, 5, 6, 1, 2] and left.tolist() == [0, 1, 2, 2, 2, 4, 4]
    with pytest.raises(L.QkError):
        S.join_place(torch.tensor([6], dtype=torch.int32), 6)


def test_no_cpu_fallback():
    from quokka_b200 import ops
    with pytest.raises(L.QkError, match="CUDA tensor"):
        ops.JoinTable.place(torch.zeros(3, dtype=torch.int32), 3)


@pytest.mark.parametrize("case", A.API_CASES, ids=lambda c: c.__name__)
def test_api_case(qc, case):
    case(qc)
