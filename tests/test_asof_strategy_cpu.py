"""OrderedStream.join_asof(strategy=..., tolerance=...) without a GPU: the numpy restatement against pandas.merge_asof, the
plan and explain(), and the API cases through the planner and the
executors on the shims."""
import datetime

import numpy as np
import pandas as pd
import pyarrow as pa
import pytest

import asof_strategy_api_cases as A
import asof_strategy_shim as S
import cpu_shim


@pytest.fixture
def qc(monkeypatch):
    cpu_shim.install(monkeypatch)
    from quokka_b200.df import QuokkaContext
    return QuokkaContext()


def _inputs(seed):
    """Heavy ties on both sides, duplicate (time, key) pairs, a key without right rows, left rows before the first and after
    the last right row."""
    rng = np.random.default_rng(seed)
    nl, nr, nk, span = int(rng.integers(0, 80)), int(rng.integers(0, 80)), int(rng.integers(1, 6)), int(rng.integers(1, 25))
    lt = np.sort(rng.integers(-3, span + 3, nl)).astype(np.int64)
    rt = np.sort(rng.integers(0, span, nr)).astype(np.int64)
    return lt, rng.integers(0, nk + 1, nl).astype(np.int64), rt, rng.integers(0, nk, nr).astype(np.int64)


@pytest.mark.parametrize("strategy", S.STRATEGIES)
@pytest.mark.parametrize("tolerance", [None, 0, 1, 4])
def test_restatement_is_pandas(strategy, tolerance):
    for seed in range(150):
        lt, lb, rt, rb = _inputs(seed)
        left = pd.DataFrame({"t": lt, "k": lb})
        right = pd.DataFrame({"t": rt, "k": rb, "j": np.arange(len(rt))})
        exp = pd.merge_asof(left, right, on="t", by="k", direction=strategy, tolerance=tolerance)["j"].fillna(-1).to_numpy(np.int64)
        assert np.array_equal(S.asof_join(lt, lb, rt, rb, strategy, tolerance), exp), seed


def test_documented_tie_examples():
    # right times 3, 7, 7 and left time 5 -> the row at 3; right times 7, 7, 13 and left time 7 -> the second 7
    assert S.asof_join([5], [0], [3, 7, 7], [0, 0, 0], "nearest").tolist() == [0]
    assert S.asof_join([7], [0], [7, 7, 13], [0, 0, 0], "nearest").tolist() == [1]
    assert S.asof_join([7], [0], [7, 7, 13], [0, 0, 0], "forward").tolist() == [0]
    assert S.asof_join([7], [0], [7, 7, 13], [0, 0, 0], "backward").tolist() == [1]


def test_plan_and_explain(qc, capsys):
    trades, quotes = A._tables(20, 20, 2, 10, 0)
    t, q = qc.from_arrow_sorted(trades, "time"), qc.from_arrow_sorted(quotes, "time")
    j = t.join_asof(q, on="time", by="symbol", strategy="nearest", tolerance=datetime.timedelta(milliseconds=5))
    assert j.schema == ["time", "symbol", "size", "it", "px", "iq"] and j.sorted_by == "time"
    assert j.schema == t.join_asof(q, on="time", by="symbol").schema
    j.explain()
    assert "strategy=nearest tolerance=0:00:00.005000" in capsys.readouterr().out
    g = qc.plan(j.node)
    ex = [a.obj for a in g.actors.values() if type(a.obj).__name__ == "SortedAsofExecutor"]
    assert len(ex) == 1 and ex[0].strategy == "nearest" and ex[0].silent_streams == "all"
    plain = [a.obj for a in qc.plan(t.join_asof(q, on="time", by="symbol").node).actors.values()
             if type(a.obj).__name__ == "SortedAsofExecutor"][0]
    assert plain.strategy == "backward" and plain.tolerance is None and plain.silent_streams == ()


def test_executor_keeps_the_reference_arguments():
    from quokka_b200.executors import SortedAsofExecutor
    ex = SortedAsofExecutor("time", "time", "symbol", "symbol", "_r")
    assert (ex.strategy, ex.tolerance, ex.suffix) == ("backward", None, "_r")
    with pytest.raises(ValueError):
        SortedAsofExecutor(strategy="sideways")


@pytest.mark.parametrize("case", A.API_CASES, ids=lambda f: f.__name__)
def test_api_case(qc, case, golden_dir):
    import inspect
    args = {"qc": qc, "golden_dir": golden_dir}
    case(*[args[p] for p in inspect.signature(case).parameters])
