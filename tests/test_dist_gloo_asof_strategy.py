"""OrderedStream.join_asof(strategy=..., tolerance=...) on two gloo ranks (kernels replaced by tests/cpu_shim.py and
tests/asof_strategy_shim.py): the time-range plan with equal quote times straddling the boundary, a gap, ranks without quotes
or trades and a symbol quoted only on the later rank; the hash-partitioned plan; the search path; every rank collects the
global join."""
import ranks


def test_asof_strategy_two_ranks_gloo(tmp_path):
    ranks.spawn(tmp_path, 2, ranks.gloo_rank, ranks.SUITES["asof_strategy"])
