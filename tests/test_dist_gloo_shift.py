"""OrderedStream.shift on two gloo ranks (kernels replaced by tests/cpu_shim.py): range-partitioned input
from from_arrow_sorted and from sort(), keys straddling the ranks' boundary and keys with fewer than |n| rows on each rank, lag
and lead, by=None; the gathered result equals the one-rank answer row for row, and ranks holding out-of-order ranges raise."""
import ranks


def test_shift_two_ranks_gloo(tmp_path):
    ranks.spawn(tmp_path, 2, ranks.gloo_rank, ranks.SUITES["shift"])
