"""DataStream.join(maintain_sort_order=...) on two gloo ranks (kernels replaced by tests/cpu_shim.py), with the build side
replicated and hash-partitioned: the ordered side stays on its rank, and the gathered result is the ordered join of the
collected inputs row for row -- string keys whose dictionaries differ by rank, fp64 keys, a rank without left or build rows,
and the ordered operators downstream without a re-sort."""
import ranks


def test_ordered_join_two_ranks_gloo(tmp_path):
    ranks.spawn(tmp_path, 2, ranks.gloo_rank, ranks.SUITES["ordered_join"])
