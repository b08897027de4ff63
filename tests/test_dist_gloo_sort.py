"""DataStream.sort on two gloo ranks (kernels replaced by tests/cpu_shim.py): the sample sort leaves rank r
with the r-th range of the first sort column, the gathered result equals the one-rank answer row for row, and a sorted stream
feeds join_asof (over the ranks' time ranges), windowed_transform, pattern_recognize, approximate_quantile and gramian."""
import ranks


def test_sort_two_ranks_gloo(tmp_path):
    ranks.spawn(tmp_path, 2, ranks.gloo_rank, ranks.SUITES["sort"])
