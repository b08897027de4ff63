"""OrderedStream.pattern_recognize on two gloo ranks (kernels replaced by tests/cpu_shim.py): every rank
reads its share of the sorted rows, the hash edge by key brings each key's rows to one channel, and collect() gathers the matches
to every rank.  Each rank must get the one-rank result of the API cases."""
import ranks


def test_pattern_two_ranks_gloo(tmp_path):
    ranks.spawn(tmp_path, 2, ranks.gloo_rank, ranks.SUITES["pattern"])
