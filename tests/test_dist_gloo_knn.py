"""Vector columns and DataStream.vector_nn_join on two gloo ranks (kernels replaced by tests/cpu_shim.py): every
rank reads its share of the rows, the per-rank candidates cross the broadcast edge with their vector column, and collect() gathers
vectors to every rank.  Each rank must get the one-rank result."""
import ranks


def test_knn_two_ranks_gloo(tmp_path):
    ranks.spawn(tmp_path, 2, ranks.gloo_rank, ranks.SUITES["knn"])
