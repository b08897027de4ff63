"""DataStream.approximate_quantile on two gloo ranks (kernels replaced by tests/cpu_shim.py): each rank sketches its share of
the rows and the final phase merges the entries of both.  Both ranks must get the one-rank answer exactly: the numpy sketch of
all the rows, bit for bit."""
import ranks


def case_quantile_shares(qc):
    import pyarrow as pa
    import quantile_cases as QC
    cols = QC.special_columns(20_011, 17)
    names = list(cols)
    qs = [0.0, 0.1, 0.5, 0.9, 1.0]
    t = qc.from_arrow(pa.table(cols)).approximate_quantile(names, qs).collect()
    QC.assert_matches(t, names, qs, [cols[c] for c in names])


def test_quantile_two_ranks_gloo(tmp_path):
    ranks.spawn(tmp_path, 2, ranks.gloo_rank, ranks.SUITES["quantile"])
