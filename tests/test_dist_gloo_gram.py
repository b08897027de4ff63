"""DataStream.gramian / covariance on two gloo ranks (kernels replaced by tests/cpu_shim.py): each rank folds its share of the
rows with its own shift, and the final phase re-centres the partials on the global mean.  Both ranks must get the one-rank
result within the summation bound of tests/gram_cases.py."""
import numpy as np

import ranks


def case_gram_shares(qc):
    import pyarrow as pa
    import gram_cases as GC
    rng = np.random.default_rng(17)
    n = 20_011
    cols = {"a": rng.normal(3e4, 5.0, n), "b": rng.integers(-1000, 1000, n).astype(np.int64),
            "c": rng.normal(-2.0, 1e-3, n).astype(np.float32), "d": rng.normal(0, 1e6, n)}
    names = list(cols)
    x = np.stack([cols[c].astype(np.float64) for c in names], axis=1)
    d = qc.from_arrow(pa.table(cols))
    g, b = GC.gram_ref(x)
    GC.assert_within(GC.table_matrix(d.gramian(names).collect(), names), g, b, "gramian")
    shift = x.mean(axis=0)
    g, b = GC.gram_ref(x, shift)
    GC.assert_within(GC.table_matrix(d.gramian(names, demean=shift).collect(), names), g, b, "gramian demean")
    c, b = GC.cov_ref(x)
    GC.assert_within(GC.table_matrix(d.covariance(names), names), c, b, "covariance")


def case_gram_device_batches(qc):
    """Every rank reads its own share of the rows from the device in batches of 997 rows: a re-entrant reader with many
    rounds, which runs on the pipeline lanes where there is a device and a peer-memory link."""
    from quokka_b200 import runtime
    from quokka_b200.columns import DeviceTable
    import gram_cases as GC
    rng = np.random.default_rng(23)
    n = 20_011
    cols = {"a": rng.normal(-7e3, 2.0, n), "b": rng.integers(-1 << 20, 1 << 20, n).astype(np.int64),
            "c": rng.normal(0.5, 1e-2, n).astype(np.float32)}
    names = list(cols)
    w, me = runtime.world_size(), runtime.rank()
    lo, hi = n * me // w, n * (me + 1) // w
    d = qc.from_device(DeviceTable.from_numpy({c: np.ascontiguousarray(v[lo:hi]) for c, v in cols.items()}), batch_rows=997)
    x = np.stack([cols[c].astype(np.float64) for c in names], axis=1)
    g, b = GC.gram_ref(x)
    GC.assert_within(GC.table_matrix(d.gramian(names).collect(), names), g, b, "gramian of device batches")
    c, b = GC.cov_ref(x)
    GC.assert_within(GC.table_matrix(d.covariance(names), names), c, b, "covariance of device batches")


def test_gram_two_ranks_gloo(tmp_path):
    ranks.spawn(tmp_path, 2, ranks.gloo_rank, ranks.SUITES["gram"])
