"""The operator API against the real sm_90a kernels (same cases as tests/test_api_cpu.py)."""
import pytest

import api_cases as A

pytestmark = pytest.mark.gpu


@pytest.fixture
def qc():
    from quokka_b200.df import QuokkaContext
    return QuokkaContext()


def test_q1_sql(qc):
    A.case_q1_sql(qc)
    # the partial aggregate of Q1 must have gone through the fused TMA kernel, not the interpreter
    from quokka_b200 import ops
    assert ops.launch_count() > 0


def test_q1_dict_api(qc): A.case_q1_dict_api(qc)
def test_q3(qc): A.case_q3(qc)
def test_q5(qc): A.case_q5(qc)
def test_join_kinds(qc, golden_dir): A.case_join_kinds(qc, golden_dir)
@pytest.mark.parametrize("tag", ["0", "1", "2"])
def test_asof(qc, golden_dir, tag): A.case_asof(qc, golden_dir, tag)
def test_asof_reference_result(qc, golden_dir): A.case_asof_reference_result(qc, golden_dir)
def test_windows(qc, golden_dir): A.case_windows(qc, golden_dir)
def test_parquet_q1(qc, tmp_path): A.case_parquet_q1(qc, tmp_path)
def test_misc_ops(qc): A.case_misc_ops(qc)
def test_scalar_aggs(qc): A.case_scalar_aggs(qc)
def test_string_key_join(qc): A.case_string_key_join(qc)
def test_agg_types(qc): A.case_agg_types(qc)
def test_count_distinct_and_writer(qc, tmp_path): A.case_count_distinct_and_writer(qc, tmp_path)
def test_executor_protocol(qc, golden_dir): A.case_executor_protocol(qc, golden_dir)


def test_q1_from_pinned_host_columns(qc):
    """The end-to-end path of bench.py: pinned host columns -> chunked, double-buffered H2D -> fused kernel."""
    import numpy as np
    import torch
    from oracle import tpch_gen as G
    li = G.gen_lineitem(A.SF)
    names = ["l_shipdate", "l_returnflag", "l_linestatus", "l_quantity", "l_extendedprice", "l_discount", "l_tax"]
    host = {n: torch.from_numpy(np.ascontiguousarray(li[n])).pin_memory() for n in names}
    s = qc.from_pinned(host, dictionaries={"l_returnflag": G.RETURNFLAG_DICT, "l_linestatus": G.LINESTATUS_DICT},
                       dates=("l_shipdate",), chunk_rows=7_001)                      # 9 ragged chunks
    f = s.filter_sql("l_shipdate <= date '1998-12-01' - interval '90' day").groupby(["l_returnflag", "l_linestatus"]).agg_sql("""
        sum(l_quantity) as sum_qty, sum(l_extendedprice) as sum_base_price,
        sum(l_extendedprice * (1 - l_discount)) as sum_disc_price,
        sum(l_extendedprice * (1 - l_discount) * (1 + l_tax)) as sum_charge,
        avg(l_quantity) as avg_qty, avg(l_extendedprice) as avg_price, avg(l_discount) as avg_disc,
        count(*) as count_order""")
    A.check_q1(f.collect())
    A.check_q1(f.collect())        # the stream can be collected again (fresh staging state)
