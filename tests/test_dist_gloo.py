"""world_size-2 runs of the SPMD driver and the all-to-all exchange on CPU (gloo), kernels replaced by
tests/cpu_shim.py: every rank must issue the same collectives, partitions must land on the rank that owns
the channel, dictionaries must be unified across ranks, and the results must equal the oracle.  The case names
are those of tests/ranks.py run_case."""
import pytest

import ranks


@pytest.mark.parametrize("cases", [["case_q1_sql", "case_q1_dict_api", "case_q3"], ["case_q5", "case_join_kinds"],
                                   ["case_q3", "cb:case_q3", "cbmix:case_q3", "cb:case_q5", "cbmix:case_q10_q18", "cb:case_join_kinds"],
                                   ["case_parquet_q1", "case_parquet_device", "case_csv_q1"],
                                   ["random_programs:33", "random_asof:35"],
                                   ["random_programs:31", "cb:random_programs:32", "random_asof:34", "bench_legs"],
                                   ["hash:case_asof", "hash:random_asof:36", "hash:case_asof_reference_result", "asof_rank_shards:41", "hash:asof_rank_shards:42"],
                                   ["case_q9_q11_q13", "case_q15_q16_q20_q22", "case_q2_q21", "case_string_funcs_and_nulls"],
                                   ["case_asof", "case_executor_protocol", "case_misc_ops", "case_scalar_aggs", "case_q6_and_semi_anti", "case_q10_q18", "case_case_like_extract", "case_custom_host_executor", "case_q14_q17_q19", "case_q4_q12",
                                    "case_string_key_join", "case_agg_types", "case_windows", "case_asof_reference_result", "case_q7_q8"]])
def test_two_ranks_gloo(tmp_path, cases):
    ranks.spawn(tmp_path, 2, ranks.gloo_rank, cases)


def test_four_ranks_gloo_asof_time_ranges(tmp_path):
    """Four ranks: trades cross more than one range boundary, a rank's carried rows come from several earlier ranks, ranks in
    the middle are empty."""
    ranks.spawn(tmp_path, 4, ranks.gloo_rank, ["asof_rank_shards:61", "hash:asof_rank_shards:62", "case_asof", "random_asof:63"])

