"""The multi-rank DataStream suites on ONE GPU: tests/inproc_link.py run_program_ranks runs W virtual ranks in threads of this
process, on the kernels, over the in-process peer-memory link (csrc/exchange.cu), with mailboxes that hold every exchange
(64 MB) and with 1 MB mailboxes, where the larger exchanges go in rounds.  So the kernels see what only several ranks produce:
the owners' matches that qk_join_place puts back in order, as-of carry tables built on other ranks, the boundary rows of a
shift, rows a sample sort received from several ranks, per-rank top-k lists and sketch entries to merge, and chunks on the
pipeline lanes.  Every case checks what each rank gathers against oracle/ or pandas; the counters of run_program_ranks show
that the multi-rank paths ran."""
import time

import pytest

import inproc_link as IL
import ranks

pytestmark = pytest.mark.gpu

MB = 1 << 20
SUITES = ["api", "--more", "sort", "shift", "knn", "pattern", "ordered_join", "asof_strategy", "gram", "quantile"]


def _run(world, names, mailbox_mb):
    t0 = time.perf_counter()
    counts = IL.run_program_ranks(world, names, "cuda", mailbox_mb * MB)
    print(f"world {world}, mailbox {mailbox_mb} MB: {time.perf_counter() - t0:.1f} s, {dict(sorted(counts.items()))}")
    return counts


@pytest.mark.parametrize("mailbox_mb", [64, 1], ids=lambda m: f"{m}MB")
@pytest.mark.parametrize("world", [2, 3], ids=lambda w: f"world{w}")
@pytest.mark.parametrize("suite", SUITES)
def test_suite_on_inproc_ranks(suite, world, mailbox_mb):
    # `--more` compares Q3's exchange count under cost-based replication with the shuffled plan's, which `api` runs
    counts = _run(world, (["case_q3"] if suite == "--more" else []) + ranks.SUITES[suite], mailbox_mb)
    missing = [k for k in IL.REACHES.get(suite, ()) if counts[k] == 0]
    assert not missing, (suite, dict(counts))
    if mailbox_mb == 1 and suite in IL.IN_ROUNDS_AT_1MB:
        assert counts["exchange_rounds"] > 0, dict(counts)
    if suite == "--more" and world == 3:        # the customers without orders (c_custkey % 3 == 0) all hash to rank 0,
        # which owns no orders: case_string_funcs_and_nulls' left join keeps them with NULL order columns
        assert counts["left_template"] > 0, dict(counts)
    if suite == "gram":             # case_gram_device_batches: a re-entrant reader with many rounds runs on the lanes
        assert counts["lanes_used"] >= 2, dict(counts)


def test_four_inproc_ranks_asof_time_ranges():
    """Four ranks: trades cross more than one range boundary, carried rows come from several earlier ranks, ranks in the
    middle hold nothing."""
    counts = _run(4, ["asof_rank_shards:61", "hash:asof_rank_shards:62", "case_asof"], 64)
    assert counts["asof_carry"] > 0, dict(counts)
