"""Per-event tumbling and session windows on two gloo ranks (kernels replaced by tests/cpu_shim.py and tests/window_events_shim.py): each rank windows the keys
it owns, and the collected rows equal the reference's on the whole input, row set for row set."""
import ranks
import window_events_cases as A


def test_window_events_two_ranks_gloo(tmp_path):
    ranks.spawn(tmp_path, 2, ranks.gloo_rank, A.SUITE)
