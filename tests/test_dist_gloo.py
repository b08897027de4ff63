"""world_size-2 runs of the SPMD driver and the all-to-all exchange on CPU (gloo), kernels replaced by
tests/cpu_shim.py: every rank must issue the same collectives, partitions must land on the rank that owns
the channel, dictionaries must be unified across ranks, and the results must equal the oracle."""
import os
import socket
import sys
import traceback

import pytest
import torch
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


class _Patch:
    def setattr(self, mod, name, value):
        setattr(mod, name, value)


def _worker(rank, world, port, case_names, out_dir):
    try:
        sys.path.insert(0, HERE)
        sys.path.insert(0, os.path.dirname(HERE))
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
        import torch.distributed as dist
        dist.init_process_group("gloo", rank=rank, world_size=world)
        import cpu_shim
        cpu_shim.install(_Patch())
        import api_cases as A
        from quokka_b200.df import QuokkaContext
        golden = os.path.join(HERE, "golden")
        calls = {}
        for name in case_names:
            qc = QuokkaContext()
            qc.set_config("broadcast_rows", 100)    # shuffle (and Bloom-reduce) every join even at test sizes
            qc.set_config("broadcast_cost_based", False)    # ... unless the case asks for cost-based replication ("cb:")
            if name.startswith("hash:"):            # as-of joins the reference's way: both streams hash-shuffled by symbol
                qc.set_config("asof_time_ranges", False)
                name = name[5:]
            if name.startswith("cb"):               # cost-based replication of build sides: "cb:" all that qualify,
                mode, name = name.split(":", 1)     # "cbmix:" only the small ones (Q3: customer replicated, orders shuffled)
                qc.set_config("broadcast_cost_based", True)
                if mode == "cbmix":
                    qc.set_config("broadcast_max_rows", 5000)
            if name == "bench_legs":                    # bench.py's multi-rank DataStream legs (strong / weak Q3, Q5, as-of)
                import test_bench_flow as TBF
                TBF.install(_Patch())
                TBF.run_multi_rank_legs(world, rank)
                continue
            if name.startswith("random_asof:"):         # streaming as-of joins in small batches, every rank drawing the same inputs
                import test_planner_random as TPR
                TPR.run_random_asof(qc, int(name.split(":")[1]), 15)
                continue
            if name.startswith("asof_rank_shards:"):    # per-rank shards of the sorted streams, cut independently (empty ranks too)
                import test_planner_random as TPR
                TPR.run_asof_rank_shards(qc, int(name.split(":")[1]))
                continue
            if name.startswith("random_programs:"):     # the planner's differential test, every rank drawing the same programs
                import test_planner_random as TPR
                TPR.run_random_programs(qc, int(name.split(":")[1]), int(os.environ.get("QK_PLANNER_TRIALS_DIST", "60")))
                continue
            fn = getattr(A, name)
            if name in ("case_join_kinds", "case_asof", "case_executor_protocol", "case_windows", "case_asof_reference_result"):
                fn(qc, golden)
            elif name in ("case_parquet_q1", "case_parquet_device", "case_csv_q1"):
                import pathlib
                d = pathlib.Path(out_dir) / f"files_{name}_{rank}"          # every rank writes and reads its own copy
                d.mkdir(exist_ok=True)
                fn(qc, d)
            else:
                fn(qc)
            if name == "case_q3":
                # both joins and the aggregate really shuffled
                assert qc.last_graph.exchange.calls > 0
                calls[qc.exec_config["broadcast_cost_based"], qc.exec_config["broadcast_max_rows"]] = qc.last_graph.exchange.calls
        if len(calls) > 1:                          # replicating a build side takes exchanges out of the plan
            base = calls[False, 1 << 26]
            assert all(v < base for k, v in calls.items() if k[0]), calls
        dist.barrier()
        dist.destroy_process_group()
        open(os.path.join(out_dir, f"ok{rank}"), "w").write("ok")
    except Exception:
        open(os.path.join(out_dir, f"fail{rank}"), "w").write(traceback.format_exc())
        raise


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
    _run_ranks(tmp_path, cases, 2)


def test_four_ranks_gloo_asof_time_ranges(tmp_path):
    """Four ranks: trades cross more than one range boundary, a rank's carried rows come from several earlier ranks, ranks in
    the middle are empty."""
    _run_ranks(tmp_path, ["asof_rank_shards:61", "hash:asof_rank_shards:62", "case_asof", "random_asof:63"], 4)


def _run_ranks(tmp_path, cases, world):
    port = _free_port()
    ctx = mp.get_context("spawn")
    procs = [ctx.Process(target=_worker, args=(r, world, port, cases, str(tmp_path))) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=600)
    fails = [open(os.path.join(tmp_path, f)).read() for f in os.listdir(tmp_path) if f.startswith("fail")]
    assert not fails, "\n".join(fails)
    assert all(os.path.exists(os.path.join(tmp_path, f"ok{r}")) for r in range(world)), [p.exitcode for p in procs]
