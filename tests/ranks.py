"""The multi-rank harness of the suite: gloo ranks on CPU (spawn + gloo_rank, kernels replaced by tests/cpu_shim.py), NCCL
ranks on GPUs (torchrun + tests/dist_nccl_check.py), and the named cases both of them run (run_cases).  Not collected by
pytest: the tests import it."""
import importlib
import inspect
import os
import pathlib
import re
import signal
import socket
import subprocess
import sys
import time
import traceback

import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden")

# the case lists that the gloo test of a feature, dist_nccl_check.py's arguments and the in-process runs
# (tests/inproc_link.py run_program_ranks) share
SUITES = {
    "api": ["case_q1_sql", "case_q1_dict_api", "case_q3", "case_q5", "case_join_kinds", "case_asof", "case_executor_protocol",
            "case_misc_ops", "case_scalar_aggs", "case_string_key_join", "case_agg_types", "case_windows", "case_asof_reference_result"],
    "--more": ["case_q6_and_semi_anti", "case_q10_q18", "case_q4_q12", "case_q14_q17_q19", "case_case_like_extract", "case_q7_q8",
               "case_custom_host_executor", "cb:case_q3", "cb:case_q5", "cbmix:case_q3", "cbmix:case_q10_q18", "case_q9_q11_q13",
               "case_q15_q16_q20_q22", "case_q2_q21", "case_string_funcs_and_nulls", "hash:case_asof", "asof_rank_shards:51",
               "hash:asof_rank_shards:52"],
    "sort": ["sort_api_cases:" + c for c in ("case_sort_ranges", "case_sort_collect", "case_sort_select_filter_keep_order",
                                             "case_sort_nulls_from_left_join", "case_sort_then_asof", "case_sort_then_window",
                                             "case_sort_then_pattern", "case_sort_then_quantile_and_gram")],
    "shift": ["shift_api_cases:" + c for c in ("case_shift_lag_lead", "case_shift_in_place", "case_shift_fills",
                                               "case_shift_nulls_from_left_join", "case_sort_then_shift", "case_shift_then_asof",
                                               "case_shift_out_of_order")],
    "knn": ["knn_cases:" + c for c in ("case_vector_roundtrip", "case_vector_ops", "case_knn_api", "case_knn_fewer_rows")],
    "pattern": ["pattern_cases:API_CASES"],
    "ordered_join": ["ordered_join_api_cases:API_CASES"],
    "asof_strategy": ["asof_strategy_api_cases:API_CASES"],
    "gram": ["test_dist_gloo_gram:case_gram_shares", "test_dist_gloo_gram:case_gram_device_batches", "gram_cases:case_gram_filtered_ints",
             "gram_cases:case_gram_empty"],
    "quantile": ["test_dist_gloo_quantile:case_quantile_shares", "quantile_cases:case_quantile_tpch_606", "quantile_cases:case_quantile_empty"],
}
NCCL_MARKER = "DIST_NCCL_OK"
_API_PREFIXES = ("hash", "cb", "cbmix", "random_programs", "random_asof", "asof_rank_shards")


def free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


class Patch:
    """The `setattr(obj, name, value)` of pytest's monkeypatch, without the undo: a rank process keeps what it installs."""

    def setattr(self, obj, name, value):
        setattr(obj, name, value)


def expand(names):
    """The case names one by one: `<module>:<LIST>` (an upper-case name, e.g. pattern_cases:API_CASES) stands for
    `<module>:<function>` of every function in that list."""
    out = []
    for name in names:
        head, _, attr = name.partition(":")
        if attr.isupper():
            out += [f"{head}:{fn.__name__}" for fn in getattr(importlib.import_module(head), attr)]
        else:
            out.append(name)
    return out


def _call(fn, qc, rank, files_dir):
    """fn with its parameters without a default filled by name: qc, golden_dir (tests/golden), tmpdir (a directory of this
    rank's own under files_dir)."""
    args = []
    for p in inspect.signature(fn).parameters.values():
        if p.default is not p.empty:
            break
        if p.name == "tmpdir":
            d = pathlib.Path(files_dir) / f"files_{fn.__name__}_{rank}"
            d.mkdir(exist_ok=True)
            args.append(d)
        else:
            args.append({"qc": qc, "golden_dir": GOLDEN}[p.name])
    fn(*args)


def run_case(name, rank, world, files_dir):
    """Runs one named case on this rank and returns its QuokkaContext.  A name is
      <module>:<function>     a case function of a tests module, on a default context;
      <function>              api_cases.<function>, on a context that shuffles (and Bloom-reduces) every join even at test
                              sizes, and so are the rest:
      hash:<name>             as-of joins the reference's way: both streams hash-shuffled by symbol;
      cb:<name>, cbmix:<name> cost-based replication of build sides: all that qualify / only the small ones (Q3: customer
                              replicated, orders shuffled);
      random_programs:<seed>  the planner's differential test, every rank drawing the same programs;
      random_asof:<seed>      streaming as-of joins in small batches, every rank drawing the same inputs;
      asof_rank_shards:<seed> per-rank shards of the sorted streams, cut independently (empty ranks too);
      bench_legs              bench.py's multi-rank DataStream legs (strong / weak Q3, Q5, as-of) on the CPU shim."""
    from quokka_b200.df import QuokkaContext
    qc = QuokkaContext()
    head, _, rest = name.partition(":")
    if rest and head not in _API_PREFIXES:
        _call(getattr(importlib.import_module(head), rest), qc, rank, files_dir)
        return qc
    qc.set_config("broadcast_rows", 100)
    qc.set_config("broadcast_cost_based", False)
    if name.startswith("hash:"):
        qc.set_config("asof_time_ranges", False)
        name = name[5:]
    if name.startswith("cb"):
        mode, name = name.split(":", 1)
        qc.set_config("broadcast_cost_based", True)
        if mode == "cbmix":
            qc.set_config("broadcast_max_rows", 5000)
    runner, _, seed = name.partition(":")
    if name == "bench_legs":
        import test_bench_flow as TBF
        TBF.install(Patch())
        TBF.run_multi_rank_legs(world, rank)
    elif runner == "random_programs":
        import test_planner_random as TPR
        TPR.run_random_programs(qc, int(seed), int(os.environ.get("QK_PLANNER_TRIALS_DIST", "60")))
    elif runner == "random_asof":
        import test_planner_random as TPR
        TPR.run_random_asof(qc, int(seed), 15)
    elif runner == "asof_rank_shards":
        import test_planner_random as TPR
        TPR.run_asof_rank_shards(qc, int(seed))
    else:
        import api_cases
        _call(getattr(api_cases, name), qc, rank, files_dir)
    return qc


def run_cases(names, rank, world, files_dir):
    """run_case for every case of `names`; rank 0 prints `<case>: ok` after each.  Q3 must shuffle, and replicating its build
    sides must take exchanges out of its plan."""
    calls = {}
    for name in expand(names):
        qc = run_case(name, rank, world, files_dir)
        g = qc.last_graph
        if name.rpartition(":")[2] == "case_q3":
            assert g.exchange.calls > 0, name
            calls[qc.exec_config["broadcast_cost_based"], qc.exec_config["broadcast_max_rows"]] = g.exchange.calls
        if rank == 0:
            print(f"{name}: ok  (exchange calls {g.exchange.calls if g else 0}, via peer memory {g.exchange.peer_calls if g else 0}, "
                  f"bytes sent by rank 0 {g.exchange.bytes_sent if g else 0})", flush=True)
    if len(calls) > 1:
        base = calls[False, 1 << 26]
        assert all(v < base for k, v in calls.items() if k[0]), calls


def gloo_rank(rank, world, port, out_dir, names):
    """One rank of `spawn` on gloo, the kernels replaced by tests/cpu_shim.py: run_cases(names)."""
    try:
        sys.path.insert(0, HERE)
        sys.path.insert(0, os.path.dirname(HERE))
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
        import torch.distributed as dist
        dist.init_process_group("gloo", rank=rank, world_size=world)
        import cpu_shim
        cpu_shim.install(Patch())
        run_cases(names, rank, world, out_dir)
        dist.barrier()
        dist.destroy_process_group()
        open(os.path.join(out_dir, f"ok{rank}"), "w").write("ok")
    except Exception:
        open(os.path.join(out_dir, f"fail{rank}"), "w").write(traceback.format_exc())
        raise


def spawn(tmp_path, world, target, *args, timeout=600):
    """target(rank, world, port, out_dir, *args) in `world` spawn-context processes, out_dir = tmp_path.  Waits at most
    `timeout` seconds for all of them, then terminates any rank still alive and fails naming it; otherwise fails with what a
    rank wrote to `fail<rank>`, or when a rank left no `ok<rank>`."""
    port = free_port()
    ctx = mp.get_context("spawn")
    procs = [ctx.Process(target=target, args=(r, world, port, str(tmp_path), *args)) for r in range(world)]
    for p in procs:
        p.start()
    deadline = time.monotonic() + timeout
    for p in procs:
        p.join(max(0.0, deadline - time.monotonic()))
    hung = [r for r, p in enumerate(procs) if p.is_alive()]
    for r in hung:
        procs[r].terminate()
        procs[r].join(10)
        if procs[r].is_alive():
            procs[r].kill()
            procs[r].join()
    assert not hung, f"rank(s) {hung} still running after {timeout} s; terminated"
    fails = [open(os.path.join(tmp_path, f)).read() for f in sorted(os.listdir(tmp_path)) if f.startswith("fail")]
    assert not fails, "\n".join(fails)
    assert all(os.path.exists(os.path.join(tmp_path, f"ok{r}")) for r in range(world)), [p.exitcode for p in procs]


def _children(pid):
    kids = []
    for d in os.listdir("/proc"):
        try:
            if d.isdigit() and int(open(f"/proc/{d}/stat").read().rsplit(")", 1)[1].split()[1]) == pid:
                kids.append(int(d))
        except OSError:
            pass
    return kids


def torchrun(script, nproc, env=None, args=(), timeout=600):
    """(exit code, output) of tests/<script> on `nproc` local ranks under torch.distributed.run.  It runs in a session of its
    own; on timeout its process group is killed, and so is the group of every rank, which torchrun starts in a session of
    its own."""
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}", "--master-addr", "127.0.0.1",
           "--master-port", str(free_port()), os.path.join(HERE, script), *args]
    p = subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, env={**os.environ, **(env or {})},
                         start_new_session=True)
    try:
        out, _ = p.communicate(timeout=timeout)
    except subprocess.TimeoutExpired:
        for group in [p.pid, *_children(p.pid)]:
            try:
                os.killpg(group, signal.SIGKILL)
            except OSError:
                pass
        out, _ = p.communicate()
        out += f"\n[killed after {timeout} s]".encode()
    return p.returncode, out.decode(errors="replace")


def nccl_suites(*suites, nproc=2):
    """tests/dist_nccl_check.py over the named suites on `nproc` GPUs: it must exit 0, print its final marker, and print
    `<case>: ok` for every case of the suites."""
    rc, out = torchrun("dist_nccl_check.py", nproc, args=suites)
    assert rc == 0 and NCCL_MARKER in out, out[-4000:]
    missing = [n for n in expand(n for s in suites for n in SUITES[s]) if not re.search(f"^{re.escape(n)}: ok", out, re.M)]
    assert not missing, f"no ok line for {missing}\n{out[-4000:]}"
