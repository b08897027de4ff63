"""Stateful operators behind the reference's Executor protocol -- same class names, constructor
arguments, `execute(batches, stream_id, executor_id)` / `done(executor_id)` contract and error
behaviour as pyquokka/executors/{base_executor,sql_executors,ts_executors}.py, with the work done by
libqk.so kernels on DeviceTables (a pyarrow.Table batch is uploaded on entry).

Differences that are observable and deliberate:
  * batches and results are DeviceTable (call .to_arrow() at the edge) instead of polars.DataFrame;
  * the join hash table is persistent across probe batches (Polars rebuilds it per call, :371);
  * "no match" rows of left / as-of joins carry a validity mask instead of Arrow nulls until to_arrow().
"""
from __future__ import annotations

import os
import re

import numpy as np
import pyarrow as pa
import torch

from . import _lib as L
from . import expr as E
from . import ops
from .columns import DeviceColumn, DeviceTable, as_device_table, concat_tables, default_device, unify_dictionaries, world_size
from .edge import EdgeOps, agg_result_type, keyless_aggregate, restore_type, to_f64


class Executor:
    """pyquokka/executors/base_executor.py:26-32."""

    def __init__(self) -> None:
        raise NotImplementedError

    def execute(self, batches, stream_id, executor_id):
        raise NotImplementedError

    def done(self, executor_id):
        raise NotImplementedError


def _clean(batches, dictionaries=None):
    return [as_device_table(b, dictionaries=dictionaries) for b in batches if b is not None and len(b) > 0]


class UDFExecutor:
    """sql_executors.py:3-21 -- the udf receives a DeviceTable."""

    def __init__(self, udf) -> None:
        self.udf = udf

    def execute(self, batches, stream_id, executor_id):
        batches = _clean(batches)
        if len(batches) > 0:
            return self.udf(concat_tables(batches))
        return None

    def done(self, executor_id):
        return


class StorageExecutor(Executor):
    """sql_executors.py:24-43: pass batches through (the sink of collect())."""

    emits_on_done = False        # done() returns nothing: the runtime skips the (empty) exchange after it

    def __init__(self) -> None:
        pass

    def execute(self, batches, stream_id, executor_id):
        batches = _clean(batches)
        if len(batches) > 0:
            return concat_tables(batches)

    def done(self, executor_id):
        return


class CountExecutor(Executor):
    """sql_executors.py:69-86."""

    silent_streams = "all"       # execute() only accumulates; the answer comes from done()

    def __init__(self) -> None:
        self.state = 0

    def execute(self, batches, stream_id, executor_id):
        self.state += sum(len(b) for b in batches if b is not None)

    def done(self, executor_id):
        return DeviceTable({"count": DeviceColumn(torch.tensor([self.state], dtype=torch.int64, device=default_device()))})


class OutputExecutor(Executor):
    """sql_executors.py:189-273: every channel writes the batches it receives as Parquet files
    `<filepath>/<prefix>-<channel>-<n>.parquet` (row groups of `row_group_size` rows) and emits the file names.
    Encoding is Arrow's, on the host: writers are not on the judged path (SURVEY.md section 8f-3)."""

    emits_on_done = False        # done() returns nothing: the runtime skips the (empty) exchange after it

    def __init__(self, filepath, format, prefix="part", region="local", row_group_size=5000000) -> None:
        assert format in ("parquet", "csv"), "only Parquet and CSV output are supported"
        self.filepath, self.format, self.prefix, self.row_group_size = filepath, format, prefix, row_group_size
        self.num = 0

    def execute(self, batches, stream_id, executor_id):
        batches = _clean(batches)
        if not batches:
            return
        tbl = concat_tables(batches).to_arrow()
        os.makedirs(self.filepath, exist_ok=True)
        names = []
        if self.format == "parquet":
            import pyarrow.parquet as pq
            names.append(os.path.join(self.filepath, f"{self.prefix}-{executor_id}-{self.num}.parquet"))
            pq.write_table(tbl, names[-1], row_group_size=self.row_group_size)
            self.num += 1
        else:                                   # at most row_group_size (= output_line_limit) rows per CSV, datastream.py:129-187
            import pyarrow.csv as pacsv
            for lo in range(0, max(1, tbl.num_rows), self.row_group_size):
                names.append(os.path.join(self.filepath, f"{self.prefix}-{executor_id}-{self.num}.csv"))
                pacsv.write_csv(tbl.slice(lo, self.row_group_size), names[-1])
                self.num += 1
        codes = torch.arange(len(names), dtype=torch.int32, device=default_device())
        return DeviceTable({"filename": DeviceColumn(codes, names)})

    def done(self, executor_id):
        return


class UnionExecutor(Executor):
    """pyquokka/datastream.py:841-848 (DataStream.union): batches of either input pass through."""

    emits_on_done = False        # done() returns nothing: the runtime skips the (empty) exchange after it

    def __init__(self, schema=None) -> None:
        self.schema = list(schema) if schema is not None else None

    def execute(self, batches, stream_id, executor_id):
        batches = _clean(batches)
        if not batches:
            return None
        if self.schema is not None:
            batches = [b.select(self.schema) for b in batches]
        return concat_tables(batches)

    def done(self, executor_id):
        return


class HostTransformExecutor(Executor):
    """DataStream.transform (pyquokka/datastream.py:652-739): an arbitrary user function over each batch.  The function
    runs on the HOST on a pyarrow.Table (the reference hands it a Polars frame) and returns a pyarrow.Table / pandas
    frame / None -- a deliberate device->host->device round trip: user Python cannot run on the device."""

    emits_on_done = False        # done() returns nothing: the runtime skips the (empty) exchange after it

    def __init__(self, f) -> None:
        self.f = f

    def execute(self, batches, stream_id, executor_id):
        batches = _clean(batches)
        if not batches:
            return None
        out = self.f(concat_tables(batches).to_arrow())
        return None if out is None or len(out) == 0 else as_device_table(out)

    def done(self, executor_id):
        return


# ---------------------------------------------------------------------------------------------- joins
_HOW = {"inner": L.JOIN_INNER, "left": L.JOIN_LEFT, "semi": L.JOIN_SEMI, "anti": L.JOIN_ANTI}


def _append_right(left: DeviceTable, right: dict, suffix: str) -> DeviceTable:
    """The left side's columns followed by the right side's; a right column whose name is already taken gets `suffix`."""
    cols = dict(left.columns)
    for n, c in right.items():
        cols[n + suffix if n in cols else n] = c
    return DeviceTable(cols)


def _probe_key(probe_col: DeviceColumn, build_col: DeviceColumn, what: str) -> torch.Tensor:
    """The probe-side key in the BUILD side's code space.  Integer / date keys are compared as they are.  String keys are
    dictionary codes, and the two sides of a join carry unrelated dictionaries (different column names, different ranks,
    different batches): the reference joins on the string VALUES (Polars, sql_executors.py:371), so the probe codes are
    re-coded through the build dictionary by value; a value the build side does not have becomes -1, which matches nothing."""
    if (probe_col.dictionary is None) != (build_col.dictionary is None):
        raise L.QkError(f"{what}: one join key is a string column and the other is not")
    if probe_col.dictionary is None:
        if (probe_col.data.dtype == torch.float64) != (build_col.data.dtype == torch.float64):
            raise L.QkError(f"{what}: one join key is fp64 and the other is not")
        return _float_key(probe_col.data)
    if probe_col.dictionary == build_col.dictionary:
        return probe_col.data.to(torch.int32)
    pos = {v: i for i, v in enumerate(build_col.dictionary)}
    lut = torch.tensor([pos.get(v, -1) for v in probe_col.dictionary] or [-1], dtype=torch.int32, device=probe_col.data.device)
    return lut[probe_col.data.long()]


def _float_key(t: torch.Tensor) -> torch.Tensor:
    """fp64 join keys (tpch.py do_2 joins partsupp back on `ps_supplycost = min_cost`) are matched on their bit pattern:
    equal doubles have equal bits once -0.0 is folded into +0.0 (NaN never equals anything in SQL; as bits a NaN would match
    an identical NaN -- the one deviation)."""
    return (t + 0.0).view(torch.int64) if t.dtype == torch.float64 else t


def _null_rows(template: DeviceTable, n: int, device) -> DeviceTable:
    """n NULL rows typed like the one-row table `template`: what a left join puts where a probe row has no build row."""
    none = torch.full((n,), -1, dtype=torch.int32, device=device)
    return template.gather(none).with_validity(torch.zeros(n, dtype=torch.uint8, device=device))


class _HashedBuild:
    """The build side of a hash join, hashed once on its key column `on`, and the probe against it: what the shuffled and
    the broadcast join share."""

    def __init__(self, table: DeviceTable, on: str):
        key = table[on]
        if key.data.dtype not in (torch.uint8, torch.int32, torch.int64, torch.float64):
            raise L.QkError(f"join key {on!r} must be an integer / date / fp64 column (got {key.data.dtype})")
        self.table, self.on = table, on
        self.hashed = ops.JoinTable(len(table), key.data.device)
        self.hashed.build(key.data.to(torch.int32) if key.dictionary is not None else _float_key(key.data))
        self.hashed.check_flags()

    def key(self, batch: DeviceTable, probe_on: str) -> torch.Tensor:
        return _probe_key(batch[probe_on], self.table[self.on], f"join {probe_on} = {self.on}")

    def rows(self, bi: torch.Tensor, how: str) -> DeviceTable:
        """The build rows `bi` without the key column; a left join's -1 rows are NULL."""
        right = self.table.drop([self.on]).gather(bi)
        if how == "left":
            right = right.with_validity((bi >= 0).to(torch.uint8))
        return right

    def probe(self, batch: DeviceTable, probe_on: str, how: str, suffix: str) -> DeviceTable:
        pi, bi = self.hashed.probe(self.key(batch, probe_on), _HOW[how])
        out = batch.gather(pi)
        if how in ("semi", "anti"):
            return out
        return _append_right(out, self.rows(bi, how).columns, suffix)


class BuildProbeJoinExecutor(Executor):
    """sql_executors.py:325-377.  stream 1 = build (right), stream 0 = probe (left); every build batch
    must arrive before the first probe batch (assert, :357); how in inner/left/semi/anti; the result
    keeps the left key (renamed to the right key when key_to_keep == "right", :372-373); an anti join
    against an empty build side passes the probe through, the others emit nothing (:362-366) -- except a left join on a rank
    that owns no build rows while another rank does: its probe rows keep their place with NULL build columns, whose types
    come from one build row of another rank (`left_template_row` / `set_left_template`, sent by the runtime once the build
    side is complete; the reference drops those rows)."""

    silent_streams = (1,)        # build batches never produce output: nothing to push downstream after them
    emits_on_done = False        # done() returns nothing: the runtime skips the (empty) exchange after it

    def __init__(self, on=None, left_on=None, right_on=None, how="inner", key_to_keep="left"):
        self.state = None
        if on is not None:
            assert left_on is None and right_on is None
            self.left_on = on
            self.right_on = on
        else:
            assert left_on is not None and right_on is not None
            self.left_on = left_on
            self.right_on = right_on
        self.phase = "build"
        assert how in {"inner", "left", "semi", "anti"}
        self.how = how
        self.key_to_keep = key_to_keep
        self.things_seen = []
        self._pending = []          # build batches, hashed once at the first probe
        self._build = None
        self._template = None       # one build row of any rank: the NULL columns of a left join without build rows here

    def build_rows(self) -> int:
        return sum(len(b) for b in self._pending) + (len(self.state) if self.state is not None else 0)

    def make_bloom(self, words: int, nparts: int):
        """Blocked Bloom filter over this channel's build keys (semi-join reduction of the probe edge)."""
        if self._pending:
            self._freeze_build()
        keys = self.state[self.right_on].data if self.state is not None else None
        return ops.Bloom.build(keys, words, nparts, default_device())

    def bloom_ok(self) -> bool:
        """String keys are compared by value across unrelated dictionaries: their codes cannot feed a filter."""
        cols = [b[self.right_on] for b in self._pending] + ([self.state[self.right_on]] if self.state is not None else [])
        return all(c.dictionary is None and c.data.dtype != torch.float64 for c in cols)

    def left_template_row(self):
        """One build row of this rank (None: it has none)."""
        if self.state is not None and len(self.state):
            return self.state.slice(0, 1)
        return next((b.slice(0, 1) for b in self._pending if len(b)), None)

    def set_left_template(self, row):
        self._template = row

    def _unmatched(self, batch: DeviceTable) -> DeviceTable:
        """A left join's probe rows with NULL build columns (typed like the template row)."""
        right = _null_rows(self._template.drop([self.right_on]), len(batch), batch[self.left_on].data.device)
        return _append_right(batch, right.columns, "_right")

    def _freeze_build(self):
        if self._build is not None:
            return
        self.state = concat_tables(self._pending)
        self._pending = []
        self._build = _HashedBuild(self.state, self.right_on)

    def execute(self, batches, stream_id, executor_id):
        batches = _clean(batches)
        if len(batches) == 0:
            return
        batch = concat_tables(batches)
        self.things_seen.append((stream_id, len(batches)))
        if stream_id == 1:
            assert self.phase == "build", (self.left_on, self.right_on, self.things_seen)
            self._pending.append(batch)
        elif stream_id == 0:
            if self.state is None and not self._pending:
                if self.how == "anti":
                    return batch
                if self.how != "left" or self._template is None:
                    return
                result = self._unmatched(batch)
            else:
                if self.phase == "build":
                    self._freeze_build()
                self.phase = "probe"
                result = self._build.probe(batch, self.left_on, self.how, "_right")
            if self.key_to_keep == "right":
                result = result.rename({self.left_on: self.right_on})
            return result

    def done(self, executor_id):
        pass


class OrderedJoinExecutor(Executor):
    """DataStream.join(maintain_sort_order=...) (pyquokka/datastream.py:1453-1469, :1536-1553): a hash join whose rows follow
    the order of one side.  Stream 0 is that side (the probe; it never leaves its rank), stream 1 the build side, numbered in
    the build stream's order (rank order, then arrival order).  The ordered probe (qk_join_probe_ordered) writes a probe row's
    matches in build-row order, so the output is in probe order with each row's matches in build order.  With
    probe_is_left the output is the probe's columns and the build's without its key; otherwise (maintain_sort_order="right",
    inner only) the build's columns and the probe's without its key -- the unordered join's columns either way.
      * streaming (the build side replicated, or one rank): every probe batch is joined as it arrives.
      * otherwise (the build side hash-partitioned across ranks), in done(): each rank sends (key, position) of its probe
        rows to the rank that owns the key's build rows; the owner probes what it received, source rank by source rank, and
        answers every source with (position, build columns) -- positions only for semi / anti; the source puts the rows into
        its order (qk_join_place) and gathers its own columns.  Only keys, positions and matched build rows cross ranks.  The
        rank holds its whole probe side in device memory until then.
    As in BuildProbeJoinExecutor, an anti join against an empty build side passes the probe side through and the other
    joins emit nothing, and a left join's owner without build rows answers with NULL build columns typed like a build row of
    another rank (`left_template_row` / `set_left_template`, sent by the runtime once the build side is complete)."""

    ordered_output = True            # rows stay on their rank, in the probe side's order
    POS = "__qk_pos"

    def __init__(self, probe_on, build_on, how, probe_is_left=True, streaming=True) -> None:
        assert how in {"inner", "left", "semi", "anti"} and (probe_is_left or how == "inner")
        self.probe_on, self.build_on, self.how, self.probe_is_left, self.streaming = probe_on, build_on, how, probe_is_left, streaming
        self.silent_streams = (1,) if streaming else "all"
        self.emits_on_done = not streaming
        self._right = _SourceRanks()
        self._left = []
        self._build, self._frozen = None, False
        self._template = None        # one build row of any rank, without its key: the NULL columns of a left join

    def left_template_row(self):
        """One build row of this rank without its key column (None: it has none)."""
        b = next((b for r in sorted(self._right.parts) for b in self._right.parts[r] if len(b)), None)
        return b.slice(0, 1).drop([self.build_on]) if b is not None else None

    def set_left_template(self, row):
        self._template = row

    def explain(self) -> str:
        return (f"ordered {self.how} join {self.probe_on} = {self.build_on}, keeps the {'left' if self.probe_is_left else 'right'} "
                f"order, {'streaming' if self.streaming else 'keys to the owners and back'}")

    def _freeze(self):
        if not self._frozen:
            t = self._right.take()
            self._build = _HashedBuild(t, self.build_on) if t is not None and len(t) else None
            self._frozen = True

    def _payload(self, bi: torch.Tensor) -> DeviceTable:
        """What the build side contributes to the output rows `bi`."""
        return self._build.rows(bi, self.how) if self.probe_is_left else self._build.table.gather(bi)

    def _combine(self, probe_rows: DeviceTable, payload: DeviceTable | None) -> DeviceTable:
        """probe_rows: the probe side's rows of the output (all columns).  The output's columns in the unordered join's order."""
        if payload is None:
            return probe_rows
        if self.probe_is_left:
            return _append_right(probe_rows, payload.columns, "_right")
        return _append_right(payload, probe_rows.drop([self.probe_on]).columns, "_right")

    def _probe(self, keys: DeviceTable):
        """(probe rows, build rows | None) of the ordered probe of `keys` (a table holding the probe key column)."""
        return self._build.hashed.probe_ordered(self._build.key(keys, self.probe_on), _HOW[self.how])

    def execute(self, batches, stream_id, executor_id):
        batches = _clean(batches)
        if stream_id == 1:
            self._right.add(batches)
            return None
        if not batches:
            return None
        if not self.streaming:
            self._left.extend(batches)
            return None
        batch = concat_tables(batches)
        self._freeze()
        if self._build is None:
            return batch if self.how == "anti" else None
        pi, bi = self._probe(batch)
        return self._combine(batch.gather(pi), None if bi is None else self._payload(bi))

    def done(self, executor_id):
        return None if self.streaming else self._round_trip()

    def _round_trip(self):
        from . import runtime as RT
        from .edge import apply_partitioner
        from .target_info import HashPartitioner
        w, me, dev = RT.world_size(), RT.rank(), default_device()
        ex = RT.Exchange(dev)
        P, self._left = (concat_tables(self._left) if self._left else None), []
        self._freeze()
        n = len(P) if P is not None else 0
        # 1. (key, position) of every probe row to the rank that owns the key's build rows -- the build edge's partition
        parts = {}
        if n:
            keys = DeviceTable({self.probe_on: P[self.probe_on], self.POS: DeviceColumn(torch.arange(n, dtype=torch.int32, device=dev))})
            parts = apply_partitioner(HashPartitioner(self.probe_on), keys, me, w)
        got = ex(parts, w, edge_key=("ordered-join-keys", id(self)))
        # 2. the owner probes the received keys in source-rank order and answers each source with (position, build columns)
        replies = {}
        if got:
            K = concat_tables(got)
            reply = None
            if self._build is not None:
                pi, bi = self._probe(K)
                reply = K.select([self.POS]).gather(pi)
                if bi is not None:
                    reply = _append_right(reply, self._payload(bi).columns, "")
            elif self.how == "anti":
                pi, reply = torch.arange(len(K), dtype=torch.int32, device=dev), K.select([self.POS])
            elif self.how == "left" and self._template is not None:
                # no build rows here, some on another rank (none anywhere: a left join emits nothing, as the unordered one)
                pi = torch.arange(len(K), dtype=torch.int32, device=dev)
                reply = _append_right(K.select([self.POS]), _null_rows(self._template, len(K), dev).columns, "")
            if reply is not None and len(reply):
                starts = torch.tensor([0] + [len(g) for g in got], device=dev).cumsum(0)
                cut = torch.searchsorted(pi.to(torch.int64), starts).tolist()     # the reply is in source order
                replies = {g.src_rank: reply.slice(cut[i], cut[i + 1]) for i, g in enumerate(got) if cut[i + 1] > cut[i]}
        back = ex(replies, w, edge_key=("ordered-join-rows", id(self)))
        # 3. the source puts what came back into its order and gathers its own columns
        if not n or not back:
            return None
        B = concat_tables(back)
        src, pos = ops.JoinTable.place(B[self.POS].data.to(torch.int32).contiguous(), n)
        payload = None if self.how in ("semi", "anti") else B.drop([self.POS]).gather(src)
        return self._combine(P.gather(pos), payload)


class BroadcastJoinExecutor(Executor):
    """sql_executors.py:275-319: probe batches against a small in-memory table held by the executor."""

    emits_on_done = False        # done() returns nothing: the runtime skips the (empty) exchange after it

    def __init__(self, small_table, on=None, small_on=None, big_on=None, suffix="_small", how="inner"):
        self.suffix = suffix
        assert how in {"inner", "left", "semi", "anti"}
        self.how = how
        self._small_src = small_table
        self.state = None
        if on is not None:
            assert small_on is None and big_on is None
            self.small_on = on
            self.big_on = on
        else:
            assert small_on is not None and big_on is not None
            self.small_on = small_on
            self.big_on = big_on
        names = small_table.column_names if hasattr(small_table, "column_names") else list(small_table.columns)
        assert self.small_on in names
        self._build = None

    def execute(self, batches, stream_id, executor_id):
        batches = _clean(batches)
        if len(batches) == 0:
            return
        batch = concat_tables(batches)
        if self._build is None:                         # opened lazily on first execute (tutorial.md:56)
            self.state = as_device_table(self._small_src)
            self._build = _HashedBuild(self.state, self.small_on)
        return self._build.probe(batch, self.big_on, self.how, self.suffix)

    def done(self, executor_id):
        return


# ---------------------------------------------------------------------------------------------- aggregates
_AGG_OPS = {"sum": L.AGG_SUM, "min": L.AGG_MIN, "max": L.AGG_MAX}


class _GrowingHashAgg:
    """The hash-aggregate state of a streaming executor.  `state` is created on the first batch with
    max(1 << 16, first_factor * rows) slots; when a batch would push the load past 1/2, the groups are re-inserted into a
    larger table first (SUM / MIN / MAX are all re-foldable)."""

    def __init__(self, agg_ops: list, first_factor: int):
        self.agg_ops, self.first_factor, self.state = agg_ops, first_factor, None

    def update(self, keys: list, vals: list):
        n = keys[0].numel()
        if self.state is None:
            self.state = ops.HashAggState([k.dtype for k in keys], self.agg_ops, max(1 << 16, self.first_factor * n), keys[0].device)
        elif self.state.rows_seen + n > self.state.capacity // 2:
            self._grow(n)
        self.state.update(keys, vals)

    def _grow(self, incoming: int):
        old = self.state
        ok, ov, _ = old.finalize()
        self.state = ops.HashAggState(old.key_dtypes, self.agg_ops, max(4 * (len(ok[0]) + incoming), 2 * old.capacity), old.device)
        if len(ok[0]):
            self.state.update(ok, ov)
        self.state.rows_seen = len(ok[0])
        # the replaced buffers may have been allocated on another lane's stream while chunks are in flight on several: the
        # allocator must not hand them out again before the kernels queued on THIS stream have read them
        for t in (getattr(old, "state", None), getattr(old, "overflow", None)):
            if isinstance(t, torch.Tensor) and t.is_cuda:
                t.record_stream(torch.cuda.current_stream())


class SQLAggExecutor(Executor):
    """sql_executors.py:556-599: the final phase of the two-phase aggregate.  `sql_statement` is the
    final select list the reference generates, e.g.
    "SUM(e0_agg_0) AS sum_qty,(SUM(e4_agg_0) / SUM(e4_agg_1)) AS avg_qty" (sql_utils.py:379-413): every
    aggregate call is a SUM / MIN / MAX over a partial column.  Partials are folded into a persistent
    hash-aggregate state as they arrive (the reference concatenates them and aggregates at done())."""

    silent_streams = "all"       # execute() folds partials; rows only leave in done()

    def __init__(self, groupby_keys, orderby_keys, sql_statement) -> None:
        assert type(groupby_keys) == list
        if orderby_keys is not None:
            assert type(orderby_keys) == list
        self.groupby_keys = groupby_keys
        self.orderby_keys = orderby_keys
        self.sql_statement = sql_statement
        self.final = E.parse_select_list(sql_statement)
        self.calls = []                                  # distinct (func, column)

        def collect(n):
            if n.kind == "agg":
                f = n.value
                if f == "count":
                    raise L.QkError("final aggregates are SUM/MIN/MAX over partial columns (COUNT partials are re-aggregated with SUM)")
                if f not in _AGG_OPS or len(n.args) != 1 or n.args[0].kind != "col":
                    raise L.QkError(f"unsupported final aggregate {n.sql()}")
                key = (f, n.args[0].value)
                if key not in self.calls:
                    self.calls.append(key)
            for a in n.args:
                collect(a)
        for e, alias in self.final:
            collect(e)
        self.state = None
        self._ha = _GrowingHashAgg([_AGG_OPS[f] for f, _ in self.calls], first_factor=2)
        self._dense = None
        self._key_meta = None
        self._types = None          # per call: (torch dtype, arrow type) of an integer / date result, None = fp64

    def execute(self, batches, stream_id, executor_id):
        batches = _clean(batches)
        if not batches:
            return
        batch = concat_tables(batches)
        if self._types is None:
            # integer partials (COUNT, integer SUM / MIN / MAX, dates) give integer results, like the reference's engines
            self._types = [agg_result_type(f, batch[c]) for f, c in self.calls]
        vals = [to_f64(batch[c].data) for _, c in self.calls]
        if not self.groupby_keys:
            self._dense = keyless_aggregate(self._dense, vals, [f for f, _ in self.calls], len(batch), batch.device, variant=1)
            return
        keys = [batch[k] for k in self.groupby_keys]
        if self._key_meta is not None:
            # keep one dictionary per key column across batches
            fixed = []
            for k, (dic, at) in zip(keys, self._key_meta):
                if dic is not None and k.dictionary != dic:
                    dic2, (a, b) = unify_dictionaries([DeviceColumn(torch.zeros(0, dtype=k.data.dtype, device=k.data.device), dic, at), k])
                    if dic2 != dic:
                        raise L.QkError("dictionary of a group key changed between batches after codes were stored")
                    k = b
                fixed.append(k)
            keys = fixed
        else:
            self._key_meta = [(k.dictionary, k.arrow_type) for k in keys]
        self._ha.update([k.data for k in keys], vals)

    def done(self, executor_id):
        if self._ha.state is None and self._dense is None:
            return None
        if self._dense is not None:
            acc = self._dense.acc
            cols = {f"__a{i}": restore_type(acc[:, i].clone(), self._types[i]) for i in range(len(self.calls))}
            if not cols:
                cols = {"__n": DeviceColumn(self._dense.cnt.to(torch.float64))}
        else:
            ok, ov, _ = self._ha.state.finalize()
            cols = {k: DeviceColumn(o, m[0], m[1]) for k, o, m in zip(self.groupby_keys, ok, self._key_meta)}
            cols.update({f"__a{i}": restore_type(v, self._types[i]) for i, v in enumerate(ov)})
        t = DeviceTable(cols)

        def lower(n):
            if n.kind == "agg":
                return E.col(f"__a{self.calls.index((n.value, n.args[0].value))}")
            return E.Node(n.kind, n.value, tuple(lower(a) for a in n.args))
        defs = {k: E.col(k) for k in self.groupby_keys}
        for i, (e, alias) in enumerate(self.final):
            defs[alias or f"col{i}"] = lower(e)
        result = EdgeOps(None, defs).apply(t, stable=True)
        if self.orderby_keys:
            result = sort_table(result, [k for k, _ in self.orderby_keys], [d == "desc" for _, d in self.orderby_keys])
        self.state = result
        return result


_SIGN = np.uint64(1 << 63)
_SIGN_I64 = -(1 << 63)          # the same bit in an int64 tensor: image ^ _SIGN_I64 orders as int64 the way the image orders


def order_image(v: np.ndarray, descending: bool) -> np.ndarray:
    """uint64 image of a sort column whose ascending order is the ORDER BY order (DESIGN.md section 2), the image
    csrc/topk.cu image_of() selects on: integers exact over their full range, -0.0 = +0.0, every NaN after +inf.
    DESC is the bitwise complement, which is monotone and cannot overflow (negating INT64_MIN does)."""
    if v.dtype.kind == "f":
        with np.errstate(invalid="ignore"):                       # a signalling NaN stays a NaN
            b = (v.astype(np.float64) + 0.0).view(np.uint64)     # + 0.0 folds -0.0 onto +0.0
        img = np.where(b >> np.uint64(63) != 0, ~b, b | _SIGN)
        img[np.isnan(v)] = ~np.uint64(0)
    elif v.dtype.kind == "i":
        img = v.astype(np.int64).view(np.uint64) ^ _SIGN
    else:
        img = v.astype(np.uint64)
    return ~img if descending else img


def sort_table(t: DeviceTable, by: list, descending: list, limit: int | None = None) -> DeviceTable:
    """ORDER BY of a (small) result on the host index space: the order is computed from the few sort
    columns, the rows are moved by the gather kernel.  NULL (valid == 0) sorts last in both directions."""
    if len(t) == 0:
        return t
    keys = []
    for c, d in zip(by, descending):
        col = t[c]
        v = col.data.cpu().numpy()
        if col.dictionary is not None:                     # order by the string value, not by the code
            rank = np.argsort(np.argsort(np.array(col.dictionary, dtype=object)))
            v = rank[v]
        img = order_image(v, d)
        if col.valid is not None:
            null = col.valid.cpu().numpy() == 0
            keys.append(null)                              # NULLS LAST; NULLs tie with each other
            img[null] = 0
        keys.append(img)
    order = np.lexsort(keys[::-1])
    if limit is not None:
        order = order[:limit]
    return t.gather(torch.from_numpy(order.astype(np.int32)).to(t.device))


_TOPK_RE = re.compile(r"^\s*select\s+\*\s+from\s+batch_arrow\s+order\s+by\s+(.+?)\s+limit\s+(\d+)\s*$", re.I)


def top_k_table(t: DeviceTable, by: list, descending: list, k: int) -> DeviceTable:
    """Radix-select candidates on the primary sort column (qk_topk_candidates), then order the few
    survivors on all sort columns.  Rows whose primary value is NULL come after every valid row: they are
    left out of the select, and only when fewer than k valid rows exist are the best of them appended."""
    if len(t) == 0:
        return t
    primary = t[by[0]]
    if primary.dictionary is not None or len(t) <= 4096:         # a few rows: ordering them on the host beats ~20 select launches
        return sort_table(t, by, descending, k)
    if primary.valid is None:
        return sort_table(t.gather(ops.topk_candidates(primary.data, k, descending[0])), by, descending, k)
    valid = primary.valid.bool()
    vidx = torch.nonzero(valid).flatten().to(torch.int32)
    if len(vidx) >= k:
        cand = vidx[ops.topk_candidates(ops.gather([primary.data], vidx)[0], k, descending[0]).long()]
        return sort_table(t.gather(cand), by, descending, k)
    nulls = t.gather(torch.nonzero(~valid).flatten().to(torch.int32))
    rest = top_k_table(nulls, by[1:], descending[1:], k - len(vidx)) if len(by) > 1 else nulls.slice(0, k - len(vidx))
    return sort_table(concat_tables([t.gather(vidx), rest]), by, descending, k)


class ConcatThenSQLExecutor(Executor):
    """sql_executors.py:45-67.  The reference runs an arbitrary DuckDB statement over the concatenated
    input at done(); the statements Quokka itself generates for this executor are the top-k form
    `select * from batch_arrow order by <cols> limit k` (datastream.py:1746), which is what is supported."""

    silent_streams = "all"       # execute() keeps candidates; the ordered result leaves in done()

    def __init__(self, sql_statement) -> None:
        self.statement = sql_statement
        self.state = None
        m = _TOPK_RE.match(sql_statement)
        if not m:
            raise NotImplementedError("ConcatThenSQLExecutor supports `select * from batch_arrow order by ... limit k`")
        self.k = int(m.group(2))
        self.by, self.desc = [], []
        for part in m.group(1).split(","):
            toks = part.split()
            self.by.append(toks[0])
            self.desc.append(len(toks) > 1 and toks[1].lower() == "desc")
        self._batches = []

    def execute(self, batches, stream_id, executor_id):
        b = _clean(batches)
        if b:
            # keep only what can still make the cut: top-k of a union = top-k of the per-batch top-ks
            self._batches.append(top_k_table(concat_tables(b), self.by, self.desc, self.k))

    def done(self, executor_id):
        if not self._batches:
            return None
        self.state = top_k_table(concat_tables(self._batches), self.by, self.desc, self.k)
        return self.state


def _sort_key(col: DeviceColumn, name: str) -> torch.Tensor:
    """The values a column sorts by: a string column by its value (the rank of every dictionary entry), not by its code."""
    if col.is_vector:
        raise L.QkError(f"sort: column {name!r} is a vector column")
    if col.dictionary is None:
        return col.data
    rank = np.argsort(np.argsort(np.array(col.dictionary, dtype=object), kind="stable"), kind="stable")
    lut = torch.from_numpy(rank.astype(np.int32) if len(rank) else np.zeros(1, np.int32)).to(col.data.device)
    return lut[col.data.long()]


def sort_perm_table(t: DeviceTable, by: list, descending: list, want_image: bool = False):
    """The permutation that puts `t` in ORDER BY by[0] [DESC], by[1] [DESC], ... order, NULLS LAST, rows that tie on every
    column in their order in `t`: a chain of stable device sorts (qk_sort_perm), last column first.  want_image: also the
    sorted order images of by[0] (int64 holding the uint64 bits) -> (perm, image)."""
    perm, image = None, None
    for i in range(len(by) - 1, -1, -1):
        col = t[by[i]]
        got = ops.sort_perm(_sort_key(col, by[i]), col.valid, bool(descending[i]), perm, want_image and i == 0)
        perm, image = got if want_image and i == 0 else (got, None)
    return (perm, image) if want_image else perm


class SortExecutor(Executor):
    """sql_executors.py:88-187 (SuperFastSortExecutor): ORDER BY over the whole stream, answered in done().  The reference
    sorts every batch with Polars, spills the runs to disk and merges them on one channel; here the rows stay in HBM, every
    rank sorts what it holds with the device radix sort and, across ranks, a sample sort leaves rank r with the r-th RANGE
    of the first sort column -- the layout of a range-partitioned sorted reader, which the ordered operators (as-of join
    over time ranges, windows, pattern search) consume as it is:
      * every rank takes SAMPLES_PER_RANK * world regularly spaced (image, NULL) samples of its sorted run; all ranks sort
        the same samples and cut them at the same world - 1 splitters;
      * a row goes to rank #{splitters <= its first-column image}, so all rows of one first-column value land on one rank
        (one value that holds most of the rows makes that rank hold most of the rows); the run is sorted, so every
        destination is one contiguous slice;
      * the received runs, in source-rank order, are sorted once more (stable: ties keep source rank, then arrival order).
    Multi-column, per-column direction, stable, NULLS LAST.  Everything must fit in device memory: nothing is spilled."""

    silent_streams = "all"
    ordered_output = True            # rank r's rows precede rank r + 1's on the first sort column
    SAMPLES_PER_RANK = 64

    def __init__(self, columns, descending) -> None:
        self.columns, self.descending = list(columns), [bool(d) for d in descending]
        self._batches = []
        self.state = None

    def explain(self) -> str:
        return "sort " + ", ".join(c + (" desc" if d else "") for c, d in zip(self.columns, self.descending))

    def execute(self, batches, stream_id, executor_id):
        self._batches.extend(_clean(batches))

    def _sorted(self, t: DeviceTable):
        perm, image = sort_perm_table(t, self.columns, self.descending, want_image=True)
        return t.gather(perm), image

    def done(self, executor_id):
        from . import runtime as RT
        t, self._batches = (concat_tables(self._batches) if self._batches else None), []
        w = RT.world_size()
        if w == 1:
            self.state = self._sorted(t)[0] if t is not None else None
            return self.state
        dev, first = default_device(), self.columns[0]
        ex = RT.Exchange(dev)
        if t is not None and t[first].dictionary is not None:
            # string first column: the ranks compare images, so they need one dictionary -- every rank's entries to everybody
            d = t[first].dictionary
            entries = DeviceTable({first: DeviceColumn(torch.arange(len(d), device=dev).to(t[first].data.dtype), d)})
        else:
            entries = None
        if ex.max_over_ranks([int(entries is not None)])[0]:
            got = ex.to_ranks(entries, ("sort-dictionary", id(self)))
            if entries is not None:
                union = DeviceColumn(torch.empty(0, dtype=t[first].data.dtype, device=dev), got[0][first].dictionary)
                t = t.with_column(first, unify_dictionaries([t[first], union])[1][0])
        run, image = self._sorted(t) if t is not None else (None, None)
        # ---- the same samples on every rank: signed images (image ^ sign bit, so int64 order is image order) + NULL flags
        samples = None
        if run is not None:
            n, s = len(run), self.SAMPLES_PER_RANK * w
            at = (torch.arange(s, device=dev, dtype=torch.int64) * n + n // 2) // s if n > s else torch.arange(n, device=dev)
            fv = run[first].valid
            null = (fv[at] == 0).to(torch.uint8) if fv is not None else torch.zeros(len(at), dtype=torch.uint8, device=dev)
            samples = DeviceTable({"image": DeviceColumn(image[at] ^ _SIGN_I64), "null": DeviceColumn(null)})
        got = ex.to_ranks(samples, ("sort-samples", id(self)))
        if not got:
            return None
        allsamp = concat_tables(got)
        order = ops.sort_perm(allsamp["image"].data.contiguous(), (1 - allsamp["null"].data).contiguous(), False)
        cut = order[(torch.arange(1, w, device=dev) * len(order)) // w].long()
        split_img, split_null = allsamp["image"].data[cut], allsamp["null"].data[cut].tolist()
        # ---- my run's slice for every rank: rows whose image is below splitter r stay left of it; NULLs are past every value
        bounds = None
        if run is not None:
            fv = run[first].valid
            nvalid = len(run) if fv is None else int(fv.sum().item())      # NULLS LAST: the run's valid rows come first
            pos = torch.searchsorted(image[:nvalid] ^ _SIGN_I64, split_img).tolist()
            bounds = [0] + [nvalid if isnull else p for p, isnull in zip(pos, split_null)] + [len(run)]
        mine = ex.hand_off(run, bounds, ("sort-rows", id(self)))
        if not mine:
            return None
        self.state = self._sorted(concat_tables(mine))[0]
        return self.state


class DistinctExecutor(Executor):
    """sql_executors.py:517-554; emits the distinct key combinations once, at done()."""

    silent_streams = "all"

    def __init__(self, keys) -> None:
        self.keys = keys
        self.state = None
        self._ha = _GrowingHashAgg([], first_factor=4)
        self._meta = None

    def execute(self, batches, stream_id, executor_id):
        batches = _clean(batches)
        if len(batches) == 0:
            return
        batch = concat_tables(batches)
        keys = [batch[k] for k in self.keys]
        if self._meta is None:
            self._meta = [(k.dictionary, k.arrow_type) for k in keys]
        self._ha.update([k.data for k in keys], [])

    def done(self, executor_id):
        if self._ha.state is None:
            return
        ok, _, _ = self._ha.state.finalize()
        self.state = DeviceTable({k: DeviceColumn(o, m[0], m[1]) for k, o, m in zip(self.keys, ok, self._meta)})
        return self.state


# ---------------------------------------------------------------------------------------------- Gram matrix
def _gram_input(col: DeviceColumn, name: str) -> torch.Tensor:
    """A column as qk_gram reads it.  Numbers only: string (dictionary) and date / time columns have no product, as np.dot
    of the reference fails on them.  A NULL (right side of a left / as-of join) becomes NaN, as Polars' to_numpy() makes it."""
    if col.dictionary is not None:
        raise L.QkError(f"gramian / covariance: column {name!r} is a string column")
    if col.arrow_type is not None and not pa.types.is_boolean(col.arrow_type):
        raise L.QkError(f"gramian / covariance: column {name!r} has type {col.arrow_type}, not a number")
    t = col.data
    if t.dtype not in (torch.float64, torch.float32, torch.int32, torch.int64):
        t = t.to(torch.int32)                              # bool / uint8 flags count as 0 / 1
    if col.valid is not None:
        t = torch.where(col.valid.bool(), t.to(torch.float64), torch.full_like(t, float("nan"), dtype=torch.float64))
    return t.contiguous()


class GramPartialExecutor(Executor):
    """Per-rank phase of DataStream.gramian / covariance (pyquokka/datastream.py:1033-1147, whose per-batch np.dot partials are
    summed by an AggExecutor per channel): every batch is folded into a GramState by qk_gram.  The shift is `demean` (gramian) or,
    with shift_first_row, the first row this rank sees (covariance: the final phase re-centres the ranks on the global mean,
    and a shift near the data keeps the fp64 sums from cancelling).  done() emits the state as ONE flat fp64 column
    [executor_id, n, c (k), s (k), G (k * k)]: the exchange carries at most 16 columns, a k-column table would not fit."""

    silent_streams = "all"       # execute() only accumulates; the state leaves in done()

    def __init__(self, columns, demean=None, shift_first_row=False) -> None:
        self.columns = list(columns)
        self.demean = None if demean is None else np.asarray(demean, dtype=np.float64)
        self.shift_first_row = shift_first_row
        self.state = None
        self.shift = None

    def execute(self, batches, stream_id, executor_id):
        for b in _clean(batches):
            xs = [_gram_input(b[c], c) for c in self.columns]
            if self.state is None:
                self.state = ops.GramState(len(self.columns), b.device)
                if self.shift_first_row:
                    self.shift = torch.cat([x[:1].to(torch.float64) for x in xs])
                elif self.demean is not None:
                    self.shift = torch.from_numpy(self.demean.copy()).to(b.device)
            self.state.update(xs, self.shift)

    def done(self, executor_id):
        if self.state is None:
            return None
        s = self.state
        shift = self.shift if self.shift is not None else torch.zeros(s.k, dtype=torch.float64, device=s.gram.device)
        head = torch.tensor([float(executor_id), float(s.n)], dtype=torch.float64, device=s.gram.device)
        flat = torch.cat([head, shift, s.sums, s.gram.reshape(-1)])
        return DeviceTable({"__gram": DeviceColumn(flat)})


class GramFinalExecutor(Executor):
    """Final phase of DataStream.gramian / covariance on one channel: sums the per-rank partials in rank order and emits the
    k x k result as a table with the schema `columns` (row i = row i of the matrix).  mode "gramian": sum of the G_r (every
    rank used the same shift).  mode "covariance": re-centres rank r's (n_r, c_r, G_r, s_r) on the global mean
    mu = sum_r (n_r c_r + s_r) / n with d_r = c_r - mu, sum_r [G_r + s_r d_r^T + d_r s_r^T + n_r d_r d_r^T], and divides by n
    (np.cov(bias=True), as the reference divides by the row count).  O(ranks k^2) fp64 work on the final state."""

    silent_streams = "all"       # the matrix leaves in done()

    def __init__(self, columns, mode="gramian") -> None:
        assert mode in ("gramian", "covariance")
        self.columns = list(columns)
        self.mode = mode
        self.parts = []
        self.state = None

    def execute(self, batches, stream_id, executor_id):
        for b in _clean(batches):
            flat = b["__gram"].data
            width = 2 + 2 * len(self.columns) + len(self.columns) ** 2
            for lo in range(0, flat.numel(), width):        # partials of several ranks may arrive in one batch
                self.parts.append(flat[lo:lo + width])

    def done(self, executor_id):
        k = len(self.columns)
        dev = self.parts[0].device if self.parts else default_device()
        parts = sorted(self.parts, key=lambda p: float(p[0]))
        n = sum(float(p[1]) for p in parts)
        G = torch.zeros(k, k, dtype=torch.float64, device=dev)
        if self.mode == "gramian":
            for p in parts:
                G += p[2 + 2 * k:].reshape(k, k)
        elif n == 0:
            G.fill_(float("nan"))
        else:
            mu = torch.zeros(k, dtype=torch.float64, device=dev)
            for p in parts:
                mu += float(p[1]) * p[2:2 + k] + p[2 + k:2 + 2 * k]
            mu /= n
            for p in parts:
                nr, c, s, g = float(p[1]), p[2:2 + k], p[2 + k:2 + 2 * k], p[2 + 2 * k:].reshape(k, k)
                d = c - mu
                G += g + torch.outer(s, d) + torch.outer(d, s) + nr * torch.outer(d, d)
            G /= n
        self.state = DeviceTable({c: DeviceColumn(G[:, j].contiguous()) for j, c in enumerate(self.columns)})
        return self.state


# ---------------------------------------------------------------------------------------------- quantile sketch
QUANTILE_ENTRY_COLUMNS = ["__qkey", "__qcount", "__qmin", "__qmax"]


def _quantile_input(col: DeviceColumn, name: str) -> tuple[torch.Tensor, torch.Tensor | None]:
    """(values, row mask or None) of a column as qk_qsketch_update reads it.  Numbers only, as for the Gram matrix: string
    (dictionary) and date / time columns raise.  Booleans and uint8 flags count as 0 / 1.  A NULL (right side of a left / as-of
    join) is not counted: its validity mask becomes the kernel's row mask."""
    if col.dictionary is not None:
        raise L.QkError(f"approximate_quantile: column {name!r} is a string column")
    if col.arrow_type is not None and not pa.types.is_boolean(col.arrow_type):
        raise L.QkError(f"approximate_quantile: column {name!r} has type {col.arrow_type}, not a number")
    t = col.data
    if t.dtype == torch.bool:
        t = t.view(torch.uint8)
    elif t.dtype not in (torch.float64, torch.float32, torch.int64, torch.int32, torch.uint8):
        t = t.to(torch.int32)
    valid = None if col.valid is None else col.valid.to(torch.uint8).contiguous()
    return t.contiguous(), valid


class QuantilePartialExecutor(Executor):
    """Per-rank phase of DataStream.approximate_quantile (pyquokka/datastream.py:905-1031, where each channel feeds a host
    t-digest): every batch is folded into one QuantileSketch by qk_qsketch_update.  done() emits the sketch's entries as four
    int64 columns (key, count, min image, max image)."""

    silent_streams = "all"       # execute() only accumulates; the entries leave in done()

    def __init__(self, columns) -> None:
        self.columns = list(columns)
        self.state = None

    def execute(self, batches, stream_id, executor_id):
        for b in _clean(batches):
            ins = [_quantile_input(b[c], c) for c in self.columns]
            if self.state is None:
                self.state = ops.QuantileSketch(len(self.columns), b.device)
            masks = [v for _, v in ins]
            self.state.update([t for t, _ in ins], None if all(m is None for m in masks) else masks)

    def done(self, executor_id):
        if self.state is None:
            return None
        return DeviceTable({n: DeviceColumn(t) for n, t in zip(QUANTILE_ENTRY_COLUMNS, self.state.entries())})


class QuantileFinalExecutor(Executor):
    """Final phase of DataStream.approximate_quantile on one channel: merges the entries of every rank into one sketch by
    qk_qsketch_merge (the merged state is the sketch of all the rows, whatever the split) and emits one fp64 row per
    quantile, in the order given, with the schema `columns`.  A column without counted rows is NULL."""

    silent_streams = "all"       # the quantiles leave in done()

    def __init__(self, columns, quantiles) -> None:
        self.columns = list(columns)
        self.quantiles = [float(q) for q in quantiles]
        self.parts = []
        self.state = None

    def execute(self, batches, stream_id, executor_id):
        for b in _clean(batches):
            self.parts.append([b[c].data for c in QUANTILE_ENTRY_COLUMNS])

    def done(self, executor_id):
        k = len(self.columns)
        dev = self.parts[0][0].device if self.parts else default_device()
        sk = ops.QuantileSketch(k, dev, capacity=4 * sum(p[0].numel() for p in self.parts))
        for p in self.parts:
            sk.merge(*p)
        vals, valid = sk.quantiles(self.quantiles)
        cols = {}
        for j, c in enumerate(self.columns):
            ok = valid[:, j]
            cols[c] = DeviceColumn(vals[:, j].contiguous(), valid=None if bool(ok.all()) else ok.to(torch.uint8).contiguous())
        self.state = DeviceTable(cols)
        return self.state


# ---------------------------------------------------------------------------------------------- nearest neighbours
KNN_HIDDEN = ["__knn_probe", "__knn_score", "__knn_key"]
_KNN_RANK_SHIFT = 56            # final key = rank << 56 | batch sequence << 32 | row


class KnnPartialExecutor(Executor):
    """Per-rank phase of DataStream.vector_nn_join (DFProbeDataStreamNNExecutor1, pyquokka/executors/vector_executors.py:8-52,
    which keeps every batch's k best rows per probe).  Every batch goes through qk_knn_topk; its <= q * k candidate rows (all
    columns, vectors included) are gathered and merged by qk_knn_merge into a running state of q * k rows, keyed by arrival
    (batch sequence << 32 | row).  done() emits the state, slot (p, j) at row p * k + j, with the hidden columns probe id, score
    and key (rank in the top bits; -1 for an empty slot)."""

    silent_streams = "all"       # execute() only accumulates; the candidates leave in done()

    def __init__(self, vec_column, probes, k) -> None:
        self.vec_column = vec_column
        self.probes_host = np.ascontiguousarray(probes, dtype=np.float32)
        self.k = int(k)
        self.probes = None
        self.state = None        # (scores [q, k], keys [q, k], DeviceTable of q * k rows)
        self.seq = 0

    def execute(self, batches, stream_id, executor_id):
        for b in _clean(batches):
            col = b[self.vec_column]
            if not col.is_vector:
                raise L.QkError(f"vector_nn_join: column {self.vec_column!r} is not a vector column")
            if col.data.shape[1] != self.probes_host.shape[1]:
                raise L.QkError(f"vector_nn_join: column {self.vec_column!r} has dimension {col.data.shape[1]}, the probes "
                                f"{self.probes_host.shape[1]}")
            if self.probes is None:
                self.probes = torch.from_numpy(self.probes_host).to(b.device)
            scores, rows = ops.knn_topk(col.data, self.probes, self.k)
            keys = torch.where(rows >= 0, rows | (self.seq << 32), torch.full_like(rows, -1))
            cand = b.gather(rows.reshape(-1).to(torch.int32))
            self.seq += 1
            if self.state is None:
                self.state = (scores, keys, cand)
                continue
            s0, k0, t0 = self.state
            ms, mk, src = ops.knn_merge(s0, k0, scores, keys, self.k)
            self.state = (ms, mk, concat_tables([t0, cand]).gather(src.reshape(-1)))

    def done(self, executor_id):
        if self.state is None:
            return None
        scores, keys, t = self.state
        q = scores.shape[0]
        dev = scores.device
        keys = torch.where(keys >= 0, keys | (int(executor_id) << _KNN_RANK_SHIFT), keys)
        probe = torch.arange(q, dtype=torch.int32, device=dev).repeat_interleave(self.k)
        return DeviceTable(dict(t.columns) | {"__knn_probe": DeviceColumn(probe), "__knn_score": DeviceColumn(scores.reshape(-1)),
                                              "__knn_key": DeviceColumn(keys.reshape(-1))})


class KnnFinalExecutor(Executor):
    """Final phase of DataStream.vector_nn_join on one channel (DFProbeDataStreamNNExecutor2): merges the per-rank candidate
    states with qk_knn_merge (the rank sits in the top bits of every key, so ties between ranks go to the lower rank) and emits,
    probe by probe in the probe table's order, its min(k, valid rows) rows best first, followed by the probe's columns and, if
    asked for, the score."""

    silent_streams = "all"       # the result leaves in done()

    def __init__(self, columns, probe_table: pa.Table, q, k, score_column=None) -> None:
        self.columns = list(columns)
        self.probe_table = probe_table
        self.q, self.k = int(q), int(k)
        self.score_column = score_column
        self.parts = []
        self.state = None

    def execute(self, batches, stream_id, executor_id):
        for b in _clean(batches):
            n = self.q * self.k
            for lo in range(0, len(b), n):             # the states of several ranks may arrive in one batch
                self.parts.append(b.slice(lo, lo + n))

    def done(self, executor_id):
        if not self.parts:
            return None
        q, k = self.q, self.k
        t = self.parts[0]
        s, key = t["__knn_score"].data.reshape(q, k), t["__knn_key"].data.reshape(q, k)
        for p in self.parts[1:]:
            s, key, src = ops.knn_merge(s, key, p["__knn_score"].data.reshape(q, k), p["__knn_key"].data.reshape(q, k), k)
            t = concat_tables([t, p]).gather(src.reshape(-1))
        keep = torch.nonzero(key.reshape(-1) >= 0).flatten().to(torch.int32)
        t = t.gather(keep)
        probe_rows = DeviceTable.from_arrow(self.probe_table, t.device).gather(t["__knn_probe"].data)
        cols = {c: t[c] for c in self.columns} | dict(probe_rows.columns)
        if self.score_column is not None:
            cols[self.score_column] = t["__knn_score"]
        self.state = DeviceTable(cols)
        return self.state


# ---------------------------------------------------------------------------------------------- ordered streams
class KeyCodes:
    """An append-only code space for the `by` column of ordered streams: codes that mean the same key in every batch of
    every stream that goes through one KeyCodes (batch dictionaries are re-sorted unions and differ from batch to batch).
    Strings are numbered in order of first appearance, integer codes are used as is."""

    def __init__(self) -> None:
        self.values, self.index, self.luts = None, None, {}        # strings: values by code, code by value, table per dictionary
        self.n_by = 0                                              # codes handed out so far are below this

    def codes(self, col: DeviceColumn) -> torch.Tensor:
        if col.dictionary is not None:
            if self.values is None:
                if self.n_by:
                    raise L.QkError("as-of `by` columns must both be strings or both be integer codes")
                self.values, self.index = [], {}
            key = (id(col.dictionary), len(col.dictionary))
            lut = self.luts.get(key)
            if lut is None:
                codes = []
                for v in col.dictionary:
                    i = self.index.get(v)
                    if i is None:
                        i = self.index[v] = len(self.values)
                        self.values.append(v)
                    codes.append(i)
                lut = (col.dictionary, torch.tensor(codes or [0], dtype=torch.int32, device=col.data.device))
                self.luts[key] = lut                                # keeps the dictionary alive, so its id stays unique
            self.n_by = max(self.n_by, len(self.values))
            return lut[1][col.data.long()]
        if self.values is not None:
            raise L.QkError("as-of `by` columns must both be strings or both be integer codes")
        codes = col.data.to(torch.int32)
        if len(codes):
            lo, hi = (int(v) for v in torch.stack(torch.aminmax(codes)).tolist())       # one pass, one read-back
            if lo < 0:
                raise L.QkError("as-of `by` codes must be non-negative")
            self.n_by = max(self.n_by, hi + 1)
        return codes

    def column(self, codes: torch.Tensor, bycol: DeviceColumn) -> DeviceColumn:
        """`codes` as a column of the type `bycol` came in."""
        if self.values is not None:
            return DeviceColumn(codes, list(self.values), None)
        return DeviceColumn(codes.to(bycol.data.dtype), None, bycol.arrow_type)


class _SourceRanks:
    """A sorted stream whose batches come from several producer ranks, each holding a contiguous TIME RANGE of it
    (range-partitioned sorted readers, dataset/ordered_readers.py:84-100).  All ranks ship their batches at once, so arrival
    order is not time order across ranks; rank r's rows all precede rank r + 1's, so the batches are kept per source rank in
    arrival order and the stream is put back together when it is complete."""

    def __init__(self) -> None:
        self.parts = {}              # source rank -> batches in arrival order

    def add(self, batches: list):
        for b in batches:
            self.parts.setdefault(getattr(b, "src_rank", 0) or 0, []).append(b)

    def take(self) -> DeviceTable | None:
        """The whole stream as one table (None when nothing arrived); its time column still has to pass _require_sorted."""
        parts = [b for r in sorted(self.parts) for b in self.parts[r]]
        self.parts = {}
        return concat_tables(parts) if parts else None


def _require_sorted(time: torch.Tensor, message: str):
    if len(time) > 1 and not bool((time[1:] >= time[:-1]).all().item()):
        raise L.QkError(message)


def _require_int64_time(*times: torch.Tensor):
    if any(t.dtype != torch.int64 for t in times):
        raise L.QkError("as-of time columns must be int64 / timestamp")


def _time_unit(tcol: DeviceColumn) -> str | None:
    """The unit of a timestamp column, None for a plain integer (or date) time column."""
    return str(tcol.arrow_type.unit) if tcol.arrow_type is not None and pa.types.is_timestamp(tcol.arrow_type) else None


# ---------------------------------------------------------------------------------------------- as-of
def check_asof_args(strategy, tolerance):
    """join_asof's strategy and tolerance, as the time-unit conversion of pattern_recognize's maxspan accepts it."""
    import datetime
    if strategy not in ("backward", "forward", "nearest"):
        raise ValueError(f"join_asof: strategy must be 'backward', 'forward' or 'nearest', not {strategy!r}")
    if tolerance is not None:
        if isinstance(tolerance, bool) or not isinstance(tolerance, (int, datetime.timedelta)):
            raise ValueError("join_asof: tolerance must be None, an int in the time column's unit or a datetime.timedelta")
        if (tolerance.total_seconds() if isinstance(tolerance, datetime.timedelta) else tolerance) < 0:
            raise ValueError("join_asof: tolerance must be >= 0")


class SortedAsofExecutor(Executor):
    """ts_executors.py:324-383: streaming backward as-of join of two time-sorted streams per symbol.
    stream 0 = trades (left), stream 1 = quotes (right).  A trade can be joined as soon as a quote NEWER
    than it has been seen (every quote at or before its time has arrived by then, :359); the rest
    waits for more quotes or for done().

    The join is the sorted-merge kernel (qk_asof_merge): one sweep over the merged timeline with a per-symbol table of
    the newest quote.  The table is CARRIED between calls, so every quote row is swept once however the two streams
    are batched, and -- like the reference, which trims its quote state to the last quote per symbol (:371-376) -- quotes
    that can no longer be the newest of their symbol are dropped from the state.  Symbol sets too large for the
    shared-memory table use the partition + search kernels (qk_asof_backward) over the whole quote state.

    strategy / tolerance (pandas.merge_asof's direction / tolerance): "backward" = the last quote of the symbol at or before
    the trade; "forward" = the first quote at or after it (the earliest in stream order among equal times); "nearest" = of
    those two the one closer in time, a distance tie going to the backward one.  tolerance (None, an int in the time
    column's unit, or a datetime.timedelta for a timestamp column) keeps a match only if |quote time - trade time| <= it.
    Backward with a tolerance streams as above (qk_asof_join).  Forward and nearest hold both streams and join in done():
    a trade's forward match may be any later quote, so nothing can be released before the quotes end.

    Across ranks over time ranges (_join_time_ranges), a trade goes to one owner rank:
      * backward: the last rank whose first quote time <= t, carrying the newest quote per symbol of earlier ranks;
      * forward: the first rank whose last quote time >= t, carrying the oldest quote per symbol of later ranks.  Equal quote
        times may straddle a boundary (last of rank k == first of rank k + 1); the backward rule would then send a trade at
        exactly that time to rank k + 1 and miss the first quotes at that time on rank k;
      * nearest: the backward owner, with both carries.  (1) Its backward candidate is exact, as for backward.  (2) A forward
        candidate later than t can only be on the owner or a later rank, since every earlier rank ends at or before the
        owner's first quote <= t.  (3) A forward candidate AT t on an earlier rank means a quote of the symbol exactly at t:
        then the backward candidate is at t too, its distance is 0 and it wins the tie.  So the owner sees both true
        candidates."""

    TRIM_ROWS = 1 << 20          # fold swept quotes into <= n_symbols carried rows once this many have piled up

    @property
    def silent_streams(self):      # across ranks over time ranges, or forward / nearest: everything is held until done()
        return "all" if self._over_time_ranges() or self.strategy != "backward" else ()

    def _over_time_ranges(self) -> bool:
        return bool(self.time_ranges) and world_size() > 1

    def __init__(self, time_col_trades="time", time_col_quotes="time", symbol_col_trades="symbol",
                 symbol_col_quotes="symbol", suffix="_right", time_ranges=False, strategy="backward", tolerance=None) -> None:
        check_asof_args(strategy, tolerance)
        self.strategy, self.tolerance = strategy, tolerance
        self.time_ranges = time_ranges   # several ranks, each holding a contiguous time range of both streams: join in place (done())
        self._held = None
        self.trade_state = None
        self.quote_state = None
        self.time_col_trades = time_col_trades
        self.time_col_quotes = time_col_quotes
        self.symbol_col_trades = symbol_col_trades
        self.symbol_col_quotes = symbol_col_quotes
        self.suffix = suffix
        self._codes = KeyCodes()     # the executor's own symbol codes, shared by both streams
        self._carry = None           # int32[n_by]: row of quote_state holding the newest swept quote of each symbol, -1 = none
        self._swept = 0              # rows of quote_state already folded into _carry
        self._whole_state = False    # too many symbols for the merge kernel: keep every quote, search the whole state
        self._by_source = None       # several producer ranks: {stream: _SourceRanks}, joined at done()

    BY = "__by"                      # hidden column: the symbol in the executor's code space

    def explain(self) -> str:
        return f"as-of join strategy={self.strategy}" + (f" tolerance={self.tolerance}" if self.tolerance is not None else "")

    def _tolerance_ticks(self, tcol: DeviceColumn) -> int | None:
        """The tolerance in the time column's unit (a timedelta needs a timestamp column)."""
        import datetime
        from .windowtypes import Window
        if isinstance(self.tolerance, datetime.timedelta) and _time_unit(tcol) is None:
            raise ValueError("join_asof: a timedelta tolerance needs a timestamp time column")
        return None if self.tolerance is None else Window.ticks(self.tolerance, _time_unit(tcol))

    def _strategy_args(self, tcol: DeviceColumn) -> dict:
        """The keyword arguments of ops.asof_merge / asof_backward for this join: none for the plain backward join."""
        tol = self._tolerance_ticks(tcol)
        return {} if self.strategy == "backward" and tol is None else {"strategy": self.strategy, "tolerance": tol}

    def _append(self, state, batch, tcol):
        if state is None or len(state) == 0:
            return batch
        if len(batch) > 0:
            assert int(state[tcol].data[-1].item()) <= int(batch[tcol].data[0].item()), "stream is not time-sorted"
        return concat_tables([state, batch])

    def _carry_table(self, device) -> torch.Tensor:
        n = max(1, self._codes.n_by)
        if self._carry is None:
            self._carry = torch.full((n,), -1, dtype=torch.int32, device=device)
        elif self._carry.numel() < n:                              # new symbols appeared
            self._carry = torch.cat([self._carry, torch.full((n - self._carry.numel(),), -1, dtype=torch.int32, device=device)])
        return self._carry

    def _join(self, trades: DeviceTable, upto: int | None) -> DeviceTable:
        """Joins `trades` (all older than every unswept quote past `upto`) against quote rows [swept, upto) + the carried
        table, then advances the sweep to `upto`."""
        quotes = self.quote_state
        upto = len(quotes) if upto is None else upto
        lt, rt = trades[self.time_col_trades].data, quotes[self.time_col_quotes].data
        _require_int64_time(lt, rt)
        lby, rby = trades[self.BY].data, quotes[self.BY].data
        n_by = max(1, self._codes.n_by)
        kw = self._strategy_args(trades[self.time_col_trades])
        ridx = None
        if not self._whole_state and self.strategy != "backward":     # held until done(): one join over both whole streams
            ridx, _ = ops.asof_merge(lt, lby, rt, rby, n_by, **kw)
            self._whole_state = ridx is None
        elif not self._whole_state:
            carry = self._carry_table(lt.device)
            if kw:
                kw["carry_time"] = rt[carry.clamp(min=0).long()] if len(rt) else torch.zeros(n_by, dtype=torch.int64, device=lt.device)
            ridx, carry_out = ops.asof_merge(lt, lby, rt[self._swept:upto], rby[self._swept:upto], n_by, carry, self._swept, want_carry=True,
                                             **kw)
            kw.pop("carry_time", None)
            if ridx is None:
                if self._swept:
                    raise L.QkError("as-of: the symbol set outgrew the merge kernel's table after quotes were trimmed")
                self._whole_state = True
            else:
                self._carry, self._swept = carry_out, upto
        if ridx is None:
            ridx = ops.asof_backward(lt, lby, rt, rby, n_by, **kw)
        right = quotes.drop([self.time_col_quotes, self.symbol_col_quotes, self.BY]).gather(ridx)
        right = right.with_validity((ridx >= 0).to(torch.uint8))
        out = _append_right(trades.drop([self.BY]), right.columns, self.suffix)
        self._trim()
        return out

    def _trim(self):
        """Swept quotes only matter as "newest of their symbol": keep those rows (<= n_symbols), drop the rest."""
        if self._whole_state or self._swept < max(self.TRIM_ROWS, 4 * self._codes.n_by):
            return
        carry = self._carry
        live = carry >= 0
        rows = carry[live]
        kept = self.quote_state.gather(rows)
        new_carry = torch.full_like(carry, -1)
        new_carry[live] = torch.arange(rows.numel(), dtype=torch.int32, device=carry.device)
        tail = self.quote_state.slice(self._swept, len(self.quote_state))
        self.quote_state = concat_tables([kept, tail]) if len(tail) else kept
        self._carry, self._swept = new_carry, int(rows.numel())

    def execute(self, batches, stream_id, executor_id):
        batches = _clean(batches)
        if not batches:
            return
        if self._over_time_ranges():
            if self._held is None:
                self._held = {0: [], 1: []}
            self._held[stream_id].extend(batches)
            return
        if self._by_source is not None or self.strategy != "backward" or any(getattr(b, "src_rank", None) is not None for b in batches):
            # the batches come from several producer ranks: once one has said so, both streams are put back together
            # per source rank (_SourceRanks) and joined when they are complete; so are those of a forward / nearest join
            if self._by_source is None:
                self._by_source = {0: _SourceRanks(), 1: _SourceRanks()}
            self._by_source[stream_id].add(batches)
            return
        batch = concat_tables(batches)
        by = self.symbol_col_trades if stream_id == 0 else self.symbol_col_quotes
        batch = batch.with_column(self.BY, DeviceColumn(self._codes.codes(batch[by])))
        if stream_id == 0:
            self.trade_state = self._append(self.trade_state, batch, self.time_col_trades)
        else:
            self.quote_state = self._append(self.quote_state, batch, self.time_col_quotes)
        if self.trade_state is None or self.quote_state is None or len(self.trade_state) == 0 or len(self.quote_state) == self._swept:
            return
        newest_quote = self.quote_state[self.time_col_quotes].data[-1:]
        t = self.trade_state[self.time_col_trades].data
        n_join = int(torch.searchsorted(t, newest_quote).item())  # trades with time < the newest quote's: sorted, so a prefix
        if n_join == 0:
            return
        joinable = self.trade_state.slice(0, n_join)
        self.trade_state = self.trade_state.slice(n_join, len(self.trade_state))
        upto = None
        if len(self.trade_state) == 0:
            # no trade is waiting: a LATER trade batch may start anywhere after the last trade seen, so only quotes up to
            # that time may be folded into the carried table; newer quotes stay unswept
            last_t = joinable[self.time_col_trades].data[-1:]
            qt = self.quote_state[self.time_col_quotes].data
            upto = self._swept + int(torch.searchsorted(qt[self._swept:], last_t, right=True).item())   # quotes with time <= last_t
        return self._join(joinable, upto)

    def _join_time_ranges(self):
        """Several ranks, rank r holding the r-th contiguous TIME RANGE of both sorted streams (range-partitioned sorted
        readers, dataset/ordered_readers.py:84-100).  The reference co-locates symbols with a hash shuffle of both streams; an
        as-of join over time ranges needs almost none of that traffic:
          * a trade belongs to the rank whose quote range contains its time -- splitters = every rank's first quote time; the
            sorted trades fall into one contiguous slice per rank, nearly all of it this rank's own (only the rows around a
            boundary move);
          * of the quotes of EARLIER ranks a trade can only ever see the newest one per symbol -- at most n_symbols rows per
            rank, found by the merge kernel's table pass (qk_asof_merge with no left rows) and sent to everybody;
          * then every rank joins locally: [newest-per-symbol rows of ranks < r, in rank order] + its own quotes is a sorted
            stream that gives its trades exactly the rows the global join would.
        Three small exchanges instead of moving both streams (at 1.05 B quotes per GPU: ~17 GB per rank through the shuffle
        before, a few MB now)."""
        from . import runtime as RT
        w, me = RT.world_size(), RT.rank()
        dev = default_device()
        ex = RT.Exchange(dev)
        held, self._held = self._held or {0: [], 1: []}, None
        trades = concat_tables(held[0]) if held[0] else None
        quotes = concat_tables(held[1]) if held[1] else None
        tt, qt = self.time_col_trades, self.time_col_quotes

        def shape(batches, t, col):                                 # rows, first time, last time, batches in time order?
            if t is None or len(t) == 0:
                return [0, 0, 0, 1]
            _require_int64_time(t[col].data)
            # the streams are declared sorted (OrderedStream); what is verified is how the pieces fit: batch against batch
            # here, rank against rank below -- not every row (two extra passes over both streams)
            ends = torch.stack([x for b in batches if len(b) for x in (b[col].data[0], b[col].data[-1])]).tolist()
            ok = int(all(ends[i] <= ends[i + 1] for i in range(len(ends) - 1)))
            return [len(t), int(ends[0]), int(ends[-1]), ok]
        rows = ex.allgather_words(shape(held[0], trades, tt) + shape(held[1], quotes, qt))
        for base, what in ((0, "trades"), (4, "quotes")):
            last = None
            for r in range(w):
                n, first, end, ok = rows[r][base:base + 4]
                if not ok or (n and last is not None and first < last):
                    raise L.QkError(f"as-of join: the ranks do not hold consecutive time ranges of the sorted {what} stream")
                if n:
                    last = end
        # ---- newest quote per symbol of every rank (backward, nearest), oldest (forward, nearest), to everybody
        newest = oldest = None
        if quotes is not None and len(quotes) > 0:
            codes = self._codes.codes(quotes[self.symbol_col_quotes])
            n_by = max(1, self._codes.n_by)
            if self.strategy != "forward":
                newest = quotes.gather(self._end_rows(quotes[qt].data, codes, n_by, forward=False))
            if self.strategy != "backward":
                oldest = quotes.gather(self._end_rows(quotes[qt].data, codes, n_by, forward=True))
        earlier, later = [], []
        if self.strategy != "forward":
            earlier = [g for g in ex.to_ranks(newest, ("asof-newest", id(self))) if g.src_rank < me]
        if self.strategy != "backward":
            later = [g for g in ex.to_ranks(oldest, ("asof-oldest", id(self))) if g.src_rank > me]
        # ---- trades to the rank whose quote range holds them: the k-th rank that has quotes takes the trades from its first quote
        #      time up to the next such rank's (the first one also takes everything earlier: those trades match nothing, but
        #      only a rank with quotes knows the columns to fill with NULLs); ranks without quotes take none.  Forward: the k-th
        #      rank with quotes takes the trades after the previous such rank's last quote time up to its own (the last one
        #      also takes everything later)
        owners = [r for r in range(w) if rows[r][4]]
        if not owners:
            if any(rows[r][0] for r in range(w)):
                raise L.QkError("as-of join: no quotes were received")
            return None
        bounds = None
        if trades is not None and len(trades) > 0:
            fwd = self.strategy == "forward"
            cuts = [rows[o][6] for o in owners[:-1]] if fwd else [rows[o][5] for o in owners[1:]]
            pos = torch.searchsorted(trades[tt].data, torch.tensor(cuts, dtype=torch.int64, device=dev), right=fwd).tolist() if cuts else []
            ends = {o: int(p_) for o, p_ in zip(owners[:-1], pos)} | {owners[-1]: len(trades)}
            bounds = [0]
            for r in range(w):
                bounds.append(ends[r] if r in ends else bounds[-1])
        mine = ex.hand_off(trades, bounds, ("asof-trades", id(self)))      # the own slice, the bulk, stays where it is
        self.trade_state = self.quote_state = None
        self._carry, self._swept, self._whole_state = None, 0, False
        all_q = earlier + ([quotes] if quotes is not None and len(quotes) > 0 else []) + later
        if not mine:
            return None
        t = concat_tables(mine)
        out = self._join_carried(t, earlier, later, quotes) if (earlier or later) and quotes is not None and len(quotes) > 0 else None
        if out is not None:
            return out
        q = concat_tables(all_q)
        self.quote_state = q.with_column(self.BY, DeviceColumn(self._codes.codes(q[self.symbol_col_quotes])))
        t = t.with_column(self.BY, DeviceColumn(self._codes.codes(t[self.symbol_col_trades])))
        return self._join(t, None)

    def _end_rows(self, time: torch.Tensor, codes: torch.Tensor, n_by: int, forward: bool) -> torch.Tensor:
        """Rows (int32, in time order) of the newest quote of every symbol, or with `forward` the oldest: the merge kernel's
        table pass (no left rows)."""
        dev = time.device
        empty_t, empty_b = torch.empty(0, dtype=torch.int64, device=dev), torch.empty(0, dtype=torch.int32, device=dev)
        _, table = ops.asof_merge(empty_t, empty_b, time, codes, n_by, want_carry=True, **({"strategy": "forward"} if forward else {}))
        if table is None:                                           # symbol set too large for the table: the last / first row of each code
            order = torch.arange(len(codes), device=dev, dtype=torch.int64)
            fill = len(codes) if forward else -1
            table = torch.full((n_by,), fill, dtype=torch.int64, device=dev).scatter_reduce(0, codes.long(), order, "amin" if forward else "amax",
                                                                                           include_self=True)
            table = torch.where(table == len(codes), -1, table) if forward else table
        return torch.sort(table[table >= 0]).values.to(torch.int32)          # row order = time order

    def _join_carried(self, trades, earlier, later, quotes):
        """trades joined against [the few carried rows of earlier ranks] + [this rank's quotes] + [those of later ranks] WITHOUT
        putting them into one table (that copy is the whole quote shard): the carried rows become the merge kernel's carry
        tables, the answer's row numbers below len(earlier rows) point into them, then the shard's, then the later ones, and the
        payload is gathered from all three.  None when the shapes call for the plain path (dictionary payload columns that
        differ, symbol sets beyond the kernel's table)."""
        E = concat_tables(earlier) if earlier else None
        F = concat_tables(later) if later else None
        carried = [x for x in (E, F) if x is not None]
        payload = [c for c in quotes.column_names if c not in (self.time_col_quotes, self.symbol_col_quotes)]
        if any((x[c].dictionary is not None or quotes[c].dictionary is not None) and x[c].dictionary != quotes[c].dictionary
               for x in carried for c in payload):
            return None
        sym = self.symbol_col_quotes
        sq, st_ = quotes[sym], trades[self.symbol_col_trades]
        parts = [x for x in (E, quotes, F) if x is not None]
        if sq.dictionary is not None or st_.dictionary is not None or any(x[sym].dictionary is not None for x in carried):
            both = concat_tables([x.select([sym]) for x in parts])     # one dictionary for all
            codes = self._codes.codes(both[sym])
            split = list(torch.split(codes, [len(x) for x in parts]))
        else:
            split = [self._codes.codes(x[sym]) for x in parts]
        e_codes = split.pop(0) if E is not None else None
        q_codes = split.pop(0)
        f_codes = split.pop(0) if F is not None else None
        t_codes = self._codes.codes(st_)
        n_by, dev = max(1, self._codes.n_by), trades.device
        lt, rt = trades[self.time_col_trades].data, quotes[self.time_col_quotes].data
        _require_int64_time(lt, rt)
        ne, nq = len(E) if E is not None else 0, len(quotes)
        none_t, none_b = torch.empty(0, dtype=torch.int64, device=dev), torch.empty(0, dtype=torch.int32, device=dev)
        kw = self._strategy_args(trades[self.time_col_trades])
        back = fwd = None
        if E is not None:
            _, back = ops.asof_merge(none_t, none_b, E[self.time_col_quotes].data, e_codes, n_by, want_carry=True)
            if back is None:
                return None
            if kw:
                kw["carry_time"] = E[self.time_col_quotes].data[back.clamp(min=0).long()]
        if F is not None:
            _, fwd = ops.asof_merge(none_t, none_b, F[self.time_col_quotes].data, f_codes, n_by, None, ne + nq, want_carry=True,
                                    strategy="forward")
            if fwd is None:
                return None
            kw["carry_fwd"], kw["carry_fwd_time"] = fwd, F[self.time_col_quotes].data[(fwd - ne - nq).clamp(min=0).long()]
        ridx, _ = ops.asof_merge(lt, t_codes, rt, q_codes, n_by, back, ne, **kw)
        if ridx is None:
            return None
        in_shard = (ridx >= ne) & (ridx < ne + nq)
        side = concat_tables([x.select(payload) for x in carried]) if len(carried) > 1 else carried[0].select(payload)
        from_shard = quotes.select(payload).gather(torch.where(in_shard, ridx - ne, torch.full_like(ridx, -1)))
        from_carry = side.gather(torch.where(in_shard, torch.full_like(ridx, -1), torch.where(ridx >= ne + nq, ridx - nq, ridx)))
        valid = (ridx >= 0).to(torch.uint8)
        if os.environ.get("QK_DEBUG_ASOF"):
            print(f"[asof] carried join: {ne + len(F) if F is not None else ne} carried rows, {int((~in_shard & (ridx >= 0)).sum())} answers from them",
                  flush=True)
        right = {n: DeviceColumn(torch.where(in_shard, from_shard[n].data, from_carry[n].data), from_shard[n].dictionary,
                                 from_shard[n].arrow_type, valid) for n in payload}
        return _append_right(trades, right, self.suffix)

    def done(self, executor_id):
        if self._over_time_ranges():
            return self._join_time_ranges()
        if self._by_source is not None:
            for sid, tcol, by in ((0, self.time_col_trades, self.symbol_col_trades), (1, self.time_col_quotes, self.symbol_col_quotes)):
                t = self._by_source[sid].take()
                if t is None:
                    continue
                _require_sorted(t[tcol].data, "as-of join: the producer ranks do not hold consecutive time ranges of a sorted stream")
                t = t.with_column(self.BY, DeviceColumn(self._codes.codes(t[by])))
                if sid == 0:
                    self.trade_state = t
                else:
                    self.quote_state = t
            self._by_source = None
        if self.trade_state is None or len(self.trade_state) == 0:
            return None
        if self.quote_state is None:
            raise L.QkError("as-of join: no quotes were received")
        out = self._join(self.trade_state, None)
        self.trade_state = None
        return out


# ---------------------------------------------------------------------------------------------- time-series windows
class _KeySegmented(Executor):
    """Input handling shared by the done-time operators over an OrderedStream hash-partitioned by a key (the windows, the
    pattern search): batches are kept per source rank in arrival order (ranks hold consecutive time ranges), put back together
    and checked to be time-sorted, and the rows are segmented by key with the stable partition kernel, so time order survives
    inside a key.  The pieces are _SourceRanks, _require_sorted and KeyCodes."""

    silent_streams = "all"       # the answer is computed when the channel's input is complete

    def _init_segments(self):
        self._input = _SourceRanks()
        self._codes = KeyCodes()

    def execute(self, batches, stream_id, executor_id):
        self._input.add(_clean(batches))

    def _sorted_input(self, time_col: str, who: str):
        """(the whole input as one table, its time column as int64), or None when nothing arrived."""
        t = self._input.take()
        if t is None:
            return None
        time = t[time_col].data.to(torch.int64)
        _require_sorted(time, f"{who}: the stream is not sorted by " + time_col)
        return t, time

    def _segment(self, codes: torch.Tensor, columns: list):
        """(columns moved into key-segmented order, segment starts int64[n_by + 1], n_by)."""
        n_by = max(1, self._codes.n_by)
        dest, seg = ops.partition_plan(codes, n_by, L.PART_CODE)
        return ops.scatter(columns, dest), seg, n_by

    def _time_column(self, time: torch.Tensor, tcol: DeviceColumn) -> DeviceColumn:
        return DeviceColumn(time.to(tcol.data.dtype), None, tcol.arrow_type)


class _WindowExecutor(_KeySegmented):
    """Common part of the three window executors (pyquokka/executors/ts_executors.py:12-288): the stream arrives sorted by
    time and hash-partitioned by the `by` column; the rows are segmented by key with the stable partition kernel (time order
    survives inside a key) and the window kernel of the subclass runs over the segments.  The windows are evaluated when the
    channel's input is complete (done()): the same rows, whatever the batching -- the reference's incremental emission
    loses rows of hopping windows across batch boundaries (ts_executors.py:41-58 keeps only rows past the last complete
    window although earlier rows still belong to later windows)."""

    def __init__(self, time_col, by_col, window, trigger) -> None:
        from .windowtypes import Trigger, Window
        assert issubclass(type(window), Window) and issubclass(type(trigger), Trigger)
        self.time_col, self.by_col, self.window, self.trigger = time_col, by_col, window, trigger
        self.state = None
        self._init_segments()

    def _segmented(self):
        """(time, by codes, seg, n_by, fp64 value columns, aggregate list, decode) in key-segmented order, or None."""
        got = self._sorted_input(self.time_col, "windowed_transform")
        if got is None:
            return None
        t, time = got
        tcol = t[self.time_col]
        bycol = t[self.by_col]
        codes = self._codes.codes(bycol)
        aggs = self.window.parsed()
        exprs, vals = [], []
        for _, op, arg in aggs:                                   # one fp64 column per distinct argument expression
            if arg is not None and arg.sql() not in exprs:
                exprs.append(arg.sql())
                e = EdgeOps(None, {"__v": arg}).apply(t.select(sorted(arg.columns(), key=t.column_names.index)), stable=True)
                vals.append(to_f64(e["__v"].data))
        moved, seg, n_by = self._segment(codes, [time, codes] + vals)
        spec = [(name, op, exprs.index(arg.sql()) if arg is not None else -1) for name, op, arg in aggs]
        return moved[0], moved[1], seg, n_by, moved[2:], spec, (bycol, tcol, _time_unit(tcol))


_WIN = {"sum": L.WIN_SUM, "min": L.WIN_MIN, "max": L.WIN_MAX, "count": L.WIN_COUNT, "avg": L.WIN_AVG}


def _int_result(op: str, v: torch.Tensor) -> DeviceColumn:
    return DeviceColumn(torch.round(v).to(torch.int64)) if op == "count" else DeviceColumn(v)


class SlidingWindowExecutor(_WindowExecutor):
    """ts_executors.py:147-195: for every row, the aggregates over the rows of its key with time in (t - size_before, t]
    (Polars groupby_rolling(period=size, by=key), closed on the right).  Output: time, key, one column per aggregate."""

    def done(self, executor_id):
        seg_in = self._segmented()
        if seg_in is None:
            return None
        time, codes, seg, n_by, vals, spec, (bycol, tcol, unit) = seg_in
        size = self.window.ticks(self.window.size_before, unit)
        outs = ops.window_sliding(time, codes, seg, n_by, size, vals, [(_WIN[op], max(src, 0)) for _, op, src in spec])
        cols = {self.time_col: self._time_column(time, tcol), self.by_col: self._codes.column(codes, bycol)}
        for (name, op, _), o in zip(spec, outs):
            cols[name] = _int_result(op, o)
        return DeviceTable(cols)


class _HashedWindow(_WindowExecutor):
    def _aggregate(self, keys: list, vals: list, spec: list):
        """hash aggregate on `keys` of the per-row values: returns (key columns, {name: column}) in the table's own order."""
        need = []                                             # (hash-aggregate op, value index)
        for _, op, src in spec:
            for h in {"sum": ["sum"], "avg": ["sum"], "min": ["min"], "max": ["max"], "count": []}[op]:
                if (h, src) not in need:
                    need.append((h, src))
        n = keys[0].numel()
        ha = ops.HashAggState([k.dtype for k in keys], [_AGG_OPS[h] for h, _ in need], max(1 << 12, 2 * n), keys[0].device)
        ha.update(keys, [vals[src] for _, src in need])
        ok, ov, oc = ha.finalize()
        out = {}
        for name, op, src in spec:
            if op == "count":
                out[name] = DeviceColumn(oc)
            elif op == "avg":
                out[name] = DeviceColumn(ov[need.index(("sum", src))] / oc.to(torch.float64))
            else:
                out[name] = DeviceColumn(ov[need.index((op, src))])
        return ok, out


    def _per_event(self, kind: int, length, key_first: bool):
        """OnEventTrigger (ts_executors.py:64-96, 109-136, 239-288: DuckDB's PARTITION BY key, window ORDER BY time RANGE
        UNBOUNDED PRECEDING): one row per input row, in key-segmented order, with its own time and the aggregates of its
        window's rows with time <= its own (qk_window_running).  `length` is the tumbling size or the session timeout; a
        timedelta is converted with Window.ticks in the time column's unit (the reference divides the int64 timestamp by
        total_seconds())."""
        seg_in = self._segmented()
        if seg_in is None:
            return None
        time, codes, seg, n_by, vals, spec, (bycol, tcol, unit) = seg_in
        outs = ops.window_sliding(time, codes, seg, n_by, self.window.ticks(length, unit), vals,
                                  [(_WIN[op], max(src, 0)) for _, op, src in spec], run=kind)
        key, tc = self._codes.column(codes, bycol), self._time_column(time, tcol)
        cols = {self.by_col: key, self.time_col: tc} if key_first else {self.time_col: tc, self.by_col: key}
        for (name, op, _), o in zip(spec, outs):
            cols[name] = _int_result(op, o)
        return DeviceTable(cols)


class HoppingWindowExecutor(_HashedWindow):
    """ts_executors.py:12-145: aggregates per key over the windows [k * hop, k * hop + size) (Polars groupby_dynamic(every=hop,
    period=size, by=key): closed on the left, labelled by the window start, windows before the key's first truncated
    timestamp are not produced, empty windows neither).  TumblingWindow = hop == size.  Output: time (window start), key, aggregates.
    A TumblingWindow with OnEventTrigger gives one row per input row instead (_per_event): time, key and the aggregates of the
    row's window [k * size, (k + 1) * size) up to its time; computed in done(), like every window here, not as the rows stream."""

    def __init__(self, time_col, by_col, window, trigger) -> None:
        from .windowtypes import HoppingWindow, OnEventTrigger, TumblingWindow
        assert issubclass(type(window), HoppingWindow)
        super().__init__(time_col, by_col, window, trigger)
        if type(trigger) == OnEventTrigger and not isinstance(window, TumblingWindow):
            raise Exception("OnEventTrigger is not supported for hopping windows")

    def done(self, executor_id):
        from .windowtypes import OnEventTrigger
        if type(self.trigger) == OnEventTrigger:
            return self._per_event(L.WIN_RUN_TUMBLING, self.window.size, key_first=False)
        seg_in = self._segmented()
        if seg_in is None:
            return None
        time, codes, seg, n_by, vals, spec, (bycol, tcol, unit) = seg_in
        size, hop = self.window.ticks(self.window.size, unit), self.window.ticks(self.window.hop, unit)
        wstart, key, src = ops.window_hop_expand(time, codes, seg, n_by, size, hop)
        prog = lambda i: [(L.OP_COL, i, 0, 0.0, 0)]
        (wstart, key, src), m = ops.scan_filter_project([wstart, key, src], [(L.OP_CMP_COL_IMM, 2, L.CMP_GE, 0.0, 0)], [prog(0), prog(1), prog(2)], stable=True)
        if m == 0:
            return None
        gathered = ops.gather(vals, src) if vals else []
        ok, out = self._aggregate([key, wstart], gathered, spec)
        cols = {self.time_col: self._time_column(ok[1], tcol), self.by_col: self._codes.column(ok[0], bycol)}
        cols.update(out)
        return DeviceTable(cols)


class SessionWindowExecutor(_HashedWindow):
    """ts_executors.py:197-288: per key, a session = a run of rows whose gaps are all <= timeout; aggregates per session.
    Output: key, time (the session's first timestamp; the reference emits its internal window id instead), aggregates.
    With OnEventTrigger one row per input row instead (_per_event): key, time and the aggregates of the row's session up to
    its time.  The time column is `order_by` (the reference's per-event path reads a column named "ts", ts_executors.py:228),
    and the result is computed in done(), not as the rows stream."""

    def __init__(self, time_col, by_col, window, trigger) -> None:
        from .windowtypes import SessionWindow
        assert issubclass(type(window), SessionWindow)
        super().__init__(time_col, by_col, window, trigger)

    def done(self, executor_id):
        from .windowtypes import OnEventTrigger
        if type(self.trigger) == OnEventTrigger:
            return self._per_event(L.WIN_RUN_SESSION, self.window.timeout, key_first=True)
        seg_in = self._segmented()
        if seg_in is None:
            return None
        time, codes, seg, n_by, vals, spec, (bycol, tcol, unit) = seg_in
        ids = ops.window_session_ids(time, codes, self.window.ticks(self.window.timeout, unit))
        ok, out = self._aggregate([ids], vals, spec)
        # the first row of session s (ids are 1-based and increase along the segmented order)
        starts = torch.nonzero(torch.diff(ids, prepend=ids[:1] - 1)).flatten()
        at = starts[ok[0] - 1]
        cols = {self.by_col: self._codes.column(codes[at], bycol), self.time_col: self._time_column(time[at], tcol)}
        cols.update(out)
        return DeviceTable(cols)


# ---------------------------------------------------------------------------------------------- pattern recognition
class CEPExecutor(_KeySegmented):
    """OrderedStream.pattern_recognize (pyquokka/executors/cep_executors.py:13-181; the reference's constructor order, plus `by`).
    Per key, in time order, every row r0 satisfying event 0 that starts at least one match -- rows r0 < r1 < ... < r(m-1) with
    strictly increasing times, t(r(m-1)) <= t(r0) + max_span and event i's predicate true with r0 .. r(i-1) bound to the earlier
    names -- gives one output row: the key and the times of the match whose (t1 .. t(m-1)) is lexicographically smallest.
    Done-time: the channel's rows are segmented by key, the row-local conjuncts of every event are evaluated by the scan kernel
    into a candidate mask, and qk_pattern_search runs the search.  A predicate that reads a NULL is false.
    `touched_columns` and `prefilter` (the OR of the events' row-local parts, pushed to the scan by the planner) as in the reference."""

    BUDGET = 1 << 24             # rows one start may test before the search gives up on it and the query fails

    def __init__(self, schema, events, time_col, max_span, by) -> None:
        import datetime
        if isinstance(max_span, bool) or not isinstance(max_span, (int, datetime.timedelta)):
            raise E.ExprError("maxspan must be an int in the time column's unit or a datetime.timedelta")
        if (max_span.total_seconds() if isinstance(max_span, datetime.timedelta) else max_span) < 0:
            raise E.ExprError("maxspan must be >= 0")
        assert time_col in schema and by in schema
        self.time_col, self.by_col, self.max_span = time_col, by, max_span
        self.preds = E.split_pattern(events, schema, by)
        self.names = list(self.preds.names)
        self.touched_columns = set(self.preds.columns) | {time_col, by}
        self.prefilter = E.pattern_prefilter(self.preds)
        E.compile_links(self.preds)              # the link programs' errors while the plan is built, not after the input is read
        self._init_segments()

    def explain(self) -> str:
        ev = ", ".join(f"{n}: {'*' if lo is None and li is None else ' and '.join(x.sql() for x in (lo, li) if x is not None)}"
                       for n, lo, li in zip(self.names, self.preds.local, self.preds.link))
        return f"pattern_recognize [{ev}] maxspan={self.max_span} by={self.by_col}"

    def _ticks(self, tcol: DeviceColumn) -> int:
        import datetime
        from .windowtypes import Window
        if isinstance(self.max_span, datetime.timedelta) and tcol.arrow_type is not None and pa.types.is_date32(tcol.arrow_type):
            days = self.max_span / datetime.timedelta(days=1)
            if not float(days).is_integer():
                raise E.ExprError("maxspan over a date column must be a whole number of days")
            return int(days)
        return Window.ticks(self.max_span, _time_unit(tcol))

    def _empty(self, tcol: DeviceColumn, bycol: DeviceColumn, dev) -> DeviceTable:
        none = torch.empty(0, dtype=torch.int64, device=dev)
        return DeviceTable({self.by_col: self._codes.column(none.to(torch.int32), bycol)} |
                           {n: self._time_column(none, tcol) for n in self.names})

    def search_inputs(self, t: DeviceTable, time: torch.Tensor) -> dict:
        """The arguments of ops.pattern_search for the rows of `t` (time = its time column as int64): the rows segmented by key,
        the candidate mask from the row-local conjuncts, the start rows and the link programs.  None when no row starts a match."""
        tcol, bycol = t[self.time_col], t[self.by_col]
        codes = self._codes.codes(bycol)
        read = sorted(self.preds.columns, key=t.column_names.index)
        plain, mask_of = t.select(read).split_validity()
        hidden = sorted(set(mask_of.values()))
        names = read + hidden
        moved, seg, n_by = self._segment(codes, [time, codes] + [plain[c].data for c in names])
        stime, scodes = moved[0], moved[1]
        seg_t = DeviceTable({c: DeviceColumn(d, plain[c].dictionary, plain[c].arrow_type) for c, d in zip(names, moved[2:])})
        dev, m, n = stime.device, len(self.names), len(stime)
        # ---- row-local conjuncts: one scan projection per event, packed into the candidate mask (bit e: may bind event e)
        cand = torch.zeros(n, dtype=torch.uint8, device=dev)
        local = {}
        for e, node in enumerate(self.preds.local):
            if node is None:
                cand |= 1 << e
                continue
            nulls = sorted({mask_of[c] for c in node.columns() if c in mask_of})
            local[e] = E.and_all([node] + [E.binop("!=", E.col(h), E.num(0)) for h in nulls])
        if local and n:
            used = sorted(set().union(*[x.columns() for x in local.values()]), key=names.index)
            sub = seg_t.select(used)
            sch = sub.schema_info()
            progs = {e: E.compile_expr(x, sch) for e, x in local.items()}
            groups, cur = [], []
            for e in progs:                                   # as many projections per scan call as its limits take
                if cur and sum(len(progs[k]) for k in cur) + len(progs[e]) > L.MAX_TOTAL_NODES:
                    groups.append(cur)
                    cur = []
                cur.append(e)
            groups.append(cur)
            for g in groups:
                outs, _ = ops.scan_filter_project([sub[c].data for c in used], None, [progs[e] for e in g], stable=True)
                for e, o in zip(g, outs):
                    cand |= (o != 0).to(torch.uint8) << e
        starts = torch.nonzero(cand & 1).flatten().to(torch.int32)
        if starts.numel() == 0:
            return None
        # ---- link conjuncts: one program per event over the columns they read
        lcols, links = E.compile_links(self.preds, seg_t.schema_info())
        return dict(time=stime, by=scodes, seg=seg, n_by=n_by, cand=cand, starts=starts, m=m, maxspan=self._ticks(tcol),
                    link_cols=[seg_t[c].data for c in lcols], link_valid=[seg_t[mask_of[c]].data if c in mask_of else None for c in lcols],
                    links=links, budget=self.BUDGET)

    def done(self, executor_id):
        got = self._sorted_input(self.time_col, "pattern_recognize")
        if got is None:
            return None
        t, time = got
        tcol, bycol = t[self.time_col], t[self.by_col]
        a = self.search_inputs(t, time)
        if a is None:
            return self._empty(tcol, bycol, time.device)
        starts, stime, scodes = a["starts"], a["time"], a["by"]
        try:
            bound = ops.pattern_search(**a)
        except ops.PatternBudgetError as err:
            r = int(starts[err.index].item())
            code = int(scodes[r].item())
            key = self._codes.values[code] if self._codes.values is not None else code
            raise L.QkError(f"pattern_recognize: the search from the row of key {key!r} at time {int(stime[r].item())} tested more "
                            f"than {self.BUDGET} rows; narrow the pattern (maxspan, more selective predicates)") from err
        keep = torch.nonzero(bound[:, 0] >= 0).flatten()
        bound = bound[keep]
        if bound.shape[0] == 0:
            return self._empty(tcol, bycol, time.device)
        out = {self.by_col: self._codes.column(ops.gather([scodes], bound[:, 0].contiguous())[0], bycol)}
        for e, name in enumerate(self.names):
            out[name] = self._time_column(ops.gather([stime], bound[:, e].contiguous())[0], tcol)
        return DeviceTable(out)


# ---------------------------------------------------------------------------------------------- shift (lag / lead)
_INT_RANGE = {torch.uint8: (0, 255), torch.int32: (-(1 << 31), (1 << 31) - 1), torch.int64: (-(1 << 63), (1 << 63) - 1)}


def shift_fill(col: DeviceColumn, name: str, value):
    """`value` as column `name` stores it, for the rows of OrderedStream.shift without a source -> (the stored value, the
    output dictionary).  None stays None (NULL); a string joins a copy of the column's dictionary when it is not in it yet.
    A value the column cannot hold raises QkError."""
    import datetime
    import numbers
    dictionary = col.dictionary
    if value is None:
        return None, dictionary
    at, dt = col.arrow_type, col.data.dtype

    def bad():
        return L.QkError(f"shift: fill value {value!r} cannot be stored in column {name!r} ({at or dt})")
    if dictionary is not None:
        if not isinstance(value, str):
            raise bad()
        if value not in dictionary:
            dictionary = list(dictionary) + [value]
        return dictionary.index(value), dictionary
    if at is not None and pa.types.is_boolean(at):
        if not isinstance(value, bool):
            raise bad()
        return int(value), None
    if isinstance(value, bool):
        raise bad()
    if at is not None and (pa.types.is_date(at) or pa.types.is_timestamp(at)):
        if isinstance(value, numbers.Integral):                     # days / milliseconds / the timestamp's unit
            v = int(value)
        elif pa.types.is_timestamp(at) and isinstance(value, datetime.datetime):
            try:
                v = pa.scalar(value, type=at).value
            except (pa.ArrowInvalid, pa.ArrowTypeError, OverflowError, ValueError):
                raise bad() from None
        elif pa.types.is_date(at) and isinstance(value, datetime.date) and not isinstance(value, datetime.datetime):
            v = (value - datetime.date(1970, 1, 1)).days * (1 if pa.types.is_date32(at) else 86_400_000)
        else:
            raise bad()
    elif dt in (torch.float32, torch.float64):
        if not isinstance(value, numbers.Real):
            raise bad()
        return float(value), None
    elif isinstance(value, numbers.Integral):
        v = int(value)
    else:
        raise bad()
    lo, hi = _INT_RANGE.get(dt, (1, 0))
    if not lo <= v <= hi:
        raise bad()
    return v, None


class ShiftExecutor(Executor):
    """OrderedStream.shift (pyquokka/orderedstream.py:13-35; the reference never defines its ShiftOperator, so the semantics are
    Polars' pl.all().shift(n, fill_value).over(by)): every row receives the values of `columns` from the row n places earlier
    (n > 0) or |n| later (n < 0) among the rows of its `by` key in stream order -- rank order, then arrival order -- or the fill.
    Rows stay where they are; answered in done(), by one path at every world size:
      * each rank holds a contiguous piece of the stream (sort(), sorted readers, from_device(sorted_by=...), or a hash edge on
        `by`), so nothing is shuffled.  A rank that has later (earlier) ranks flags the last n rows of each of its keys (first
        |n| for a lead; qk_shift_plan with want_edge) and sends them to every later (earlier) rank -- at most |n| x keys rows;
      * every rank then plans over the KeyCodes codes of [earlier ranks' tails in rank order | own rows] (lead: [own rows |
        later ranks' heads]) -- the stable code partition and qk_shift_plan (source rows and the order check in one pass) --
        and gathers the payload from its shard and from that small boundary table (qk_shift_gather, every shifted column in
        one launch); unshifted columns are passed on as they are.  At one rank there is no boundary table.
    A key with fewer than |n| rows on the neighbouring rank still finds its rows, because the tails of ALL earlier ranks
    arrive.  String payload columns of the boundary table are re-coded onto the shard's dictionary (new entries appended);
    the shard is not re-coded.
    When `time_col` (the stream's sorted_by) is an integer, date or timestamp column, rows of a key whose time falls below the
    previous row's raise QkError, across rank boundaries too (NULL times count as the largest, where sort() puts them)."""

    silent_streams = "all"
    ordered_output = True            # rows stay in place: rank r's rows precede rank r + 1's
    HUGE = 1 << 31                   # |n| at or above this: no row has a source

    def __init__(self, n, by, fill_value, columns, suffix=None, time_col=None) -> None:
        self.n, self.by, self.fill_value, self.columns = int(n), by, fill_value, list(columns)
        self.suffix, self.time_col = suffix, time_col
        self._batches = []
        self._codes = KeyCodes()
        self.state = None

    def explain(self) -> str:
        return (f"shift n={self.n} by={self.by} columns={self.columns}" + (f" suffix={self.suffix}" if self.suffix else "")
                + (f" checked on {self.time_col}" if self.time_col else ""))

    def execute(self, batches, stream_id, executor_id):
        self._batches.extend(_clean(batches))

    def _fill_of(self, c):
        return self.fill_value.get(c) if isinstance(self.fill_value, dict) else self.fill_value

    def _time(self, t: DeviceTable):
        """The column the order check reads as int64 (NULL = largest), or None when there is nothing to check."""
        if self.time_col is None or self.time_col not in t:
            return None
        c = t[self.time_col]
        if c.dictionary is not None or c.is_vector or c.data.dtype not in (torch.int32, torch.int64):
            return None
        time = c.data.to(torch.int64)
        if c.valid is not None:
            time = torch.where(c.valid.bool(), time, torch.full_like(time, (1 << 63) - 1))
        return time

    def _key_codes(self, t: DeviceTable) -> torch.Tensor:
        col = t[self.by]
        if col.dictionary is None and col.data.dtype not in (torch.uint8, torch.int32, torch.int64):
            raise L.QkError(f"shift: `by` column {self.by!r} must be a string column or integer codes")
        return self._codes.codes(col)

    def _gather(self, t: DeviceTable, boundary: DeviceTable | None, src: torch.Tensor) -> DeviceTable:
        a, b, av, bv, fills, dicts = [], [], [], [], [], []
        for c in self.columns:
            col = t[c]
            if col.is_vector:
                raise L.QkError(f"shift: column {c!r} is a vector column")
            ad, bcol = col.data, boundary[c] if boundary is not None else None
            bd, dic = (bcol.data if bcol is not None else None), col.dictionary
            if dic is not None and bcol is not None and bcol.dictionary != dic:
                dic = list(dic)                                       # the boundary's strings join the shard's dictionary
                index = {v: i for i, v in enumerate(dic)}
                lut = []
                for v in bcol.dictionary:
                    if v not in index:
                        index[v] = len(dic)
                        dic.append(v)
                    lut.append(index[v])
                bd = torch.tensor(lut or [0], dtype=torch.int64, device=ad.device)[bd.long()]
            fill, dic = shift_fill(DeviceColumn(ad, dic, col.arrow_type), c, self._fill_of(c))
            if dic is not None and len(dic) > 255 and ad.dtype == torch.uint8:
                ad = ad.to(torch.int32)                               # codes past 255 need a wider column
            if bd is not None and bd.dtype != ad.dtype:
                bd = bd.to(ad.dtype)
            a.append(ad)
            b.append(bd)
            av.append(col.valid)
            bv.append(bcol.valid if bcol is not None else None)
            fills.append(fill)
            dicts.append(dic)
        outs, valids = ops.shift_gather(a, b if boundary is not None else None, src, fills, av, bv)
        cols = dict(t.columns)
        for c, o, v, dic in zip(self.columns, outs, valids, dicts):
            cols[c if self.suffix is None else c + self.suffix] = DeviceColumn(o, dic, t[c].arrow_type, v)
        return DeviceTable(cols)

    def _unchanged(self, t: DeviceTable) -> DeviceTable:
        if self.suffix is None:
            return t
        return DeviceTable(dict(t.columns) | {c + self.suffix: t[c] for c in self.columns})

    def _plan(self, n: int, nrows: int, codes: torch.Tensor | None, **kw):
        """ops.shift_plan over the key codes `codes` (None: the whole stream is one key) and their stable code partition."""
        if codes is None:
            return ops.shift_plan(n, nrows, **kw)
        n_by = max(1, self._codes.n_by)
        return ops.shift_plan(n, nrows, codes, n_by, *ops.partition_plan(codes, n_by, L.PART_CODE), **kw)

    def done(self, executor_id):
        from . import runtime as RT
        t, self._batches = (concat_tables(self._batches) if self._batches else None), []
        if self.n == 0:
            self.state = self._unchanged(t) if t is not None else None
            return self.state
        w, me, dev = RT.world_size(), RT.rank(), default_device()
        ex = RT.Exchange(dev)
        lag = self.n > 0
        receivers = range(me + 1, w) if lag else range(me)              # the ranks that need this rank's boundary rows
        # a shift past 2^31 rows has no sources; the boundary then only serves the order check: one row per key
        edge_n = self.n if abs(self.n) < self.HUGE else (1 if lag else -1)
        na = len(t) if t is not None else 0
        boundary = codes = time = None
        if na:
            time = self._time(t)
            codes = self._key_codes(t) if self.by is not None else None
        if na and len(receivers):
            _, edge, _ = self._plan(edge_n, na, codes, lo=0, hi=0, want_edge=True, device=t.device)
            rows = torch.nonzero(edge).flatten().to(torch.int32)
            if rows.numel():
                need = list(dict.fromkeys(self.columns + ([self.by] if self.by is not None else [])
                                          + ([self.time_col] if time is not None else [])))
                boundary = t.select(need).gather(rows)
        got = ex.to_ranks(boundary, ("shift-boundary", id(self)), ranks=receivers)
        B = concat_tables(got) if got else None
        nb = len(B) if B is not None else 0
        bad = 0
        if na:
            lo = nb if lag else 0
            allcodes, alltime = codes, None
            if nb and self.by is not None:
                bcodes = self._key_codes(B)
                allcodes = torch.cat([bcodes, codes] if lag else [codes, bcodes])
            if time is not None:
                btime = self._time(B) if nb else None
                alltime = time if btime is None else torch.cat([btime, time] if lag else [time, btime])
            src, _, bad = self._plan(self.n, na + nb, allcodes, lo=lo, hi=lo + na, time=alltime, device=t.device)
        if ex.max_over_ranks([int(bad or 0)])[0]:          # every rank raises, or none does
            raise L.QkError(f"shift: the stream is not sorted by {self.time_col}")
        self.state = self._gather(t, B if nb else None, src) if na else None
        return self.state
