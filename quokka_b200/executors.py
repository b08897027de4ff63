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
from .columns import DeviceColumn, DeviceTable, as_device_table, concat_tables, default_device, unify_dictionaries
from .edge import EdgeOps, agg_result_type, restore_type, to_f64


class Executor:
    """pyquokka/executors/base_executor.py:26-32."""

    def __init__(self) -> None:
        raise NotImplementedError

    def execute(self, batches, stream_id, executor_id):
        raise NotImplementedError

    def done(self, executor_id):
        raise NotImplementedError


def _retire(state):
    """A state buffer replaced while chunks are in flight on several lanes: it may have been allocated on another lane's
    stream, so the allocator must not hand it out again before the kernels queued on THIS stream have read it."""
    for t in (getattr(state, "state", None), getattr(state, "overflow", None)):
        if isinstance(t, torch.Tensor) and t.is_cuda:
            t.record_stream(torch.cuda.current_stream())


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
        import os
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


def _join_output(probe: DeviceTable, build: DeviceTable | None, pi, bi, left_on, right_on, how, suffix):
    out = probe.gather(pi)
    if how in ("semi", "anti") or build is None:
        return out
    right = build.drop([right_on]).gather(bi)
    valid = None
    if how == "left":
        valid = (bi >= 0).to(torch.uint8)
        right = right.with_validity(valid)
    cols = dict(out.columns)
    for n, c in right.columns.items():
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


def _world() -> int:
    import torch.distributed as dist
    return dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1


def _build_key(build_col: DeviceColumn) -> torch.Tensor:
    return build_col.data.to(torch.int32) if build_col.dictionary is not None else _float_key(build_col.data)


class BuildProbeJoinExecutor(Executor):
    silent_streams = (1,)        # build batches never produce output: nothing to push downstream after them

    """sql_executors.py:325-377.  stream 1 = build (right), stream 0 = probe (left); every build batch
    must arrive before the first probe batch (assert, :357); how in inner/left/semi/anti; the result
    keeps the left key (renamed to the right key when key_to_keep == "right", :372-373); an anti join
    against an empty build side passes the probe through, the others emit nothing (:362-366)."""

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
        self._table = None

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

    def _freeze_build(self):
        if self._table is not None:
            return
        self.state = concat_tables(self._pending)
        self._pending = []
        key = self.state[self.right_on].data
        if key.dtype not in (torch.uint8, torch.int32, torch.int64, torch.float64):
            raise L.QkError(f"join key {self.right_on!r} must be an integer / date / fp64 column (got {key.dtype})")
        self._table = ops.JoinTable(len(self.state), key.device)
        self._table.build(_build_key(self.state[self.right_on]))
        self._table.check_flags()

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
                return
            if self.phase == "build":
                self._freeze_build()
            self.phase = "probe"
            key = _probe_key(batch[self.left_on], self.state[self.right_on], f"join {self.left_on} = {self.right_on}")
            pi, bi = self._table.probe(key, _HOW[self.how])
            result = _join_output(batch, self.state, pi, bi, self.left_on, self.right_on, self.how, "_right")
            if self.key_to_keep == "right":
                result = result.rename({self.left_on: self.right_on})
            return result

    def done(self, executor_id):
        pass


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
        self._table = None

    def execute(self, batches, stream_id, executor_id):
        batches = _clean(batches)
        if len(batches) == 0:
            return
        batch = concat_tables(batches)
        if self._table is None:                         # opened lazily on first execute (tutorial.md:56)
            self.state = as_device_table(self._small_src)
            self._table = ops.JoinTable(len(self.state), batch.device)
            self._table.build(_build_key(self.state[self.small_on]))
            self._table.check_flags()
        key = _probe_key(batch[self.big_on], self.state[self.small_on], f"join {self.big_on} = {self.small_on}")
        pi, bi = self._table.probe(key, _HOW[self.how])
        return _join_output(batch, self.state, pi, bi, self.big_on, self.small_on, self.how, self.suffix)

    def done(self, executor_id):
        return


# ---------------------------------------------------------------------------------------------- aggregates
_AGG_OPS = {"sum": L.AGG_SUM, "min": L.AGG_MIN, "max": L.AGG_MAX}


def _to_f64(col: DeviceColumn) -> torch.Tensor:
    return to_f64(col.data)


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
        self._ha = None
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
        vals = [_to_f64(batch[c]) for _, c in self.calls]
        if not self.groupby_keys:
            if self._dense is None:
                self._dense = ops.DenseAggState([], [_AGG_OPS[f] for f, _ in self.calls], batch.device)
            cols_in = vals or [torch.zeros(len(batch), dtype=torch.uint8, device=batch.device)]
            self._dense.update(cols_in, None, [], [[(L.OP_COL, i, 0, 0.0, 0)] for i in range(len(vals))], variant=1)
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
        if self._ha is None:
            self._ha = ops.HashAggState([k.data.dtype for k in keys], [_AGG_OPS[f] for f, _ in self.calls],
                                        max(1 << 16, 2 * len(batch)), batch.device)
        elif self._ha.rows_seen + len(batch) > self._ha.capacity // 2:
            self._grow(len(batch))
        self._ha.update([k.data for k in keys], vals)

    def _grow(self, incoming):
        """Re-insert the current groups into a table twice as large (SUM/MIN/MAX are all re-foldable)."""
        ok, ov, oc = self._ha.finalize()
        new = ops.HashAggState(self._ha.key_dtypes, [_AGG_OPS[f] for f, _ in self.calls],
                               max(4 * (len(ok[0]) + incoming), 2 * self._ha.capacity), self._ha.device)
        if len(ok[0]):
            new.update(ok, ov)
        new.rows_seen = len(ok[0])
        _retire(self._ha)
        self._ha = new

    def done(self, executor_id):
        if self._ha is None and self._dense is None:
            return None
        if self._dense is not None:
            acc = self._dense.acc
            cols = {f"__a{i}": restore_type(acc[:, i].clone(), self._types[i]) for i in range(len(self.calls))}
            if not cols:
                cols = {"__n": DeviceColumn(self._dense.cnt.to(torch.float64))}
        else:
            ok, ov, _ = self._ha.finalize()
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


class DistinctExecutor(Executor):
    """sql_executors.py:517-554; emits the distinct key combinations once, at done()."""

    silent_streams = "all"

    def __init__(self, keys) -> None:
        self.keys = keys
        self.state = None
        self._ha = None
        self._meta = None

    def execute(self, batches, stream_id, executor_id):
        batches = _clean(batches)
        if len(batches) == 0:
            return
        batch = concat_tables(batches)
        keys = [batch[k] for k in self.keys]
        if self._ha is None:
            self._meta = [(k.dictionary, k.arrow_type) for k in keys]
            self._ha = ops.HashAggState([k.data.dtype for k in keys], [], max(1 << 16, 4 * len(batch)), batch.device)
        elif self._ha.rows_seen + len(batch) > self._ha.capacity // 2:
            ok, _, _ = self._ha.finalize()
            new = ops.HashAggState(self._ha.key_dtypes, [], max(4 * (len(ok[0]) + len(batch)), 2 * self._ha.capacity), batch.device)
            if len(ok[0]):
                new.update(ok, [])
            new.rows_seen = len(ok[0])
            _retire(self._ha)
            self._ha = new
        self._ha.update([k.data for k in keys], [])

    def done(self, executor_id):
        if self._ha is None:
            return
        ok, _, _ = self._ha.finalize()
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


# ---------------------------------------------------------------------------------------------- as-of
class SortedAsofExecutor(Executor):
    """ts_executors.py:324-383: streaming backward as-of join of two time-sorted streams per symbol.
    stream 0 = trades (left), stream 1 = quotes (right).  A trade can be joined as soon as a quote NEWER
    than it has been seen (every quote at or before its time has arrived by then, :359); the rest
    waits for more quotes or for done().

    The join is the sorted-merge kernel (qk_asof_merge): one sweep over the merged timeline with a per-symbol table of
    the newest quote.  The table is CARRIED between calls, so every quote row is swept once however the two streams
    are batched, and -- like the reference, which trims its quote state to the last quote per symbol (:371-376) -- quotes
    that can no longer be the newest of their symbol are dropped from the state.  Symbol sets too large for the
    shared-memory table use the partition + search kernels (qk_asof_backward) over the whole quote state."""

    TRIM_ROWS = 1 << 20          # fold swept quotes into <= n_symbols carried rows once this many have piled up

    @property
    def silent_streams(self):      # across ranks over time ranges everything is held until done(); streaming otherwise
        return "all" if (self.time_ranges and _world() > 1) else ()

    def __init__(self, time_col_trades="time", time_col_quotes="time", symbol_col_trades="symbol",
                 symbol_col_quotes="symbol", suffix="_right", time_ranges=False) -> None:
        self.time_ranges = time_ranges   # several ranks, each holding a contiguous time range of both streams: join in place (done())
        self._held = None
        self.trade_state = None
        self.quote_state = None
        self.time_col_trades = time_col_trades
        self.time_col_quotes = time_col_quotes
        self.symbol_col_trades = symbol_col_trades
        self.symbol_col_quotes = symbol_col_quotes
        self.suffix = suffix
        self._values, self._index, self._luts = None, None, {}     # the executor's own, append-only symbol codes
        self._n_by = 0
        self._carry = None           # int32[n_by]: row of quote_state holding the newest swept quote of each symbol, -1 = none
        self._swept = 0              # rows of quote_state already folded into _carry
        self._whole_state = False    # too many symbols for the merge kernel: keep every quote, search the whole state
        self._by_source = None       # several producer ranks: {stream: {source rank: [batches in arrival order]}}, joined at done()

    BY = "__by"                      # hidden column: the symbol in the executor's code space

    def _stable_codes(self, col: DeviceColumn) -> torch.Tensor:
        """Codes that mean the same symbol in every batch of both streams (batch dictionaries are re-sorted unions and
        differ from batch to batch): strings are numbered in order of first appearance, integer codes are used as is."""
        if col.dictionary is not None:
            if self._values is None:
                if self._n_by:
                    raise L.QkError("as-of `by` columns must both be strings or both be integer codes")
                self._values, self._index = [], {}
            key = (id(col.dictionary), len(col.dictionary))
            lut = self._luts.get(key)
            if lut is None:
                codes = []
                for v in col.dictionary:
                    i = self._index.get(v)
                    if i is None:
                        i = self._index[v] = len(self._values)
                        self._values.append(v)
                    codes.append(i)
                lut = (col.dictionary, torch.tensor(codes or [0], dtype=torch.int32, device=col.data.device))
                self._luts[key] = lut                               # keeps the dictionary alive, so its id stays unique
            self._n_by = max(self._n_by, len(self._values))
            return lut[1][col.data.long()]
        if self._values is not None:
            raise L.QkError("as-of `by` columns must both be strings or both be integer codes")
        codes = col.data.to(torch.int32)
        if len(codes):
            lo, hi = (int(v) for v in torch.stack(torch.aminmax(codes)).tolist())       # one pass, one read-back
            if lo < 0:
                raise L.QkError("as-of `by` codes must be non-negative")
            self._n_by = max(self._n_by, hi + 1)
        return codes

    def _append(self, state, batch, tcol):
        if state is None or len(state) == 0:
            return batch
        if len(batch) > 0:
            assert int(state[tcol].data[-1].item()) <= int(batch[tcol].data[0].item()), "stream is not time-sorted"
        return concat_tables([state, batch])

    def _carry_table(self, device) -> torch.Tensor:
        n = max(1, self._n_by)
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
        if lt.dtype != torch.int64 or rt.dtype != torch.int64:
            raise L.QkError("as-of time columns must be int64 / timestamp")
        lby, rby = trades[self.BY].data, quotes[self.BY].data
        n_by = max(1, self._n_by)
        ridx = None
        if not self._whole_state:
            carry = self._carry_table(lt.device)
            ridx, carry_out = ops.asof_merge(lt, lby, rt[self._swept:upto], rby[self._swept:upto], n_by, carry, self._swept, want_carry=True)
            if ridx is None:
                if self._swept:
                    raise L.QkError("as-of: the symbol set outgrew the merge kernel's table after quotes were trimmed")
                self._whole_state = True
            else:
                self._carry, self._swept = carry_out, upto
        if ridx is None:
            ridx = ops.asof_backward(lt, lby, rt, rby, n_by)
        right = quotes.drop([self.time_col_quotes, self.symbol_col_quotes, self.BY]).gather(ridx)
        right = right.with_validity((ridx >= 0).to(torch.uint8))
        cols = dict(trades.drop([self.BY]).columns)
        for n, c in right.columns.items():
            cols[n + self.suffix if n in cols else n] = c
        self._trim()
        return DeviceTable(cols)

    def _trim(self):
        """Swept quotes only matter as "newest of their symbol": keep those rows (<= n_symbols), drop the rest."""
        if self._whole_state or self._swept < max(self.TRIM_ROWS, 4 * self._n_by):
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
        if self.time_ranges and _world() > 1:
            if self._held is None:
                self._held = {0: [], 1: []}
            self._held[stream_id].extend(batches)
            return
        if self._by_source is not None or any(getattr(b, "src_rank", None) is not None for b in batches):
            # The batches come from several producer ranks, each holding a contiguous TIME RANGE of the sorted stream
            # (range-partitioned sorted readers, dataset/ordered_readers.py:84-100), and all ranks ship their batches at
            # once: arrival order is not time order across ranks.  Rank r's rows all precede rank r + 1's, so the
            # stream is put back together per source rank, in arrival order, and joined when it is complete.
            if self._by_source is None:
                self._by_source = {0: {}, 1: {}}
            for b in batches:
                self._by_source[stream_id].setdefault(getattr(b, "src_rank", 0) or 0, []).append(b)
            return
        batch = concat_tables(batches)
        by = self.symbol_col_trades if stream_id == 0 else self.symbol_col_quotes
        batch = batch.with_column(self.BY, DeviceColumn(self._stable_codes(batch[by])))
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
            d = t[col].data
            if d.dtype != torch.int64:
                raise L.QkError("as-of time columns must be int64 / timestamp")
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
        # ---- newest quote per symbol of every rank, to everybody
        newest = None
        if quotes is not None and len(quotes) > 0:
            codes = self._stable_codes(quotes[self.symbol_col_quotes])
            n_by = max(1, self._n_by)
            empty_t, empty_b = torch.empty(0, dtype=torch.int64, device=dev), torch.empty(0, dtype=torch.int32, device=dev)
            _, table = ops.asof_merge(empty_t, empty_b, quotes[qt].data, codes, n_by, want_carry=True)
            if table is None:                                       # symbol set too large for the table: the last row of each code
                order = torch.arange(len(codes), device=dev, dtype=torch.int64)
                table = torch.full((n_by,), -1, dtype=torch.int64, device=dev).scatter_reduce(0, codes.long(), order, "amax", include_self=True)
            idx = torch.sort(table[table >= 0]).values.to(torch.int32)          # row order = time order
            newest = quotes.gather(idx)
        got = ex({r: newest for r in range(w)} if newest is not None and len(newest) > 0 else {}, w, edge_key=("asof-newest", id(self)))
        earlier = [g for g in sorted(got, key=lambda g: g.src_rank) if g.src_rank < me]
        # ---- trades to the rank whose quote range holds them: the k-th rank that has quotes takes the trades from its first quote
        #      time up to the next such rank's (the first one also takes everything earlier: those trades match nothing, but
        #      only a rank with quotes knows the columns to fill with NULLs); ranks without quotes take none
        owners = [r for r in range(w) if rows[r][4]]
        if not owners:
            if any(rows[r][0] for r in range(w)):
                raise L.QkError("as-of join: no quotes were received")
            return None
        parts, own = {}, None
        if trades is not None and len(trades) > 0:
            cuts = [rows[o][5] for o in owners[1:]]
            pos = torch.searchsorted(trades[tt].data, torch.tensor(cuts, dtype=torch.int64, device=dev)).tolist() if cuts else []
            ends = {o: int(p_) for o, p_ in zip(owners[:-1], pos)} | {owners[-1]: len(trades)}
            bounds = [0]
            for r in range(w):
                bounds.append(ends[r] if r in ends else bounds[-1])
            parts = {r: trades.slice(bounds[r], bounds[r + 1]) for r in range(w) if r != me and bounds[r + 1] > bounds[r]}
            own = trades.slice(bounds[me], bounds[me + 1])           # the bulk: stays where it is
        mine = ex(parts, w, edge_key=("asof-trades", id(self)))
        if own is not None and len(own) > 0:
            own.src_rank = me
            mine = list(mine) + [own]
        mine = sorted(mine, key=lambda g: g.src_rank)
        self.trade_state = self.quote_state = None
        self._carry, self._swept, self._whole_state = None, 0, False
        all_q = earlier + ([quotes] if quotes is not None and len(quotes) > 0 else [])
        if not mine:
            return None
        t = concat_tables(mine)
        out = self._join_carried(t, earlier, quotes) if earlier and quotes is not None and len(quotes) > 0 else None
        if out is not None:
            return out
        q = concat_tables(all_q)
        self.quote_state = q.with_column(self.BY, DeviceColumn(self._stable_codes(q[self.symbol_col_quotes])))
        t = t.with_column(self.BY, DeviceColumn(self._stable_codes(t[self.symbol_col_trades])))
        return self._join(t, None)

    def _join_carried(self, trades, earlier, quotes):
        """trades joined against [the few carried rows of earlier ranks] + [this rank's quotes] WITHOUT putting the two into one
        table (that copy is the whole quote shard): the carried rows become the merge kernel's carry-in table, the answer's row
        numbers below len(carried) point into them, the others into the shard, and the payload is gathered from both.  None when
        the shapes call for the plain path (dictionary payload columns that differ, symbol sets beyond the kernel's table)."""
        E = concat_tables(earlier)
        payload = [c for c in quotes.column_names if c not in (self.time_col_quotes, self.symbol_col_quotes)]
        if any((E[c].dictionary is not None or quotes[c].dictionary is not None) and E[c].dictionary != quotes[c].dictionary for c in payload):
            return None
        sq, st_ = quotes[self.symbol_col_quotes], trades[self.symbol_col_trades]
        if sq.dictionary is not None or st_.dictionary is not None or E[self.symbol_col_quotes].dictionary is not None:
            both = concat_tables([E.select([self.symbol_col_quotes]), quotes.select([self.symbol_col_quotes])])     # one dictionary for both
            codes = self._stable_codes(both[self.symbol_col_quotes])
            e_codes, q_codes = codes[:len(E)], codes[len(E):]
        else:
            e_codes, q_codes = self._stable_codes(E[self.symbol_col_quotes]), self._stable_codes(sq)
        t_codes = self._stable_codes(st_)
        n_by, dev = max(1, self._n_by), trades.device
        lt, rt = trades[self.time_col_trades].data, quotes[self.time_col_quotes].data
        if lt.dtype != torch.int64 or rt.dtype != torch.int64:
            raise L.QkError("as-of time columns must be int64 / timestamp")
        none_t, none_b = torch.empty(0, dtype=torch.int64, device=dev), torch.empty(0, dtype=torch.int32, device=dev)
        _, carried = ops.asof_merge(none_t, none_b, E[self.time_col_quotes].data, e_codes, n_by, want_carry=True)
        if carried is None:
            return None
        ridx, _ = ops.asof_merge(lt, t_codes, rt, q_codes, n_by, carried, len(E))
        if ridx is None:
            return None
        in_shard = ridx >= len(E)
        from_shard = quotes.select(payload).gather(torch.where(in_shard, ridx - len(E), torch.full_like(ridx, -1)))
        from_carry = E.select(payload).gather(torch.where(in_shard, torch.full_like(ridx, -1), ridx))
        valid = (ridx >= 0).to(torch.uint8)
        if os.environ.get("QK_DEBUG_ASOF"):
            print(f"[asof] carried join: {len(E)} carried rows, {int((~in_shard & (ridx >= 0)).sum())} answers from them", flush=True)
        cols = dict(trades.columns)
        for n in payload:
            a, b_ = from_shard[n], from_carry[n]
            cols[n + self.suffix if n in cols else n] = DeviceColumn(torch.where(in_shard, a.data, b_.data), a.dictionary, a.arrow_type, valid)
        return DeviceTable(cols)

    def done(self, executor_id):
        if self.time_ranges and _world() > 1:
            return self._join_time_ranges()
        if self._by_source is not None:
            for sid, tcol, by in ((0, self.time_col_trades, self.symbol_col_trades), (1, self.time_col_quotes, self.symbol_col_quotes)):
                parts = [b for r in sorted(self._by_source[sid]) for b in self._by_source[sid][r]]
                if not parts:
                    continue
                t = concat_tables(parts)
                tt = t[tcol].data
                if len(tt) > 1 and not bool((tt[1:] >= tt[:-1]).all().item()):
                    raise L.QkError("as-of join: the producer ranks do not hold consecutive time ranges of a sorted stream")
                t = t.with_column(self.BY, DeviceColumn(self._stable_codes(t[by])))
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
class _WindowExecutor(Executor):
    """Common part of the three window executors (pyquokka/executors/ts_executors.py:12-288): the stream arrives sorted by
    time and hash-partitioned by the `by` column; the rows are segmented by key with the stable partition kernel (time order
    survives inside a key) and the window kernel of the subclass runs over the segments.  The windows are evaluated when the
    channel's input is complete (done()): the same rows, whatever the batching -- the reference's incremental emission
    loses rows of hopping windows across batch boundaries (ts_executors.py:41-58 keeps only rows past the last complete
    window although earlier rows still belong to later windows)."""

    silent_streams = "all"       # windows are evaluated when the channel's input is complete

    def __init__(self, time_col, by_col, window, trigger) -> None:
        from .windowtypes import Trigger, Window
        assert issubclass(type(window), Window) and issubclass(type(trigger), Trigger)
        self.time_col, self.by_col, self.window, self.trigger = time_col, by_col, window, trigger
        self.state = None
        self._parts = {}             # source rank -> batches in arrival order (ranks hold consecutive time ranges)
        self._codes = SortedAsofExecutor()      # only for its append-only symbol codes

    def execute(self, batches, stream_id, executor_id):
        for b in _clean(batches):
            self._parts.setdefault(getattr(b, "src_rank", 0) or 0, []).append(b)

    def _segmented(self):
        """(time, by codes, seg, n_by, fp64 value columns, aggregate list, decode) in key-segmented order, or None."""
        parts = [b for r in sorted(self._parts) for b in self._parts[r]]
        self._parts = {}
        if not parts:
            return None
        t = concat_tables(parts)
        tcol = t[self.time_col]
        time = tcol.data.to(torch.int64)
        if len(time) > 1 and not bool((time[1:] >= time[:-1]).all().item()):
            raise L.QkError("windowed_transform: the stream is not sorted by " + self.time_col)
        bycol = t[self.by_col]
        codes = self._codes._stable_codes(bycol)
        n_by = max(1, self._codes._n_by)
        aggs = self.window.parsed()
        exprs, vals = [], []
        for _, op, arg in aggs:                                   # one fp64 column per distinct argument expression
            if arg is not None and arg.sql() not in exprs:
                exprs.append(arg.sql())
                e = EdgeOps(None, {"__v": arg}).apply(t.select(sorted(arg.columns(), key=t.column_names.index)), stable=True)
                vals.append(to_f64(e["__v"].data))
        dest, seg = ops.partition_plan(codes, n_by, L.PART_CODE)
        moved = ops.scatter([time, codes] + vals, dest)
        spec = [(name, op, exprs.index(arg.sql()) if arg is not None else -1) for name, op, arg in aggs]
        unit = str(tcol.arrow_type.unit) if tcol.arrow_type is not None and pa_is_timestamp(tcol.arrow_type) else None
        return moved[0], moved[1], seg, n_by, moved[2:], spec, (bycol, tcol, unit)

    def _by_column(self, codes: torch.Tensor, bycol: DeviceColumn) -> DeviceColumn:
        if self._codes._values is not None:
            return DeviceColumn(codes, list(self._codes._values), None)
        return DeviceColumn(codes.to(bycol.data.dtype), None, bycol.arrow_type)

    def _time_column(self, time: torch.Tensor, tcol: DeviceColumn) -> DeviceColumn:
        return DeviceColumn(time.to(tcol.data.dtype), None, tcol.arrow_type)


def pa_is_timestamp(t) -> bool:
    import pyarrow as pa
    return pa.types.is_timestamp(t)


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
        cols = {self.time_col: self._time_column(time, tcol), self.by_col: self._by_column(codes, bycol)}
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


class HoppingWindowExecutor(_HashedWindow):
    """ts_executors.py:12-145: aggregates per key over the windows [k * hop, k * hop + size) (Polars groupby_dynamic(every=hop,
    period=size, by=key): closed on the left, labelled by the window start, windows before the key's first truncated
    timestamp are not produced, empty windows neither).  TumblingWindow = hop == size.  Output: time (window start), key, aggregates."""

    def __init__(self, time_col, by_col, window, trigger) -> None:
        from .windowtypes import HoppingWindow, OnEventTrigger
        assert issubclass(type(window), HoppingWindow)
        super().__init__(time_col, by_col, window, trigger)
        if type(trigger) == OnEventTrigger and type(window) == HoppingWindow:
            raise Exception("OnEventTrigger is not supported for hopping windows")

    def done(self, executor_id):
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
        cols = {self.time_col: self._time_column(ok[1], tcol), self.by_col: self._by_column(ok[0], bycol)}
        cols.update(out)
        return DeviceTable(cols)


class SessionWindowExecutor(_HashedWindow):
    """ts_executors.py:197-288: per key, a session = a run of rows whose gaps are all <= timeout; aggregates per session.
    Output: key, time (the session's first timestamp; the reference emits its internal window id instead), aggregates."""

    def __init__(self, time_col, by_col, window, trigger) -> None:
        from .windowtypes import SessionWindow
        assert issubclass(type(window), SessionWindow)
        super().__init__(time_col, by_col, window, trigger)

    def done(self, executor_id):
        seg_in = self._segmented()
        if seg_in is None:
            return None
        time, codes, seg, n_by, vals, spec, (bycol, tcol, unit) = seg_in
        ids = ops.window_session_ids(time, codes, self.window.ticks(self.window.timeout, unit))
        ok, out = self._aggregate([ids], vals, spec)
        # the first row of session s (ids are 1-based and increase along the segmented order)
        starts = torch.nonzero(torch.diff(ids, prepend=ids[:1] - 1)).flatten()
        at = starts[ok[0] - 1]
        cols = {self.by_col: self._by_column(codes[at], bycol), self.time_col: self._time_column(time[at], tcol)}
        cols.update(out)
        return DeviceTable(cols)
