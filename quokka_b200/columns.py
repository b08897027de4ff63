"""Device-resident column batches: the currency every operator exchanges.

A `DeviceTable` is what the reference passes around as `pyarrow.Table` / `polars.DataFrame`
(pyquokka/core.py:32-35,152-195) -- here each column is a contiguous torch CUDA tensor in Arrow's
fixed-width layout (int64 / int32 / date32-as-int32 / float64 / float32 / uint8), and string columns are
dictionary codes with the value list kept on the host (SURVEY.md section 7 "Strings").  Conversion to
and from Arrow happens only at the edges (readers, collect()).

A vector column (fixed_size_list / list of floats, the embeddings of DataStream.vector_nn_join) is a contiguous 2-D tensor
(n, d) of float32 or float16, 1 <= d <= 4096."""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import torch
import torch.distributed as dist

from . import _lib as L
from . import ops


def _default_device():
    """The CUDA device of this process.  There is deliberately no CPU alternative."""
    if not torch.cuda.is_available():
        raise L.QkError("quokka_b200 needs a CUDA device: there is no CPU execution path")
    return torch.device("cuda", torch.cuda.current_device())


def default_device():
    return _default_device()


def world_size() -> int:
    """How many ranks (one process per GPU) there are: the one definition, here because every module imports this one."""
    return dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1


def rank() -> int:
    return dist.get_rank() if dist.is_available() and dist.is_initialized() else 0


@dataclass
class DeviceColumn:
    data: torch.Tensor
    dictionary: list | None = None          # host-side values of a dictionary-coded string column
    arrow_type: pa.DataType | None = None   # logical type to restore in to_arrow() (date32, timestamp, bool...)
    valid: torch.Tensor | None = None       # uint8 mask, only ever produced by left / as-of joins ("no match")

    def __len__(self):
        return self.data.shape[0] if self.data.dim() == 2 else self.data.numel()

    @property
    def is_vector(self) -> bool:
        return self.data.dim() == 2

    @property
    def qk_dtype(self) -> int:
        return ops.qk_dtype(self.data)


class DeviceTable:
    def __init__(self, columns: dict | None = None):
        self.columns: dict[str, DeviceColumn] = dict(columns or {})
        n = {len(c) for c in self.columns.values()}
        if len(n) > 1:
            raise L.QkError(f"ragged DeviceTable: column lengths {n}")

    # ---- basic protocol (what executors use; mirrors the bits of polars.DataFrame the reference touches)
    def __len__(self):
        for c in self.columns.values():
            return len(c)
        return 0

    num_rows = property(__len__)

    @property
    def column_names(self):
        return list(self.columns)

    @property
    def device(self):
        for c in self.columns.values():
            return c.data.device
        return default_device()

    def __getitem__(self, name):
        return self.columns[name]

    def __contains__(self, name):
        return name in self.columns

    def select(self, names):
        missing = [n for n in names if n not in self.columns]
        if missing:
            raise L.QkError(f"columns {missing} not in {self.column_names}")
        return DeviceTable({n: self.columns[n] for n in names})

    def drop(self, names):
        return DeviceTable({n: c for n, c in self.columns.items() if n not in set(names)})

    def rename(self, mapping):
        return DeviceTable({mapping.get(n, n): c for n, c in self.columns.items()})

    def with_column(self, name, col: DeviceColumn):
        d = dict(self.columns)
        d[name] = col
        return DeviceTable(d)

    def sorted_columns(self):
        """Alphabetical column order, as every edge of the reference emits (core.py:190-193)."""
        return DeviceTable({n: self.columns[n] for n in sorted(self.columns)})

    def slice(self, lo, hi):
        return DeviceTable({n: DeviceColumn(c.data[lo:hi], c.dictionary, c.arrow_type, None if c.valid is None else c.valid[lo:hi])
                            for n, c in self.columns.items()})

    def gather(self, idx: torch.Tensor):
        names = list(self.columns)
        masks = {}                                     # distinct validity masks travel with their rows
        for c in self.columns.values():
            if c.valid is not None:
                masks.setdefault(id(c.valid), c.valid)
        outs = ops.gather([self.columns[n].data for n in names] + list(masks.values()), idx)
        moved = dict(zip(masks, outs[len(names):]))
        return DeviceTable({n: DeviceColumn(o, self.columns[n].dictionary, self.columns[n].arrow_type,
                                            None if self.columns[n].valid is None else moved[id(self.columns[n].valid)])
                            for n, o in zip(names, outs)})

    def split_validity(self):
        """(table without masks but with every distinct mask as a hidden uint8 column, {column: hidden mask column}) -- how
        nullable tables (right side of a left / as-of join) go through kernels that know nothing about NULL."""
        hidden, of = {}, {}
        for n, c in self.columns.items():
            if c.valid is not None:
                name = hidden.setdefault(id(c.valid), (f"__valid{len(hidden)}", c.valid))[0]
                of[n] = name
        cols = {n: DeviceColumn(c.data, c.dictionary, c.arrow_type) for n, c in self.columns.items()}
        for name, m in hidden.values():
            cols[name] = DeviceColumn(m)
        return DeviceTable(cols), of

    def drop_nulls(self):
        """Rows where every column is valid (the apps call .drop_nulls() after an as-of join)."""
        masks = [c.valid for c in self.columns.values() if c.valid is not None]
        if not masks:
            return self
        ok = masks[0].bool()
        for m in masks[1:]:
            ok &= m.bool()
        idx = torch.nonzero(ok).flatten().to(torch.int32)
        return self.gather(idx)

    def with_validity(self, valid: torch.Tensor):
        return DeviceTable({n: DeviceColumn(c.data, c.dictionary, c.arrow_type, valid) for n, c in self.columns.items()})

    def schema_info(self):
        """name -> expr.ColumnInfo for the expression compiler."""
        from .expr import ColumnInfo
        return {n: ColumnInfo(i, c.qk_dtype, c.dictionary, c.arrow_type is not None and pa.types.is_date(c.arrow_type))
                for i, (n, c) in enumerate(self.columns.items())}

    # ---- Arrow edges
    @staticmethod
    def from_arrow(tbl: pa.Table, device=None, dictionaries: "DictionaryRegistry | None" = None) -> "DeviceTable":
        cols = {}
        device = device or default_device()
        for name in tbl.column_names:
            cols[name] = _arrow_to_device(name, tbl[name], device, dictionaries)
        return DeviceTable(cols)

    def to_arrow(self) -> pa.Table:
        arrays, names = [], []
        for n, c in self.columns.items():
            h = c.data.cpu().numpy()
            if c.is_vector:
                arr = pa.FixedSizeListArray.from_arrays(pa.array(h.reshape(-1)), h.shape[1])
            elif c.dictionary is not None:
                arr = pa.DictionaryArray.from_arrays(pa.array(h.astype(np.int32)), pa.array(c.dictionary, type=pa.string())).cast(pa.string())
            elif c.arrow_type is not None and pa.types.is_boolean(c.arrow_type):
                arr = pa.array(h.astype(bool))
            elif c.arrow_type is not None:
                arr = pa.array(h).cast(c.arrow_type) if not pa.types.is_date32(c.arrow_type) else pa.array(h.astype(np.int32), type=pa.int32()).cast(pa.date32())
            else:
                arr = pa.array(h)
            if c.valid is not None:
                ok = pa.array(c.valid.cpu().numpy().astype(bool))
                arr = pc.if_else(ok, arr, pa.scalar(None, arr.type))
            arrays.append(arr)
            names.append(n)
        return pa.table(arrays, names=names)

    def to_numpy(self) -> dict:
        return {n: c.data.cpu().numpy() for n, c in self.columns.items()}

    @staticmethod
    def from_numpy(cols: dict, device=None, dictionaries: dict | None = None, dates=()):
        out = {}
        device = device or default_device()
        for n, v in cols.items():
            t = torch.from_numpy(np.ascontiguousarray(v)).to(device)
            if t.dim() == 2 and not (t.dtype in (torch.float32, torch.float16) and 1 <= t.shape[1] <= MAX_VECTOR_DIM):
                raise L.QkError(f"column {n!r}: a 2-D column must be float32 / float16 with 1 <= d <= {MAX_VECTOR_DIM}")
            out[n] = DeviceColumn(t, (dictionaries or {}).get(n), pa.date32() if n in dates else None)
        return DeviceTable(out)


def concat_tables(tables: list) -> DeviceTable:
    """vstack of batches with identical column sets (`polars.concat`, sql_executors.py:351).  Dictionary
    columns are re-coded onto the union dictionary when they differ."""
    tables = [t for t in tables if t is not None and len(t.columns) > 0]
    if not tables:
        return DeviceTable()
    if len(tables) == 1:
        return tables[0]
    names = tables[0].column_names
    out = {}
    for n in names:
        parts = [t[n] for t in tables]
        dic = parts[0].dictionary
        if dic is not None and any(p.dictionary != dic for p in parts):
            dic, parts = unify_dictionaries(parts)
        valid = None
        if any(p.valid is not None for p in parts):
            valid = torch.cat([p.valid if p.valid is not None else torch.ones(len(p), dtype=torch.uint8, device=p.data.device)
                               for p in parts])
        datas = [p.data for p in parts]
        if any(x.dim() == 2 for x in datas):          # vector rows: an empty part may not know the row length
            datas = [x for x in datas if x.shape[0] > 0] or datas[:1]
        out[n] = DeviceColumn(torch.cat(datas), dic, parts[0].arrow_type, valid)
    return DeviceTable(out)


def unify_dictionaries(parts: list):
    """Re-code dictionary columns onto the sorted union of their dictionaries (codes are data movement:
    a lookup-table gather on the device)."""
    union = sorted(set().union(*[set(p.dictionary) for p in parts]))
    pos = {v: i for i, v in enumerate(union)}
    out = []
    for p in parts:
        if p.dictionary == union:
            out.append(p)
            continue
        lut = torch.tensor([pos[v] for v in p.dictionary] or [0], dtype=p.data.dtype, device=p.data.device)
        if len(union) > 255 and p.data.dtype == torch.uint8:
            raise L.QkError("dictionary grew past 255 entries for a uint8 code column")
        out.append(DeviceColumn(lut[p.data.long()], union, p.arrow_type, p.valid))
    return union, out


class DictionaryRegistry:
    """Per-context, per-column value lists so that every batch of a column uses the same codes."""

    def __init__(self):
        self.values: dict[str, list] = {}
        self.index: dict[str, dict] = {}

    def codes_for(self, name: str, local: list) -> list:
        """Global codes of a chunk-local dictionary (new values are appended to the column's value list)."""
        vals = self.values.setdefault(name, [])
        idx = self.index.setdefault(name, {})
        for v in local:
            if v not in idx:
                idx[v] = len(vals)
                vals.append(v)
        return [idx[v] for v in local]

    def encode(self, name: str, arr: pa.ChunkedArray | pa.Array):
        if isinstance(arr, pa.ChunkedArray):
            arr = arr.combine_chunks()
        if not pa.types.is_dictionary(arr.type):
            arr = pc.dictionary_encode(arr)
        if isinstance(arr, pa.ChunkedArray):
            arr = arr.combine_chunks()
        local = arr.dictionary.to_pylist()
        vals = self.values.setdefault(name, [])
        idx = self.index.setdefault(name, {})
        for v in local:
            if v not in idx:
                idx[v] = len(vals)
                vals.append(v)
        codes = arr.indices.to_numpy(zero_copy_only=False)
        lut = np.array([idx[v] for v in local] or [0], dtype=np.int64)
        return lut[codes], vals


def _from_numpy(h):
    """Arrow buffers are read-only; the tensor is only ever the source of a host->device copy."""
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", UserWarning)
        return torch.from_numpy(np.ascontiguousarray(h))


MAX_VECTOR_DIM = 4096


def is_vector_type(t: pa.DataType) -> bool:
    return pa.types.is_fixed_size_list(t) or pa.types.is_list(t) or pa.types.is_large_list(t)


def vector_columns(schema: pa.Schema) -> list:
    """Names of the list-typed fields of an Arrow schema: the columns that load as vector columns."""
    return [f.name for f in schema if is_vector_type(f.type)]


def _vector_to_device(name, col, device) -> DeviceColumn:
    """fixed_size_list<float32 | float16, d> is stored as it is; list / large_list<float*> whose rows all have one length are
    accepted too, and float64 elements are rounded to float32 once, here (as DECIMAL becomes fp64 at the reader).  Ragged
    lists, null rows or elements, non-float elements and d > 4096 raise."""
    arr = col.combine_chunks() if isinstance(col, pa.ChunkedArray) else col
    t = arr.type
    vt = t.value_type
    if not pa.types.is_floating(vt):
        raise L.QkError(f"column {name!r}: vector elements must be floats, not {vt}")
    if arr.null_count:
        raise L.QkError(f"column {name!r}: a vector column cannot hold null rows")
    n = len(arr)
    if pa.types.is_fixed_size_list(t):
        d = t.list_size
        values = arr.values.slice(arr.offset * d, n * d)
    else:
        offs = arr.offsets.to_numpy(zero_copy_only=False).astype(np.int64)
        lens = np.diff(offs)
        d = int(lens[0]) if n else 0
        if n and (lens != d).any():
            raise L.QkError(f"column {name!r}: ragged list column (row lengths {int(lens.min())} .. {int(lens.max())}); vector columns need one length")
        values = arr.values.slice(int(offs[0]) if n else 0, n * d)
    if n and not 1 <= d <= MAX_VECTOR_DIM:
        raise L.QkError(f"column {name!r}: vector dimension {d} outside [1, {MAX_VECTOR_DIM}]")
    if values.null_count:
        raise L.QkError(f"column {name!r}: a vector column cannot hold null elements")
    h = values.to_numpy(zero_copy_only=False)
    if h.dtype == np.float64:
        h = h.astype(np.float32)
    # an empty chunk of a variable-size list has no row length: (0, 1); concat_tables drops empty vector parts
    return DeviceColumn(_from_numpy(h.reshape(n, d if (n or pa.types.is_fixed_size_list(t)) else 1)).to(device), None, None)


def _arrow_to_device(name, col, device, dictionaries) -> DeviceColumn:
    if is_vector_type(col.type):
        return _vector_to_device(name, col, device)
    if isinstance(col, pa.ChunkedArray):
        if col.null_count:
            raise L.QkError(f"column {name!r} has nulls: validity bitmaps are not supported on the hot path")
        t = col.type
    else:
        t = col.type
    if pa.types.is_dictionary(t) or pa.types.is_string(t) or pa.types.is_large_string(t):
        reg = dictionaries if dictionaries is not None else DictionaryRegistry()
        codes, vals = reg.encode(name, col)
        # small dictionaries stay 1 byte per row (TPC-H flags / segments: SURVEY.md section 8)
        dt = np.uint8 if len(vals) <= 255 and (pa.types.is_dictionary(t) and t.index_type.bit_width == 8) else np.int32
        return DeviceColumn(torch.from_numpy(codes.astype(dt)).to(device), vals, None)
    arr = col.combine_chunks() if isinstance(col, pa.ChunkedArray) else col
    if pa.types.is_decimal(t):
        # the Spark-written TPC-H set stores measures as DECIMAL(10,2) (benchmark/spark/convert.py:11-14); on the device
        # they are fp64 (north_star): value = unscaled integer / 10^scale, ONE correctly rounded division -- the double
        # nearest to the decimal, the same bits the device decoder produces (Arrow's own cast multiplies by 10^-scale
        # and is off by an ulp for ~13 % of two-decimal values)
        if not pa.types.is_decimal128(t) or t.precision > 18:
            raise L.QkError(f"column {name!r}: {t} does not fit a 64-bit unscaled integer")
        if arr.null_count:
            raise L.QkError(f"column {name!r} has nulls: validity bitmaps are not supported on the hot path")
        unscaled = np.frombuffer(arr.buffers()[1], dtype=np.int64)[2 * arr.offset:2 * (arr.offset + len(arr)):2]
        h = unscaled / float(10 ** t.scale) if t.scale else unscaled.astype(np.float64)
        return DeviceColumn(_from_numpy(h).to(device), None, None)
    if pa.types.is_date32(t):
        h = arr.cast(pa.int32()).to_numpy(zero_copy_only=False)
        return DeviceColumn(_from_numpy(h).to(device), None, pa.date32())
    if pa.types.is_timestamp(t) or pa.types.is_date64(t):
        h = arr.cast(pa.int64()).to_numpy(zero_copy_only=False)
        return DeviceColumn(_from_numpy(h).to(device), None, t)
    if pa.types.is_boolean(t):
        h = arr.to_numpy(zero_copy_only=False).astype(np.uint8)
        return DeviceColumn(torch.from_numpy(h).to(device), None, pa.bool_())
    if pa.types.is_integer(t) or pa.types.is_floating(t):
        h = arr.to_numpy(zero_copy_only=False)
        if h.dtype in (np.int8, np.int16, np.uint16):
            h = h.astype(np.int32)
        elif h.dtype in (np.uint32, np.uint64):
            h = h.astype(np.int64)
        elif h.dtype == np.float16:
            h = h.astype(np.float32)
        return DeviceColumn(_from_numpy(h).to(device), None, None)
    raise L.QkError(f"column {name!r}: Arrow type {t} is not supported")


def as_device_table(batch, device=None, dictionaries=None) -> DeviceTable:
    """Accepts what the reference's runtime would hand an Executor (pyarrow.Table) or a DeviceTable."""
    if batch is None:
        return None
    if isinstance(batch, DeviceTable):
        return batch
    if isinstance(batch, pa.Table):
        return DeviceTable.from_arrow(batch, device, dictionaries)
    if isinstance(batch, pa.RecordBatch):
        return DeviceTable.from_arrow(pa.Table.from_batches([batch]), device, dictionaries)
    try:
        import pandas as pd
        if isinstance(batch, pd.DataFrame):
            return DeviceTable.from_arrow(pa.Table.from_pandas(batch, preserve_index=False), device, dictionaries)
    except ImportError:
        pass
    raise L.QkError(f"cannot use {type(batch)} as a batch")
