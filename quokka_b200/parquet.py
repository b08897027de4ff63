"""Parquet row groups decoded on the device (SURVEY.md section 8(f).1).

The reference's readers hand Parquet to Arrow C++ on the host (`pq.ParquetFile(...).read_row_groups`,
pyquokka/dataset/unordered_readers.py:51,98-99) and ship decoded Arrow buffers.  Here the ENCODED bytes of the
selected column chunks are read as they lie in the file into pinned memory, copied to the device, and turned into
Arrow-layout columns by `qk_parquet_decode`; the host only walks the page and run headers
(`qk_parquet_walk_chunk`, a few bytes per several hundred values).  What crosses PCIe is the file's encoding
(dictionary-coded columns: a few bits per value), not 4-8 bytes per value.

Scope (loud `QkError` outside it): flat schemas, no nulls, PLAIN and RLE_DICTIONARY pages (V1 / V2), BOOLEAN /
INT32 / INT64 / FLOAT / DOUBLE values and dictionary-coded strings (a string column written WITHOUT a dictionary is
dictionary-coded by Arrow on the host -- strings never live on the device, only their codes), UNCOMPRESSED pages (the layout the bench files
use, SURVEY.md section 8(d) "Synthetic inputs": the host walks page and run headers) and SNAPPY / ZSTD / GZIP pages (Spark's
and pyarrow's default / Polars' default / Athena's default: the host sees only page headers; pages are inflated and their run headers
walked on the device)."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import torch

from . import _lib as L
from . import ops
from .columns import DeviceColumn, DeviceTable, DictionaryRegistry

RUN_DTYPE = np.dtype([("dense_start", "<i8"), ("payload", "<i8"), ("dict_base", "<i4"), ("kind", "u1"),
                      ("bit_width", "u1"), ("reserved", "<u2")])
assert RUN_DTYPE.itemsize == C.sizeof(L.qk_pq_run) == 24

_PHYSICAL = {"BOOLEAN": L.PQ_BOOLEAN, "INT32": L.PQ_INT32, "INT64": L.PQ_INT64, "INT96": L.PQ_INT96, "FLOAT": L.PQ_FLOAT,
             "DOUBLE": L.PQ_DOUBLE, "BYTE_ARRAY": L.PQ_BYTE_ARRAY, "FIXED_LEN_BYTE_ARRAY": L.PQ_FIXED_LEN_BYTE_ARRAY}
_OUT_DTYPE = {L.PQ_BOOLEAN: torch.uint8, L.PQ_INT32: torch.int32, L.PQ_INT64: torch.int64, L.PQ_FLOAT: torch.float32,
              L.PQ_DOUBLE: torch.float64, L.PQ_BYTE_ARRAY: torch.int32}


def _arrow_type_to_keep(t: pa.DataType, name: str):
    """The logical type `DeviceTable.to_arrow` restores; raises for types whose device layout differs from the
    Parquet physical layout (they would need a widening pass the host reader does with numpy)."""
    if pa.types.is_date32(t) or pa.types.is_timestamp(t) or pa.types.is_date64(t):
        return t
    if pa.types.is_boolean(t):
        return pa.bool_()
    if pa.types.is_string(t) or pa.types.is_large_string(t) or pa.types.is_dictionary(t):
        return None
    if pa.types.is_unsigned_integer(t) and t.bit_width >= 32:
        raise L.QkError(f"column {name!r}: {t} needs widening; not supported by the device Parquet decoder")
    if pa.types.is_integer(t) or pa.types.is_floating(t) or pa.types.is_decimal(t):
        return None                               # decimals become fp64 on the device (see _decimal_to_f64)
    raise L.QkError(f"column {name!r}: Arrow type {t} is not supported by the device Parquet decoder")


class _ColumnPlan:
    """All chunks of one column for one batch of row groups: where their bytes go in the staging buffer."""

    def __init__(self, name, physical, max_def, arrow_type):
        self.name, self.physical, self.max_def, self.arrow_type = name, physical, max_def, arrow_type
        self.chunks = []            # (file index, file offset, bytes, num_values, compression name)
        self.total_bytes = 0
        self.total_values = 0

    def add(self, fi, start, size, nvals, compression):
        self.chunks.append((fi, start, size, nvals, compression, self.total_bytes))
        self.total_bytes += size
        self.total_values += nvals


def plan_batch(units, columns=None):
    """units: [(path, row_group), ...] -> (list of paths, {column: _ColumnPlan}, rows)."""
    paths, plans, rows = [], {}, 0
    meta = {}
    for path, g in units:
        if path not in meta:
            pf = pq.ParquetFile(path)
            meta[path] = (len(paths), pf.metadata, pf.schema, pf.schema_arrow)
            paths.append(path)
        fi, md, schema, arrow_schema = meta[path]
        rg = md.row_group(g)
        rows += rg.num_rows
        names = schema.names
        want = columns if columns is not None else list(arrow_schema.names)
        for name in want:
            if name in arrow_schema.names and pa.types.is_list(arrow_schema.field(name).type) | \
                    pa.types.is_large_list(arrow_schema.field(name).type) | pa.types.is_fixed_size_list(arrow_schema.field(name).type):
                raise L.QkError(f"{path}: column {name!r} is a nested list (vector) column, which the device Parquet decoder "
                                "does not read; set device_parquet to False to read it through Arrow")
            if name not in names:
                raise L.QkError(f"{path}: no column {name!r} (nested columns are not supported)")
            ci = names.index(name)
            cs = schema.column(ci)
            if cs.max_repetition_level != 0 or cs.path != name:
                raise L.QkError(f"{path}: column {name!r} is nested; only flat schemas are supported")
            if name not in plans:
                plans[name] = _ColumnPlan(name, _PHYSICAL[cs.physical_type], cs.max_definition_level,
                                          arrow_schema.field(name).type)
                _arrow_type_to_keep(plans[name].arrow_type, name)
            p = plans[name]
            if p.physical != _PHYSICAL[cs.physical_type]:
                raise L.QkError(f"column {name!r}: physical type differs between files")
            cc = rg.column(ci)
            start = cc.data_page_offset
            if cc.has_dictionary_page and cc.dictionary_page_offset:
                start = min(start, cc.dictionary_page_offset)
            p.add(fi, start, cc.total_compressed_size, cc.num_values, cc.compression)
    for p in plans.values():
        if p.total_values != rows:
            raise L.QkError(f"column {p.name!r}: {p.total_values} values for {rows} rows (nulls / nesting are not supported)")
    return paths, plans, rows


def walk_chunk(buf_ptr, off, size, nvals, physical, max_def, compression, dict_base, runs, n_runs, dense):
    """qk_parquet_walk_chunk with a growing run table.  -> (runs, n_runs, dense, info)"""
    lib = L.lib()
    info = L.qk_pq_chunk_info()
    while True:
        nr, d = C.c_int64(n_runs), C.c_int64(dense)
        rc = lib.qk_parquet_walk_chunk(buf_ptr, off, size, nvals, physical, max_def, compression, dict_base,
                                       runs.ctypes.data, len(runs) - 1, C.byref(nr), C.byref(d), C.byref(info))
        if rc == L.ERR_CAPACITY:
            runs = np.concatenate([runs, np.zeros(len(runs), RUN_DTYPE)])
            continue
        L.check(rc, "qk_parquet_walk_chunk")
        return runs, nr.value, d.value, info


def _dictionary_strings(view, off, nbytes, n):
    """PLAIN BYTE_ARRAY dictionary page -> list of str (4-byte little-endian length + bytes each)."""
    out, p, end = [], off, off + nbytes
    for _ in range(n):
        if p + 4 > end:
            raise L.QkError("Parquet dictionary page is truncated")
        ln = int.from_bytes(view[p:p + 4], "little")
        p += 4
        if p + ln > end:
            raise L.QkError("Parquet dictionary page is truncated")
        try:
            out.append(bytes(view[p:p + ln]).decode("utf-8"))
        except UnicodeDecodeError:
            raise L.QkError("Parquet dictionary page holds bytes that are not UTF-8") from None
        p += ln
    return out


def _sentinel(runs, n_runs, n_values):
    runs = runs[:n_runs + 1]
    runs[n_runs] = (n_values, 0, 0, 0, 0, 0)
    return runs


PAGE_DTYPE = np.dtype([("src_offset", "<i8"), ("dst_offset", "<i8"), ("dense_start", "<i8"), ("src_bytes", "<i4"),
                       ("dst_bytes", "<i4"), ("num_values", "<i4"), ("dict_base", "<i4"), ("n_runs", "<i4"), ("kind", "u1"),
                       ("encoding", "u1"), ("compressed", "u1"), ("max_def", "u1"), ("status", "<i4"), ("reserved", "<i4")])
assert PAGE_DTYPE.itemsize == C.sizeof(L.qk_pq_page) == 56
_CODEC = {"UNCOMPRESSED": L.PQ_CODEC_NONE, "SNAPPY": L.PQ_CODEC_SNAPPY, "ZSTD": L.PQ_CODEC_ZSTD, "GZIP": L.PQ_CODEC_GZIP}
_ARROW_CODEC = {L.PQ_CODEC_SNAPPY: "snappy", L.PQ_CODEC_ZSTD: "zstd", L.PQ_CODEC_GZIP: "gzip"}


def walk_pages(buf_ptr, off, size, nvals, physical, max_def, codec, dict_base, pages, n_pages, dense, scratch):
    """qk_parquet_walk_pages with a growing page table.  -> (pages, n_pages, dense, scratch_bytes, info)"""
    lib = L.lib()
    info = L.qk_pq_chunk_info()
    while True:
        np_, d, sc = C.c_int64(n_pages), C.c_int64(dense), C.c_int64(scratch)
        rc = lib.qk_parquet_walk_pages(buf_ptr, off, size, nvals, physical, max_def, codec, dict_base, pages.ctypes.data,
                                       len(pages), C.byref(np_), C.byref(d), C.byref(sc), C.byref(info))
        if rc == L.ERR_CAPACITY:
            pages = np.concatenate([pages, np.zeros(len(pages), PAGE_DTYPE)])
            continue
        L.check(rc, "qk_parquet_walk_pages")
        return pages, np_.value, d.value, sc.value, info


def _stage_alloc(plan, pin):
    """The (pinned) host buffer for a column's chunks.  Allocated on the caller's thread: a pinned allocation binds to
    the thread's current CUDA device, which worker threads do not inherit."""
    return torch.empty((plan.total_bytes + 7) // 8 * 8 + ops.PQ_PAD, dtype=torch.uint8, pin_memory=pin)


def _stage_chunks(plan, paths, files, stage):
    """The column's chunks, as they lie in the files, into `stage`.  `files` are raw descriptors; preadv keeps
    concurrent column readers off each other's file position."""
    view = stage.numpy()
    mv = memoryview(view)
    for fi, start, size, nvals, compression, off in plan.chunks:
        got = 0
        while got < size:
            n = os.preadv(files[fi], [mv[off + got:off + size]], start + got)
            if n <= 0:
                raise L.QkError(f"{paths[fi]}: short read of column chunk {plan.name!r}")
            got += n
    return view


def _decode_with_tables(plan, raw, runs_dev, n_runs, dense, dict_runs, dict_total, remap, registry, device, status):
    """The two decode launches (dictionary entries, then values) over `raw` = the bytes the run tables point into."""
    is_string = plan.physical == L.PQ_BYTE_ARRAY
    elem_dtype = _OUT_DTYPE[plan.physical]
    out = torch.empty(dense, dtype=elem_dtype, device=device)
    dictionary = None
    if is_string:
        dictionary = torch.tensor(remap or [0], dtype=torch.int32).to(device, non_blocking=True)
    elif plan.physical == L.PQ_BOOLEAN:
        dictionary = torch.tensor([0, 1], dtype=torch.uint8).to(device, non_blocking=True)     # RLE-coded booleans (V2 pages)
    elif dict_total:
        dr = np.array(dict_runs + [(dict_total, 0, 0, 0, 0, 0)], dtype=RUN_DTYPE)
        dr_dev = torch.from_numpy(dr.view(np.uint8).reshape(-1)).to(device, non_blocking=True)
        dictionary = torch.empty(dict_total, dtype=elem_dtype, device=device)
        ops.parquet_decode(raw, dr_dev, len(dict_runs), dict_total, None, dictionary, status)
    ops.parquet_decode(raw, runs_dev, n_runs, dense, dictionary, out, status)
    keep = _arrow_type_to_keep(plan.arrow_type, plan.name)
    if pa.types.is_decimal(plan.arrow_type):
        out = _decimal_to_f64(out, plan.arrow_type.scale)
    return DeviceColumn(out, registry.values[plan.name] if is_string else None, keep)


def _decimal_to_f64(unscaled: torch.Tensor, scale: int) -> torch.Tensor:
    """DECIMAL(p, s) stored as INT32 / INT64 (Spark's layout for p <= 18) -> fp64 = unscaled / 10^s: one pass of the
    projection kernel (K1); an IEEE division of two exactly representable numbers, i.e. the double nearest to the decimal."""
    if len(unscaled) == 0 or scale == 0:
        return unscaled.to(torch.float64)
    outs, _ = ops.scan_filter_project([unscaled], None, [[(L.OP_COL, 0, 0, 0.0, 0), (L.OP_CONST, 0, 0, float(10 ** scale), 0),
                                                         (L.OP_DIV, 0, 0, 0.0, 0)]], stable=True)
    return outs[0]


class _Prepared:
    """Host phase of one column: staged bytes + run table (UNCOMPRESSED) or page table (SNAPPY) + dictionary facts."""
    __slots__ = ("plan", "stage", "paged", "table", "n", "dense", "scratch_bytes", "dict_runs", "dict_total", "local_dicts")


def prepare_column(plan: _ColumnPlan, paths, files, stage) -> _Prepared:
    """Everything that needs no device and no shared state: read the chunks, walk their headers.  Runs on a worker
    thread (file reads and the libqk walker release the GIL)."""
    if plan.physical not in _OUT_DTYPE:
        raise L.QkError(f"column {plan.name!r}: physical type {plan.physical} is not supported")
    codecs = {c[4] for c in plan.chunks}
    if codecs - set(_CODEC):
        raise L.QkError(f"column {plan.name!r}: {sorted(codecs - set(_CODEC))} pages are not supported by the device decoder "
                        "(UNCOMPRESSED, SNAPPY, ZSTD and GZIP are; use the host reader for this file)")
    pr = _Prepared()
    pr.plan, pr.paged = plan, codecs != {"UNCOMPRESSED"}
    pr.stage = stage
    view = _stage_chunks(plan, paths, files, stage)
    is_string = plan.physical == L.PQ_BYTE_ARRAY
    pr.dict_runs, pr.dict_total, pr.local_dicts = [], 0, []
    pr.n = pr.dense = pr.scratch_bytes = 0
    pr.table = np.zeros(max(16, 4 * len(plan.chunks)), PAGE_DTYPE) if pr.paged else \
        np.zeros(max(64, plan.total_values // 256 + 4 * len(plan.chunks) + 2), RUN_DTYPE)
    for fi, start, size, nvals, compression, off in plan.chunks:
        first = pr.n
        if pr.paged:
            pr.table, pr.n, pr.dense, pr.scratch_bytes, info = walk_pages(view.ctypes.data, off, size, nvals, plan.physical, plan.max_def,
                                                                        _CODEC[compression], pr.dict_total, pr.table, pr.n, pr.dense,
                                                                        pr.scratch_bytes)
        else:
            pr.table, pr.n, pr.dense, info = walk_chunk(view.ctypes.data, off, size, nvals, plan.physical, plan.max_def, 0,
                                                        pr.dict_total, pr.table, pr.n, pr.dense)
        if info.dict_offset >= 0:
            if is_string and pr.paged:          # the (small) dictionary page is inflated on the host as well: its strings stay here
                dp = [p for p in pr.table[first:pr.n] if p["kind"] == L.PQ_PAGE_DICT][-1]
                body = view[int(dp["src_offset"]):int(dp["src_offset"]) + int(dp["src_bytes"])]
                if dp["compressed"]:
                    codec = _ARROW_CODEC[int(dp["compressed"])]
                    try:
                        body = np.frombuffer(pa.Codec(codec).decompress(body.tobytes(), decompressed_size=int(dp["dst_bytes"])), dtype=np.uint8)
                    except Exception as e:
                        raise L.QkError(f"column {plan.name!r}: corrupt {codec} dictionary page ({type(e).__name__})") from None
                pr.local_dicts.append(_dictionary_strings(body, 0, len(body), info.dict_num_values))
            elif is_string:
                pr.local_dicts.append(_dictionary_strings(view, info.dict_offset, info.dict_bytes, info.dict_num_values))
            else:
                pr.dict_runs.append((pr.dict_total, info.dict_offset, 0, L.PQ_RUN_PLAIN, 0, 0))
            pr.dict_total += info.dict_num_values
    if pr.dense != plan.total_values:
        raise L.QkError(f"column {plan.name!r}: decoded {pr.dense} of {plan.total_values} values")
    return pr


def decode_prepared(pr: _Prepared, device, registry: DictionaryRegistry, status) -> DeviceColumn:
    """Device phase: upload, (inflate + walk), decode.  Main thread, current stream."""
    plan = pr.plan
    remap = []
    for vals in pr.local_dicts:                 # registry order = column order = deterministic codes per rank
        remap.extend(registry.codes_for(plan.name, vals))
    raw = torch.empty(pr.stage.numel(), dtype=torch.uint8, device=device)
    raw.copy_(pr.stage, non_blocking=True)
    if pr.paged:
        return _decode_paged(pr, raw, remap, device, registry, status)
    runs = _sentinel(pr.table, pr.n, pr.dense)
    runs_dev = torch.from_numpy(runs.view(np.uint8).reshape(-1)).to(device, non_blocking=True)
    return _decode_with_tables(plan, raw, runs_dev, pr.n, pr.dense, pr.dict_runs, pr.dict_total, remap, registry, device, status)


class _PlainStrings(Exception):
    """A compressed string column turned out (after inflation) to hold PLAIN values, i.e. no dictionary codes."""


_PAGE_STATUS = ((2, "the column holds nulls (validity is outside the hot path)"), (4, "a value encoding outside PLAIN / RLE_DICTIONARY"),
                (8, "a corrupt compressed stream"), (16, "no inflate workspace"), (1, "a malformed page"))


def _decode_paged(pr: _Prepared, raw, remap, device, registry, status):
    """Chunks with a page codec: the host saw only page headers; pages are inflated, their run headers walked (count,
    then fill) and their values decoded on the device.  One host sync (the per-page run counts) sizes the run table."""
    plan, n_pages = pr.plan, pr.n
    pages_dev = torch.from_numpy(pr.table[:n_pages].view(np.uint8).reshape(-1)).to(device, non_blocking=True)
    scratch = torch.empty(pr.scratch_bytes + ops.PQ_PAD, dtype=torch.uint8, device=device)
    work = ops.parquet_inflate_workspace(int(np.count_nonzero(pr.table[:n_pages]["compressed"] >= L.PQ_CODEC_ZSTD)), device)
    ops.parquet_inflate(raw, pages_dev, n_pages, scratch, work)
    ops.parquet_page_runs(scratch, pages_dev, n_pages, plan.physical)                 # count pass
    table = pages_dev.cpu().numpy().view(PAGE_DTYPE)                                 # the one sync: run counts + page status
    bad = int(np.bitwise_or.reduce(table["status"])) if n_pages else 0
    if bad == 4 and plan.physical == L.PQ_BYTE_ARRAY:
        raise _PlainStrings()                           # strings without a dictionary: see read_row_groups
    for bit, what in _PAGE_STATUS:
        if bad & bit:
            raise L.QkError(f"column {plan.name!r}: {what}")
    counts = table["n_runs"].astype(np.int64)
    offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    n_runs = int(offsets[-1])
    runs_dev = torch.zeros((n_runs + 1) * RUN_DTYPE.itemsize, dtype=torch.uint8, device=device)
    runs_dev[n_runs * RUN_DTYPE.itemsize:].view(torch.int64)[0] = pr.dense             # the sentinel's dense_start
    ops.parquet_page_runs(scratch, pages_dev, n_pages, plan.physical, torch.from_numpy(offsets[:-1].copy()).to(device), runs_dev, n_runs)
    return _decode_with_tables(plan, scratch, runs_dev, n_runs, pr.dense, pr.dict_runs, pr.dict_total, remap, registry, device, status)


def _host_string_column(units, name, device, registry) -> DeviceColumn:
    """A string column stored without a dictionary: Arrow reads and dictionary-codes it on the host, the codes go up.
    (Also serves DECIMAL columns stored as FIXED_LEN_BYTE_ARRAY: Arrow casts them to fp64 on the host.)"""
    by_file = {}
    for path, g in units:
        by_file.setdefault(path, []).append(g)
    parts = [pq.ParquetFile(path).read_row_groups(groups, columns=[name])[name] for path, groups in by_file.items()]
    arr = pa.chunked_array([c for p in parts for c in p.chunks], type=parts[0].type)
    if arr.null_count:
        raise L.QkError(f"column {name!r} has nulls: validity bitmaps are not supported on the hot path")
    if pa.types.is_decimal(arr.type):
        from .columns import _arrow_to_device
        return _arrow_to_device(name, arr, device, registry)
    codes, vals = registry.encode(name, arr)
    return DeviceColumn(torch.from_numpy(codes.astype(np.int32)).to(device), vals, None)


def read_row_groups(units, columns=None, device=None, registry: DictionaryRegistry | None = None, nthreads: int = 4) -> DeviceTable:
    """[(path, row_group), ...] -> DeviceTable, decoded on `device`.  The host phase of the columns (file reads +
    header walks) runs on `nthreads` workers; the device phase follows column by column on the caller's stream."""
    from concurrent.futures import ThreadPoolExecutor
    from .columns import default_device
    device = device or default_device()
    registry = registry if registry is not None else DictionaryRegistry()
    paths, plans, rows = plan_batch(units, columns)
    pin = torch.device(device).type == "cuda"
    status = torch.zeros(1, dtype=torch.int32, device=device)
    order = columns if columns is not None else list(plans)
    host_side = set()
    for name in order:                              # outside-scope columns fail before anything is read
        if plans[name].physical == L.PQ_FIXED_LEN_BYTE_ARRAY and pa.types.is_decimal(plans[name].arrow_type):
            host_side.add(name)                     # DECIMAL as big-endian bytes (pyarrow's default layout): Arrow casts it
        elif plans[name].physical not in _OUT_DTYPE:
            raise L.QkError(f"column {name!r}: physical type {plans[name].physical} is not supported")
    stages = {name: _stage_alloc(plans[name], pin) for name in order if name not in host_side}
    files = [os.open(p, os.O_RDONLY) for p in paths]
    def prepare(name):
        if name in host_side:
            return None
        try:
            return prepare_column(plans[name], paths, files, stages[name])
        except L.QkError as e:
            # Strings live on the device only as dictionary codes whose value list stays on the host (DESIGN.md section 3).
            # A string column the writer did NOT dictionary-code has no codes in the file: its dictionary is built where
            # strings are handled anyway -- on the host, by Arrow -- and only the codes are uploaded.
            if plans[name].physical == L.PQ_BYTE_ARRAY and "PLAIN BYTE_ARRAY" in str(e):
                return None
            raise

    try:
        if nthreads > 1 and len(order) > 1:
            with ThreadPoolExecutor(min(nthreads, len(order))) as pool:
                prepared = list(pool.map(prepare, order))
        else:
            prepared = [prepare(name) for name in order]
    finally:
        for fd in files:
            os.close(fd)
    cols = {}
    for name, pr in zip(order, prepared):
        try:
            cols[name] = _host_string_column(units, name, device, registry) if pr is None else decode_prepared(pr, device, registry, status)
        except _PlainStrings:
            cols[name] = _host_string_column(units, name, device, registry)
    if int(status.item()):                          # also orders the pinned staging buffers' release after the copies
        raise L.QkError("Parquet decode: a dictionary index points outside its dictionary (corrupt file)")
    del prepared, stages
    return DeviceTable(cols)


# ---------------------------------------------------------------------------------------------- row-group pruning
def _cmp_possible(op, lo, hi, val):
    """Can any x in [lo, hi] satisfy `x op val`?"""
    try:
        if op in ("=", "=="):
            return lo <= val <= hi
        if op == "<":
            return lo < val
        if op == "<=":
            return lo <= val
        if op == ">":
            return hi > val
        if op == ">=":
            return hi >= val
        if op == "in":
            return any(lo <= v <= hi for v in val)
        # "!=" never prunes: min == max == literal does not rule out NaN rows, which satisfy x != literal
    except TypeError:
        return True
    return True


def _days(v):
    """date32 statistics / literals as days since the epoch (the device layout of a date column)."""
    import datetime as dt
    return (v - dt.date(1970, 1, 1)).days if type(v) is dt.date else v


def row_group_may_match(md, g, hints) -> bool:
    """hints: AND-ed [(column, op, literal)] -- False only when the row group's min/max statistics prove that no row
    can pass (the use the reference's sorted reader makes of statistics, pyquokka/dataset/ordered_readers.py:33-50)."""
    if not hints:
        return True
    names = md.schema.names
    rg = md.row_group(g)
    for col, op, val in hints:
        if col not in names:
            continue
        st = rg.column(names.index(col)).statistics
        if st is None or not st.has_min_max:
            continue
        v = [_days(x) for x in val] if isinstance(val, (list, tuple, set)) else _days(val)
        if not _cmp_possible(op, _days(st.min), _days(st.max), v):
            return False
    return True


_FLIP = {"<": ">", "<=": ">=", ">": "<", ">=": "<=", "=": "=", "!=": "!="}


def prune_hints(pred) -> list:
    """The `column op literal` conjuncts of a predicate (expr.Node), as row-group pruning hints.  The predicate itself
    still runs on the edge (K1); a hint only lets the reader skip row groups that cannot contribute."""
    from . import expr as E
    out = []
    for c in E.conjuncts(pred):
        if c.kind != "bin" or c.value not in _FLIP:
            continue
        a, b, op = c.args[0], c.args[1], c.value
        if a.kind != "col":
            a, b, op = b, a, _FLIP[op]
        if a.kind == "col" and b.kind in ("num", "date", "str"):
            out.append((a.value, op, b.value))
    return out


def filter_predicate(filters):
    """[(col, op, literal), ...] AND-ed (pyquokka/sql_utils.py:44-83) -> expr.Node for the device-side exact filter."""
    import datetime as dt
    from . import expr as E

    def lit(v):
        if isinstance(v, bool):
            return str(int(v))
        if type(v) is dt.date:
            return f"date '{v.isoformat()}'"
        if isinstance(v, str):
            return "'" + v.replace("'", "''") + "'"
        return repr(v)
    parts = []
    for col, op, val in filters:
        if op in ("in", "not in"):
            e = f"{col} in ({', '.join(lit(v) for v in val)})"
            parts.append(e if op == "in" else f"not ({e})")
        else:
            parts.append(f"{col} {'=' if op == '==' else op} {lit(val)}")
    return E.parse(" and ".join(f"({p})" for p in parts))
