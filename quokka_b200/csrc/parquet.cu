// parquet.cu -- Parquet column chunks decoded in HBM (include/qk.h: qk_parquet_walk_chunk, qk_parquet_decode).
//
// Stands in for the Arrow C++ reader the reference scans with (pyquokka/dataset/unordered_readers.py:51,98-99).
// Split of labour: the HOST walks the page headers (a few hundred bytes per page, Thrift compact protocol) and the
// run headers of dictionary-coded pages (one byte or two per <= 504 values) and writes a run table; the DEVICE turns
// the raw page bytes, copied as they lie in the file, into Arrow-layout columns -- one thread per value, output
// fully coalesced, every value byte read once.  Algorithmic bytes per value: encoded bytes in + elem_bytes out.
#include "common.cuh"
#include "parquet_core.h"
#include "zstd_core.h"
#include "deflate_core.h"

namespace {
using namespace qkpq;

// ------------------------------------------------------------------------------------ Thrift compact protocol
enum { T_STOP = 0, T_TRUE = 1, T_FALSE = 2, T_BYTE = 3, T_I16 = 4, T_I32 = 5, T_I64 = 6, T_DOUBLE = 7, T_BINARY = 8,
       T_LIST = 9, T_SET = 10, T_MAP = 11, T_STRUCT = 12 };

void skip_value(Cursor& c, int type, int depth);

void skip_struct(Cursor& c, int depth) {
    if (depth > 16) { c.ok = false; return; }
    while (c.ok) {
        if (c.pos >= c.end) { c.ok = false; return; }
        const uint8_t b = c.p[c.pos++];
        if (b == T_STOP) return;
        if ((b >> 4) == 0) read_zigzag(c);              // long-form field id
        skip_value(c, b & 0x0f, depth + 1);
    }
}
void skip_value(Cursor& c, int type, int depth) {
    if (depth > 16) { c.ok = false; return; }
    switch (type) {
        case T_TRUE: case T_FALSE: return;                    // value lives in the field header
        case T_BYTE: c.pos += 1; break;
        case T_I16: case T_I32: case T_I64: read_uvarint(c); break;
        case T_DOUBLE: c.pos += 8; break;
        case T_BINARY: { const uint64_t n = read_uvarint(c); c.pos += (int64_t)n; } break;
        case T_LIST: case T_SET: {
            if (c.pos >= c.end) { c.ok = false; return; }
            const uint8_t h = c.p[c.pos++];
            uint64_t n = h >> 4;
            if (n == 15) n = read_uvarint(c);
            const int et = h & 0x0f;
            for (uint64_t i = 0; i < n && c.ok; i++) {
                if (et == T_TRUE || et == T_FALSE) c.pos += 1;   // list elements of type bool take a byte each
                else skip_value(c, et, depth + 1);
            }
        } break;
        case T_MAP: {
            const uint64_t n = read_uvarint(c);
            if (n) {
                if (c.pos >= c.end) { c.ok = false; return; }
                const uint8_t kv = c.p[c.pos++];
                for (uint64_t i = 0; i < n && c.ok; i++) { skip_value(c, kv >> 4, depth + 1); skip_value(c, kv & 0x0f, depth + 1); }
            }
        } break;
        case T_STRUCT: skip_struct(c, depth + 1); break;
        default: c.ok = false;
    }
    if (c.pos > c.end) c.ok = false;
}

// Iterates the fields of the struct at the cursor: returns the field id and wire type, 0 at STOP.
int next_field(Cursor& c, int& last_id, int& type) {
    if (c.pos >= c.end) { c.ok = false; return 0; }
    const uint8_t b = c.p[c.pos++];
    if (b == T_STOP) return 0;
    type = b & 0x0f;
    const int delta = b >> 4;
    last_id = delta ? last_id + delta : (int)read_zigzag(c);
    return c.ok ? last_id : 0;
}

// parquet.thrift PageHeader and the three page-type headers, reduced to what the decoder needs
enum { PAGE_DATA = 0, PAGE_INDEX = 1, PAGE_DICT = 2, PAGE_DATA_V2 = 3 };
enum { ENC_PLAIN = PQ_ENC_PLAIN, ENC_PLAIN_DICT = PQ_ENC_PLAIN_DICT, ENC_RLE = PQ_ENC_RLE, ENC_RLE_DICT = PQ_ENC_RLE_DICT };
struct PageHeader {
    int type = -1;
    int64_t uncompressed = -1, compressed = -1;
    int64_t num_values = -1;
    int encoding = -1, def_encoding = -1, rep_encoding = -1;
    int64_t num_nulls = 0, def_bytes = 0, rep_bytes = 0;          // V2
    bool is_compressed = true;                                     // V2 (default true)
};

void parse_inner(Cursor& c, PageHeader& h, int which) {
    int id = 0, type = 0;
    while (c.ok && next_field(c, id, type)) {
        const bool is_int = type == T_I32 || type == T_I16 || type == T_I64;
        if (which == PAGE_DATA && is_int && id >= 1 && id <= 4) {
            const int64_t v = read_zigzag(c);
            if (id == 1) h.num_values = v; else if (id == 2) h.encoding = (int)v;
            else if (id == 3) h.def_encoding = (int)v; else h.rep_encoding = (int)v;
        } else if (which == PAGE_DICT && is_int && id >= 1 && id <= 2) {
            const int64_t v = read_zigzag(c);
            if (id == 1) h.num_values = v; else h.encoding = (int)v;
        } else if (which == PAGE_DATA_V2 && is_int && id >= 1 && id <= 6) {
            const int64_t v = read_zigzag(c);
            if (id == 1) h.num_values = v; else if (id == 2) h.num_nulls = v; else if (id == 4) h.encoding = (int)v;
            else if (id == 5) h.def_bytes = v; else if (id == 6) h.rep_bytes = v;
        } else if (which == PAGE_DATA_V2 && id == 7 && (type == T_TRUE || type == T_FALSE)) {
            h.is_compressed = type == T_TRUE;
        } else {
            skip_value(c, type, 0);
        }
    }
}

bool parse_page_header(Cursor& c, PageHeader& h) {
    int id = 0, type = 0;
    while (c.ok && next_field(c, id, type)) {
        if (id == 1 && type == T_I32) h.type = (int)read_zigzag(c);
        else if (id == 2 && type == T_I32) h.uncompressed = read_zigzag(c);
        else if (id == 3 && type == T_I32) h.compressed = read_zigzag(c);
        else if (id == 5 && type == T_STRUCT) parse_inner(c, h, PAGE_DATA);
        else if (id == 7 && type == T_STRUCT) parse_inner(c, h, PAGE_DICT);
        else if (id == 8 && type == T_STRUCT) parse_inner(c, h, PAGE_DATA_V2);
        else skip_value(c, type, 0);
    }
    return c.ok && h.type >= 0 && h.compressed >= 0;
}

const char* encoding_name(int e) {
    switch (e) {
        case 0: return "PLAIN"; case 2: return "PLAIN_DICTIONARY"; case 3: return "RLE"; case 4: return "BIT_PACKED";
        case 5: return "DELTA_BINARY_PACKED"; case 6: return "DELTA_LENGTH_BYTE_ARRAY"; case 7: return "DELTA_BYTE_ARRAY";
        case 8: return "RLE_DICTIONARY"; case 9: return "BYTE_STREAM_SPLIT"; default: return "unknown";
    }
}

// ------------------------------------------------------------------------------------ device decode
constexpr int PQ_THREADS = 256;
constexpr int PQ_ITEMS = 8;     // values per thread: a CTA covers 2048 consecutive values

template <int EB>
__global__ void __launch_bounds__(PQ_THREADS) k_pq_decode(const uint8_t* __restrict__ bytes, const qk_pq_run* __restrict__ runs,
                                                          int64_t n_runs, int64_t n_values, const void* __restrict__ dictionary,
                                                          int64_t dict_len, typename ElemOf<EB>::type* __restrict__ out,
                                                          int32_t* __restrict__ status) {
    __shared__ int64_t s_run[2];
    const int64_t tile = (int64_t)blockIdx.x * (PQ_THREADS * PQ_ITEMS);
    const int64_t tile_end = min(tile + (int64_t)PQ_THREADS * PQ_ITEMS, n_values);
    // the runs that overlap this tile: two searches of the whole table, then every thread searches only that window
    if (threadIdx.x == 0) s_run[0] = find_run(runs, n_runs, tile);
    if (threadIdx.x == 32) s_run[1] = find_run(runs, n_runs, tile_end - 1);
    __syncthreads();
    const int64_t r0 = s_run[0], nr = s_run[1] - s_run[0] + 1;
    int bad = 0;
#pragma unroll
    for (int j = 0; j < PQ_ITEMS; j++) {
        const int64_t t = tile + (int64_t)j * PQ_THREADS + threadIdx.x;
        if (t < tile_end) {
            const qk_pq_run r = runs[r0 + find_run(runs + r0, nr, t)];
            out[t] = decode_value<EB>(bytes, r, t, dictionary, dict_len, &bad);
        }
    }
    if (bad && status) atomicOr(status, 1);
}

}  // namespace

// ------------------------------------------------------------------------------------ C-ABI
namespace {

int elem_of(int physical_type) {                    // 0 BOOLEAN, 4 / 8 fixed width, -1 BYTE_ARRAY, -2 unsupported
    switch (physical_type) {
        case QK_PQ_BOOLEAN: return 0;
        case QK_PQ_INT32: case QK_PQ_FLOAT: return 4;
        case QK_PQ_INT64: case QK_PQ_DOUBLE: return 8;
        case QK_PQ_BYTE_ARRAY: return -1;
        default: return -2;
    }
}

// One pass over the page headers of a column chunk.  `on_dict(header, payload, page_end)` / `on_data(...)` return 0 or
// an error code (after QK_FAIL-style set_err).
template <class OnDict, class OnData>
int for_each_page(const char* who, const uint8_t* bytes, int64_t chunk_offset, int64_t chunk_bytes, int64_t num_values,
                  OnDict on_dict, OnData on_data) {
    int64_t pos = chunk_offset, seen = 0;
    const int64_t end = chunk_offset + chunk_bytes;
    while (seen < num_values) {
        if (pos >= end) QK_FAIL(QK_ERR_INVALID, "%s: chunk ends after %lld of %lld values", who, (long long)seen, (long long)num_values);
        Cursor c{bytes, pos, end, true};
        PageHeader h;
        if (!parse_page_header(c, h)) QK_FAIL(QK_ERR_INVALID, "%s: malformed page header at byte %lld", who, (long long)pos);
        const int64_t data = c.pos, page_end = data + h.compressed;
        if (page_end > end) QK_FAIL(QK_ERR_INVALID, "%s: page at byte %lld runs past the chunk", who, (long long)pos);
        pos = page_end;
        if (h.type == PAGE_INDEX) continue;
        if (h.type == PAGE_DICT) {
            if (h.encoding != ENC_PLAIN && h.encoding != ENC_PLAIN_DICT)
                QK_FAIL(QK_ERR_UNSUPPORTED, "%s: dictionary page encoding %s is not supported", who, encoding_name(h.encoding));
            if (h.num_values < 0 || h.num_values > 0x7fffffffLL) QK_FAIL(QK_ERR_INVALID, "%s: dictionary page value count", who);
            const int rc = on_dict(h, data, page_end);
            if (rc) return rc;
            continue;
        }
        if (h.type != PAGE_DATA && h.type != PAGE_DATA_V2) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: page type %d", who, h.type);
        if (h.num_values < 0 || seen + h.num_values > num_values)
            QK_FAIL(QK_ERR_INVALID, "%s: page value counts exceed the chunk's %lld values", who, (long long)num_values);
        if (h.type == PAGE_DATA_V2) {
            if (h.num_nulls != 0) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: the column holds nulls (validity is outside the hot path)", who);
            if (h.rep_bytes != 0) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: repeated (nested) columns are not supported", who);
            if (h.def_bytes < 0 || data + h.def_bytes > page_end) QK_FAIL(QK_ERR_INVALID, "%s: level bytes exceed the page", who);
        }
        const int rc = on_data(h, data, page_end, seen);
        if (rc) return rc;
        seen += h.num_values;
    }
    return QK_OK;
}

int values_error(const char* who, int rc, int encoding, int64_t page_at, long long cap) {
    switch (rc) {
        case PQ_OK: return QK_OK;
        case PQ_E_FULL: QK_FAIL(QK_ERR_CAPACITY, "%s: run table full (%lld)", who, cap);
        case PQ_E_PLAIN_BYTE_ARRAY: QK_FAIL(QK_ERR_UNSUPPORTED, "%s: PLAIN BYTE_ARRAY values (strings are supported as dictionary codes only)", who);
        case PQ_E_ENCODING: QK_FAIL(QK_ERR_UNSUPPORTED, "%s: value encoding %s is not supported", who, encoding_name(encoding));
        case PQ_E_SHORT: QK_FAIL(QK_ERR_INVALID, "%s: the page at byte %lld is shorter than its values", who, (long long)page_at);
        case PQ_E_WIDTH: QK_FAIL(QK_ERR_INVALID, "%s: index bit width out of range in the page at byte %lld", who, (long long)page_at);
        default: QK_FAIL(QK_ERR_INVALID, "%s: malformed RLE / bit-packed run in the page at byte %lld", who, (long long)page_at);
    }
}

constexpr int INFLATE_WARPS = 4;      // warps per CTA of the inflate kernel
constexpr size_t ZSTD_SLOT_BYTES = (sizeof(qkzstd::ZstdWork) + 15) / 16 * 16 + qkzstd::ZS_BLOCK_MAX;

// Warp w handles pages w, w + W, w + 2W, ... (W = warps in the grid).  Stored pages: a byte copy.  Snappy pages: lane 0
// walks the element tags, every lane moves its share of the element's bytes; __syncwarp() orders an element's writes
// before the next element's reads.  ZSTD / GZIP pages: lane 0 runs the sequential decoder with the warp's workspace slot.
__global__ void __launch_bounds__(INFLATE_WARPS * 32) k_pq_inflate(const uint8_t* __restrict__ bytes, qk_pq_page* __restrict__ pages,
                                                                  int64_t n_pages, uint8_t* __restrict__ scratch, uint8_t* work,
                                                                  int64_t n_slots) {
    const int64_t warp = (int64_t)blockIdx.x * INFLATE_WARPS + (threadIdx.x >> 5);
    const int64_t n_warps = (int64_t)gridDim.x * INFLATE_WARPS;
    const int lane = threadIdx.x & 31;
    for (int64_t pi = warp; pi < n_pages; pi += n_warps) {
        const qk_pq_page p = pages[pi];
        uint8_t* dst = scratch + p.dst_offset;
        const uint8_t* src = bytes + p.src_offset;
        if (p.compressed == QK_PQ_CODEC_NONE) {
            const int64_t n = p.src_bytes < p.dst_bytes ? p.src_bytes : p.dst_bytes;
            for (int64_t i = lane; i < n; i += 32) dst[i] = src[i];
            if (lane == 0 && p.src_bytes != p.dst_bytes) pages[pi].status |= 8;
        } else if (p.compressed == QK_PQ_CODEC_ZSTD || p.compressed == QK_PQ_CODEC_GZIP) {
            if (lane == 0) {
                if (warp >= n_slots || !work) {
                    pages[pi].status |= 16;
                } else if (p.compressed == QK_PQ_CODEC_ZSTD) {
                    uint8_t* slot = work + warp * ZSTD_SLOT_BYTES;
                    qkzstd::ZstdWork& w = *(qkzstd::ZstdWork*)slot;
                    uint8_t* lit = slot + (sizeof(qkzstd::ZstdWork) + 15) / 16 * 16;
                    if (qkzstd::zstd_decompress(w, src, p.src_bytes, dst, p.dst_bytes, lit, qkzstd::ZS_BLOCK_MAX) != qkzstd::ZS_OK)
                        pages[pi].status |= 8;
                } else {
                    qkdeflate::InflateWork& w = *(qkdeflate::InflateWork*)(work + warp * ZSTD_SLOT_BYTES);
                    if (qkdeflate::gzip_decompress(w, src, p.src_bytes, dst, p.dst_bytes) != qkdeflate::DF_OK) pages[pi].status |= 8;
                }
            }
        } else {
            int64_t ip = 0, op = 0;
            int bad = 0;
            if (lane == 0) {
                Cursor c{src, 0, p.src_bytes, true};
                const uint64_t ulen = read_uvarint(c);
                ip = c.pos;
                if (!c.ok || (int64_t)ulen != p.dst_bytes) bad = 1;
            }
            bad = __shfl_sync(0xffffffffu, bad, 0);
            while (!bad) {
                SnappyElem e;
                int more = 0;
                if (lane == 0) {
                    more = ip < p.src_bytes ? 1 : 0;
                    if (more) {
                        if (!snappy_next(src, ip, p.src_bytes, e)) more = -1;
                        else if (op + e.len > p.dst_bytes || (e.is_copy && (e.arg <= 0 || e.arg > op))) more = -1;
                    }
                }
                more = __shfl_sync(0xffffffffu, more, 0);
                if (more <= 0) { bad = more < 0; break; }
                e.is_copy = __shfl_sync(0xffffffffu, e.is_copy, 0);
                e.len = __shfl_sync(0xffffffffu, e.len, 0);
                e.arg = __shfl_sync(0xffffffffu, e.arg, 0);
                snappy_apply(dst, op, src, e, lane, 32);
                op += e.len;
                __syncwarp();
            }
            if (lane == 0 && (bad || op != p.dst_bytes)) pages[pi].status |= 8;
        }
        __syncwarp();
    }
}

// One thread per page: the run-header walk over the inflated images (count pass, then fill pass).
__global__ void __launch_bounds__(128) k_pq_page_runs(const uint8_t* __restrict__ img, qk_pq_page* __restrict__ pages, int64_t n_pages,
                                                      int elem, const int64_t* __restrict__ run_offsets, qk_pq_run* __restrict__ runs,
                                                      int64_t runs_cap) {
    const int64_t pi = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (pi >= n_pages) return;
    const qk_pq_page p = pages[pi];
    int status = 0;
    if (run_offsets) {
        const int64_t at = run_offsets[pi];
        const int64_t cap = at + p.n_runs <= runs_cap ? p.n_runs : 0;
        const int64_t n = page_runs(img, p, elem, cap ? runs + at : nullptr, cap, &status);
        if (n != p.n_runs || (p.n_runs && !cap)) status |= 1;
    } else {
        const int64_t n = page_runs(img, p, elem, nullptr, 0, &status);
        pages[pi].n_runs = n > 0x7fffffffLL ? 0x7fffffff : (int32_t)n;
    }
    if (status) pages[pi].status |= status;
}

}  // namespace

extern "C" {

int qk_parquet_walk_chunk(const uint8_t* bytes, int64_t chunk_offset, int64_t chunk_bytes, int64_t num_values,
                          int32_t physical_type, int32_t max_def_level, int32_t compression, int32_t dict_base,
                          qk_pq_run* runs, int64_t runs_cap, int64_t* n_runs, int64_t* dense, qk_pq_chunk_info* info) {
    const char* who = "qk_parquet_walk_chunk";
    if (!bytes || !n_runs || !dense || !info || (!runs && runs_cap > 0)) QK_FAIL(QK_ERR_INVALID, "%s: null argument", who);
    if (chunk_offset < 0 || chunk_bytes < 0 || num_values < 0 || *n_runs < 0 || *dense < 0) QK_FAIL(QK_ERR_INVALID, "%s: negative size", who);
    if (max_def_level < 0 || max_def_level > 1) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: nested columns (max definition level %d) are not supported", who, max_def_level);
    if (compression != 0) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: compressed pages (codec %d) need the paged path (qk_parquet_walk_pages)", who, compression);
    const int elem = elem_of(physical_type);
    if (elem == -2) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: physical type %d (INT96 / FIXED_LEN_BYTE_ARRAY) is not supported", who, physical_type);
    qk_pq_chunk_info ci;
    ci.dict_offset = -1; ci.dict_bytes = 0; ci.n_values = 0; ci.dict_num_values = 0; ci.n_data_pages = 0;
    FillSink sink{runs, *n_runs, runs_cap};
    const int64_t dense0 = *dense;
    const int rc = for_each_page(who, bytes, chunk_offset, chunk_bytes, num_values,
        [&](const PageHeader& h, int64_t data, int64_t page_end) -> int {
            if (elem == 0) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: dictionary-coded BOOLEAN column", who);
            if (elem > 0 && h.num_values * elem > page_end - data) QK_FAIL(QK_ERR_INVALID, "%s: dictionary page shorter than its %lld values", who, (long long)h.num_values);
            ci.dict_offset = data; ci.dict_bytes = page_end - data; ci.dict_num_values = (int32_t)h.num_values;
            return 0;
        },
        [&](const PageHeader& h, int64_t data, int64_t page_end, int64_t seen) -> int {
            int64_t v0 = data;
            if (h.type == PAGE_DATA) {
                if (max_def_level > 0) {
                    if (h.def_encoding != ENC_RLE) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: definition levels encoded as %s", who, encoding_name(h.def_encoding));
                    if (v0 + 4 > page_end) QK_FAIL(QK_ERR_INVALID, "%s: truncated definition levels", who);
                    const int64_t len = (int64_t)bytes[v0] | ((int64_t)bytes[v0 + 1] << 8) | ((int64_t)bytes[v0 + 2] << 16) | ((int64_t)bytes[v0 + 3] << 24);
                    if (v0 + 4 + len > page_end) QK_FAIL(QK_ERR_INVALID, "%s: truncated definition levels", who);
                    const int ok = levels_all_defined(bytes, v0 + 4, v0 + 4 + len, h.num_values, max_def_level);
                    if (ok < 0) QK_FAIL(QK_ERR_INVALID, "%s: malformed definition levels", who);
                    if (ok == 0) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: the column holds nulls (validity is outside the hot path)", who);
                    v0 += 4 + len;
                }
            } else {
                v0 += h.rep_bytes + h.def_bytes;
            }
            if ((h.encoding == ENC_RLE_DICT || h.encoding == ENC_PLAIN_DICT) && ci.dict_offset < 0)
                QK_FAIL(QK_ERR_INVALID, "%s: dictionary-coded page without a dictionary page", who);
            const int vrc = walk_values(bytes, v0, page_end, h.num_values, h.encoding, elem, dict_base, dense0 + seen, sink);
            if (vrc) return values_error(who, vrc, h.encoding, data, (long long)runs_cap);
            ci.n_values += h.num_values;
            ci.n_data_pages++;
            return 0;
        });
    if (rc) return rc;
    *n_runs = sink.n;
    *dense = dense0 + ci.n_values;
    *info = ci;
    return QK_OK;
}

int qk_parquet_walk_pages(const uint8_t* bytes, int64_t chunk_offset, int64_t chunk_bytes, int64_t num_values,
                          int32_t physical_type, int32_t max_def_level, int32_t compression, int32_t dict_base,
                          qk_pq_page* pages, int64_t pages_cap, int64_t* n_pages, int64_t* dense, int64_t* scratch_bytes,
                          qk_pq_chunk_info* info) {
    const char* who = "qk_parquet_walk_pages";
    if (!bytes || !n_pages || !dense || !scratch_bytes || !info || (!pages && pages_cap > 0)) QK_FAIL(QK_ERR_INVALID, "%s: null argument", who);
    if (chunk_offset < 0 || chunk_bytes < 0 || num_values < 0 || *n_pages < 0 || *dense < 0 || *scratch_bytes < 0) QK_FAIL(QK_ERR_INVALID, "%s: negative size", who);
    if (max_def_level < 0 || max_def_level > 1) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: nested columns (max definition level %d) are not supported", who, max_def_level);
    if (compression < QK_PQ_CODEC_NONE || compression > QK_PQ_CODEC_GZIP)
        QK_FAIL(QK_ERR_UNSUPPORTED, "%s: page codec %d is not supported (UNCOMPRESSED, SNAPPY, ZSTD and GZIP are)", who, compression);
    const int elem = elem_of(physical_type);
    if (elem == -2) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: physical type %d (INT96 / FIXED_LEN_BYTE_ARRAY) is not supported", who, physical_type);
    qk_pq_chunk_info ci;
    ci.dict_offset = -1; ci.dict_bytes = 0; ci.n_values = 0; ci.dict_num_values = 0; ci.n_data_pages = 0;
    int64_t np = *n_pages, scratch = *scratch_bytes;
    const int64_t dense0 = *dense;
    auto push = [&](const PageHeader& h, int kind, int64_t src, int64_t src_bytes, int64_t dst_bytes, int64_t dense_start, int codec) -> int {
        if (np >= pages_cap) QK_FAIL(QK_ERR_CAPACITY, "%s: page table full (%lld)", who, (long long)pages_cap);
        if (src_bytes < 0 || dst_bytes < 0 || src_bytes > 0x7fffffffLL || dst_bytes > 0x7fffffffLL) QK_FAIL(QK_ERR_INVALID, "%s: page size out of range", who);
        qk_pq_page& p = pages[np++];
        p.src_offset = src; p.dst_offset = scratch; p.dense_start = dense_start;
        p.src_bytes = (int32_t)src_bytes; p.dst_bytes = (int32_t)dst_bytes; p.num_values = (int32_t)h.num_values;
        p.dict_base = dict_base; p.n_runs = 0; p.kind = (uint8_t)kind; p.encoding = (uint8_t)h.encoding;
        p.compressed = (uint8_t)codec; p.max_def = (uint8_t)max_def_level; p.status = 0; p.reserved = 0;
        scratch += (dst_bytes + 7) / 8 * 8;
        return 0;
    };
    const int rc = for_each_page(who, bytes, chunk_offset, chunk_bytes, num_values,
        [&](const PageHeader& h, int64_t data, int64_t page_end) -> int {
            if (elem == 0) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: dictionary-coded BOOLEAN column", who);
            if (h.uncompressed < 0) QK_FAIL(QK_ERR_INVALID, "%s: page header without an uncompressed size", who);
            if (elem > 0 && h.num_values * elem > h.uncompressed) QK_FAIL(QK_ERR_INVALID, "%s: dictionary page shorter than its %lld values", who, (long long)h.num_values);
            ci.dict_offset = scratch; ci.dict_bytes = h.uncompressed; ci.dict_num_values = (int32_t)h.num_values;
            return push(h, QK_PQ_PAGE_DICT, data, page_end - data, h.uncompressed, dict_base, compression);
        },
        [&](const PageHeader& h, int64_t data, int64_t page_end, int64_t seen) -> int {
            if (h.uncompressed < 0) QK_FAIL(QK_ERR_INVALID, "%s: page header without an uncompressed size", who);
            if (h.encoding < 0 || h.encoding > 255) QK_FAIL(QK_ERR_INVALID, "%s: bad encoding id", who);
            if ((h.encoding == ENC_RLE_DICT || h.encoding == ENC_PLAIN_DICT) && ci.dict_offset < 0)
                QK_FAIL(QK_ERR_INVALID, "%s: dictionary-coded page without a dictionary page", who);
            if (h.num_values > 0x7fffffffLL) QK_FAIL(QK_ERR_INVALID, "%s: page value count out of range", who);
            int prc;
            if (h.type == PAGE_DATA) {
                if (max_def_level > 0 && h.def_encoding != ENC_RLE) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: definition levels encoded as %s", who, encoding_name(h.def_encoding));
                prc = push(h, QK_PQ_PAGE_DATA_V1, data, page_end - data, h.uncompressed, dense0 + seen, compression);
            } else {
                const int64_t lv = h.rep_bytes + h.def_bytes;           // stored in front of the (optionally compressed) values
                if (h.uncompressed < lv) QK_FAIL(QK_ERR_INVALID, "%s: level bytes exceed the page", who);
                prc = push(h, QK_PQ_PAGE_DATA_V2, data + lv, page_end - data - lv, h.uncompressed - lv, dense0 + seen,
                           h.is_compressed ? compression : QK_PQ_CODEC_NONE);
            }
            if (prc) return prc;
            ci.n_values += h.num_values;
            ci.n_data_pages++;
            return 0;
        });
    if (rc) return rc;
    *n_pages = np;
    *dense = dense0 + ci.n_values;
    *scratch_bytes = scratch;
    *info = ci;
    return QK_OK;
}

// one slot per ZSTD / GZIP page in flight: at most 8 per SM, in whole CTAs
size_t qk_parquet_inflate_workspace_bytes(int64_t n_zstd_pages) {
    if (n_zstd_pages <= 0) return 0;
    const int64_t cap = (int64_t)qk::sm_count() * 8;
    const int64_t slots = n_zstd_pages < cap ? n_zstd_pages : cap;
    return (size_t)((slots + INFLATE_WARPS - 1) / INFLATE_WARPS * INFLATE_WARPS) * ZSTD_SLOT_BYTES;
}

int qk_parquet_inflate(const uint8_t* bytes, int64_t n_bytes, qk_pq_page* pages, int64_t n_pages, uint8_t* scratch,
                       int64_t scratch_bytes, void* work, int64_t work_bytes, void* stream) {
    const char* who = "qk_parquet_inflate";
    if (n_pages < 0 || n_bytes < 0 || scratch_bytes < 0 || work_bytes < 0) QK_FAIL(QK_ERR_INVALID, "%s: negative size", who);
    if (n_pages == 0) return QK_OK;
    if (!bytes || !pages || !scratch) QK_FAIL(QK_ERR_INVALID, "%s: null argument", who);
    if (work && ((uintptr_t)work & 15)) QK_FAIL(QK_ERR_INVALID, "%s: workspace must be 16-byte aligned", who);
    // one warp per page; with a workspace, no more warps than slots (a ZSTD page needs its warp's slot), in whole CTAs
    int64_t grid = (n_pages + INFLATE_WARPS - 1) / INFLATE_WARPS;
    int64_t n_slots = 0;
    if (work) {
        const int64_t ctas = work_bytes / (int64_t)(ZSTD_SLOT_BYTES * INFLATE_WARPS);
        if (ctas < 1) QK_FAIL(QK_ERR_CAPACITY, "%s: workspace smaller than %d slots of %zu bytes", who, INFLATE_WARPS, ZSTD_SLOT_BYTES);
        if (grid > ctas) grid = ctas;
        n_slots = grid * INFLATE_WARPS;
    }
    if (grid > 0x7fffffffLL) QK_FAIL(QK_ERR_INVALID, "%s: too many pages", who);
    k_pq_inflate<<<(unsigned)grid, INFLATE_WARPS * 32, 0, (cudaStream_t)stream>>>(bytes, pages, n_pages, scratch, (uint8_t*)work, n_slots);
    QK_LAUNCH_CHECK(who);
    return QK_OK;
}

int qk_parquet_page_runs(const uint8_t* scratch, int64_t scratch_bytes, qk_pq_page* pages, int64_t n_pages, int32_t physical_type,
                         const int64_t* run_offsets, qk_pq_run* runs, int64_t runs_cap, void* stream) {
    const char* who = "qk_parquet_page_runs";
    if (n_pages < 0 || scratch_bytes < 0 || runs_cap < 0) QK_FAIL(QK_ERR_INVALID, "%s: negative size", who);
    if (n_pages == 0) return QK_OK;
    if (!scratch || !pages || (run_offsets && !runs && runs_cap > 0)) QK_FAIL(QK_ERR_INVALID, "%s: null argument", who);
    const int elem = elem_of(physical_type);
    if (elem == -2) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: physical type %d is not supported", who, physical_type);
    const int64_t grid = (n_pages + 127) / 128;
    k_pq_page_runs<<<(unsigned)grid, 128, 0, (cudaStream_t)stream>>>(scratch, pages, n_pages, elem, run_offsets, runs, runs_cap);
    QK_LAUNCH_CHECK(who);
    return QK_OK;
}

int qk_parquet_decode(const uint8_t* bytes, int64_t n_bytes, const qk_pq_run* runs, int64_t n_runs, int64_t n_values,
                      const void* dictionary, int64_t dict_len, int32_t elem_bytes, void* out, int32_t* status, void* stream) {
    const char* who = "qk_parquet_decode";
    if (n_values < 0 || n_runs < 0 || n_bytes < 0 || dict_len < 0) QK_FAIL(QK_ERR_INVALID, "%s: negative size", who);
    if (n_values == 0) return QK_OK;
    if (!bytes || !runs || !out || n_runs == 0) QK_FAIL(QK_ERR_INVALID, "%s: null argument", who);
    if (((uintptr_t)bytes & 7) || ((uintptr_t)runs & 7)) QK_FAIL(QK_ERR_INVALID, "%s: bytes / runs must be 8-byte aligned", who);
    if (dict_len > 0 && !dictionary) QK_FAIL(QK_ERR_INVALID, "%s: null dictionary", who);
    if ((uintptr_t)out % (elem_bytes > 0 ? elem_bytes : 1)) QK_FAIL(QK_ERR_INVALID, "%s: misaligned output", who);
    const int64_t per_cta = (int64_t)PQ_THREADS * PQ_ITEMS;
    const int64_t grid = (n_values + per_cta - 1) / per_cta;
    if (grid > 0x7fffffffLL) QK_FAIL(QK_ERR_INVALID, "%s: too many values", who);
    cudaStream_t s = (cudaStream_t)stream;
    switch (elem_bytes) {
        case 1: k_pq_decode<1><<<(unsigned)grid, PQ_THREADS, 0, s>>>(bytes, runs, n_runs, n_values, dictionary, dict_len, (uint8_t*)out, status); break;
        case 4: k_pq_decode<4><<<(unsigned)grid, PQ_THREADS, 0, s>>>(bytes, runs, n_runs, n_values, dictionary, dict_len, (uint32_t*)out, status); break;
        case 8: k_pq_decode<8><<<(unsigned)grid, PQ_THREADS, 0, s>>>(bytes, runs, n_runs, n_values, dictionary, dict_len, (uint64_t*)out, status); break;
        default: QK_FAIL(QK_ERR_INVALID, "%s: elem_bytes must be 1, 4 or 8", who);
    }
    QK_LAUNCH_CHECK(who);
    return QK_OK;
}

}  // extern "C"
