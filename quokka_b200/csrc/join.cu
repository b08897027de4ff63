// join.cu -- K4 hash build / K5 hash probe (BuildProbeJoinExecutor, sql_executors.py:325-377).
//
// Open addressing, linear probing, 16-byte slots {int64 key, int32 build_row, pad}: one 16-byte load
// fetches key and payload index, and a probe touches one 32-byte DRAM sector in the common case.
// Bound: HBM random access -- 16 B/build row written, >= 32 B sector per probe row read (DESIGN.md).
// Duplicate build keys each own a slot (Polars multiplies rows); the probe counts matches first, a warp
// shuffle scan turns counts into offsets and ONE atomic per warp reserves output space (ballot/shfl
// conflict resolution instead of one atomic per row), then the chain is re-walked (L1/L2 hits) to write.
//
// The ordered probe (DataStream.join(maintain_sort_order=...)) writes the same pairs in a fixed order instead: a count pass,
// the shared count-to-offsets scan, and a write pass that puts probe row i's pairs at its offset, its matches in ascending
// build-row number.  The build inserts duplicate keys into slots in nondeterministic chain order, so a row's matches are
// sorted where they are written: up to ORDER_INLINE by the thread that wrote them, more by one CTA per row (bitonic).
// qk_join_place puts rows that come back from the key owners into left order: a count per position, the same scan, and
// offset + index within the position's run.
#include "common.cuh"

namespace qk {
namespace {

constexpr long long EMPTY_KEY = (long long)0x8000000000000000ULL;
struct __align__(16) Slot { long long key; int idx; int pad; };

__global__ void __launch_bounds__(256) k_join_init(Slot* slots, int64_t capacity) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < capacity; i += (int64_t)gridDim.x * blockDim.x)
        slots[i] = Slot{EMPTY_KEY, -1, 0};
}

__global__ void __launch_bounds__(256) k_join_build(Slot* slots, uint64_t mask, const void* key, int dt, int64_t n,
                                                    int row_base, int* flags) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const long long k = load_i64(key, dt, i);
        if (k == EMPTY_KEY) { if (flags) atomicOr(flags, 2); continue; }
        uint64_t s = mix64((uint64_t)k) & mask;
        bool placed = false;
        for (uint64_t tries = 0; tries <= mask; ++tries) {
            const long long old = (long long)atomicCAS((unsigned long long*)&slots[s].key, (unsigned long long)EMPTY_KEY, (unsigned long long)k);
            if (old == EMPTY_KEY) { slots[s].idx = row_base + (int)i; placed = true; break; }
            if (old == k && flags) atomicOr(flags, 4);
            s = (s + 1) & mask;
        }
        if (!placed && flags) atomicOr(flags, 1);
    }
}

__device__ __forceinline__ Slot load_slot(const Slot* p) {
    const int4 v = *reinterpret_cast<const int4*>(p);
    Slot s;
    s.key = ((long long)(unsigned)v.y << 32) | (unsigned)v.x;
    s.idx = v.z; s.pad = 0;
    return s;
}

__global__ void __launch_bounds__(256) k_join_probe(const Slot* slots, uint64_t mask, const void* key, int dt, int64_t n, int how,
                                                    int* out_probe, int* out_build, int64_t cap, unsigned long long* out_count) {
    const int64_t nround = (n + 31) / 32 * 32;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nround; i += (int64_t)gridDim.x * blockDim.x) {
        const bool valid = i < n;
        long long k = 0;
        uint64_t s0 = 0;
        int matches = 0;
        if (valid) {
            k = load_i64(key, dt, i);
            s0 = mix64((uint64_t)k) & mask;
            if (k != EMPTY_KEY) {
                uint64_t s = s0;
                for (uint64_t tries = 0; tries <= mask; ++tries) {
                    const Slot sl = load_slot(&slots[s]);
                    if (sl.key == EMPTY_KEY) break;
                    if (sl.key == k) { matches++; if (how >= QK_JOIN_SEMI) break; }
                    s = (s + 1) & mask;
                }
            }
        }
        int emit;
        switch (how) {
            case QK_JOIN_INNER: emit = matches; break;
            case QK_JOIN_LEFT: emit = valid ? (matches > 0 ? matches : 1) : 0; break;
            case QK_JOIN_SEMI: emit = matches > 0 ? 1 : 0; break;
            default: emit = (valid && matches == 0) ? 1 : 0; break;
        }
        const int x = warp_inclusive_scan(emit);
        const int total = __shfl_sync(0xffffffffu, x, 31);
        if (total == 0) continue;
        unsigned long long base = 0;
        if (lane_id() == 31) base = atomicAdd(out_count, (unsigned long long)total);
        base = __shfl_sync(0xffffffffu, base, 31);
        int64_t pos = (int64_t)base + x - emit;
        if (emit == 0) continue;
        if (how == QK_JOIN_SEMI || how == QK_JOIN_ANTI || matches == 0) {
            if (pos < cap) { out_probe[pos] = (int)i; if (out_build) out_build[pos] = -1; }
            continue;
        }
        uint64_t s = s0;
        for (uint64_t tries = 0; tries <= mask; ++tries) {
            const Slot sl = load_slot(&slots[s]);
            if (sl.key == EMPTY_KEY) break;
            if (sl.key == k) {
                if (pos < cap) { out_probe[pos] = (int)i; out_build[pos] = sl.idx; }
                pos++;
            }
            s = (s + 1) & mask;
        }
    }
}

bool pow2(int64_t x) { return x > 0 && (x & (x - 1)) == 0; }

// ---- ordered probe / placement: rows are counted in chunks of ORDER_CHUNK, each chunk scanned by one CTA, then the chunk
// totals by one more (count_offsets twice), so the scan is as parallel as the count
constexpr int64_t ORDER_CHUNK = 4096;
constexpr int ORDER_INLINE = 16;      // a row with more matches is sorted by a CTA of its own

// matches of key k in the chain that starts at its home slot; semi / anti stop at the first
__device__ __forceinline__ int chain_matches(const Slot* slots, uint64_t mask, long long k, bool first_only) {
    int matches = 0;
    if (k == EMPTY_KEY) return 0;
    uint64_t s = mix64((uint64_t)k) & mask;
    for (uint64_t tries = 0; tries <= mask; ++tries) {
        const Slot sl = load_slot(&slots[s]);
        if (sl.key == EMPTY_KEY) break;
        if (sl.key == k) { ++matches; if (first_only) break; }
        s = (s + 1) & mask;
    }
    return matches;
}

__device__ __forceinline__ int emit_rows(int how, int matches) {
    switch (how) {
        case QK_JOIN_INNER: return matches;
        case QK_JOIN_LEFT: return matches > 0 ? matches : 1;
        case QK_JOIN_SEMI: return matches > 0 ? 1 : 0;
        default: return matches == 0 ? 1 : 0;
    }
}

__global__ void __launch_bounds__(256) k_join_count(const Slot* slots, uint64_t mask, const void* key, int dt, int64_t n,
                                                    int64_t npad, int how, uint32_t* counts, int* big, int* nbig) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < npad; i += (int64_t)gridDim.x * blockDim.x) {
        int emit = 0;
        if (i < n) {
            const int matches = chain_matches(slots, mask, load_i64(key, dt, i), how >= QK_JOIN_SEMI);
            emit = emit_rows(how, matches);
            if (matches > ORDER_INLINE) big[atomicAdd(nbig, 1)] = (int)i;
        }
        counts[i] = (uint32_t)emit;
    }
}

__device__ __forceinline__ int64_t out_offset(const int64_t* offsets, const int64_t* chunk_base, int64_t i) {
    return offsets[i] + chunk_base[i / ORDER_CHUNK];
}

__global__ void __launch_bounds__(256) k_join_write(const Slot* slots, uint64_t mask, const void* key, int dt, int64_t n, int how,
                                                    const uint32_t* counts, const int64_t* offsets, const int64_t* chunk_base,
                                                    int* out_probe, int* out_build, int64_t cap) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int emit = (int)counts[i];
        const int64_t pos = out_offset(offsets, chunk_base, i);
        if (emit == 0 || pos + emit > cap) continue;
        if (how >= QK_JOIN_SEMI) { out_probe[pos] = (int)i; continue; }
        const long long k = load_i64(key, dt, i);
        int m = 0;
        if (k != EMPTY_KEY) {
            uint64_t s = mix64((uint64_t)k) & mask;
            for (uint64_t tries = 0; tries <= mask && m < emit; ++tries) {
                const Slot sl = load_slot(&slots[s]);
                if (sl.key == EMPTY_KEY) break;
                if (sl.key == k) { out_probe[pos + m] = (int)i; out_build[pos + m] = sl.idx; m++; }
                s = (s + 1) & mask;
            }
        }
        if (m == 0) { out_probe[pos] = (int)i; out_build[pos] = -1; continue; }      // a left join's unmatched row
        if (m > ORDER_INLINE) continue;                                                // k_join_sort_big orders it
        int* b = out_build + pos;
        for (int a = 1; a < m; ++a) {                                                  // insertion sort, L1 hits
            const int v = b[a];
            int j = a - 1;
            while (j >= 0 && b[j] > v) { b[j + 1] = b[j]; --j; }
            b[j + 1] = v;
        }
    }
}

// One CTA per row with more than ORDER_INLINE matches: a bitonic network over its build-row numbers in place, in the form whose
// every comparator puts the smaller value at the lower index, so the elements past m act as +inf and are never touched.
__global__ void __launch_bounds__(512) k_join_sort_big(const uint32_t* counts, const int64_t* offsets, const int64_t* chunk_base,
                                                       const int* big, const int* nbig, int* out_build, int64_t cap) {
    const int nb = *nbig;
    for (int r = blockIdx.x; r < nb; r += gridDim.x) {
        const int64_t i = big[r];
        const int64_t m = counts[i], pos = out_offset(offsets, chunk_base, i);
        if (pos + m > cap) continue;
        int* b = out_build + pos;
        int64_t p2 = 1;
        while (p2 < m) p2 <<= 1;
        for (int64_t k = 2; k <= p2; k <<= 1) {
            for (int64_t j = k >> 1; j > 0; j >>= 1) {
                for (int64_t t = threadIdx.x; t < p2 / 2; t += blockDim.x) {
                    const int64_t lo = 2 * j * (t / j) + (t % j);
                    const int64_t hi = j == (k >> 1) ? (lo ^ (k - 1)) : lo + j;
                    if (hi < m) {
                        const int x = b[lo], y = b[hi];
                        if (x > y) { b[lo] = y; b[hi] = x; }
                    }
                }
                __syncthreads();
            }
        }
    }
}

__global__ void __launch_bounds__(256) k_place_count(const int* pos, int64_t nrecv, int64_t nleft, uint32_t* counts, int* first) {
    for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < nrecv; r += (int64_t)gridDim.x * blockDim.x) {
        const int p = pos[r];
        if (p < 0 || p >= nleft) continue;
        atomicAdd(&counts[p], 1u);
        if (r == 0 || pos[r - 1] != p) first[p] = (int)r;
    }
}

__global__ void __launch_bounds__(256) k_place_write(const int* pos, int64_t nrecv, int64_t nleft, const int64_t* offsets,
                                                     const int64_t* chunk_base, const int* first, int* out_src, int* out_left) {
    for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < nrecv; r += (int64_t)gridDim.x * blockDim.x) {
        const int p = pos[r];
        if (p < 0 || p >= nleft) continue;
        const int64_t d = out_offset(offsets, chunk_base, p) + r - first[p];
        out_src[d] = (int)r;
        if (out_left) out_left[d] = p;
    }
}

// The counts, their offsets and the chunk bases of the ordered probe and the placement (rows = probe rows / left positions),
// and the pieces only one of them takes: the rows sorted by a CTA (probe), each position's first received row (placement).
struct OrderedLayout {
    uint32_t* counts; int64_t* offsets; int64_t* chunk_tot; int64_t* chunk_base; int* big; int* nbig; int* first;
    int64_t npad, nchunks;
    OrderedLayout(Carve& c, int64_t rows, bool probe) {
        nchunks = rows > 0 ? (rows + ORDER_CHUNK - 1) / ORDER_CHUNK : 1;
        npad = nchunks * ORDER_CHUNK;
        counts = c.take<uint32_t>(npad);
        offsets = c.take<int64_t>(npad);
        chunk_tot = c.take<int64_t>(nchunks);
        chunk_base = c.take<int64_t>(nchunks + 1);
        big = probe ? c.take<int>(rows) : nullptr;
        nbig = probe ? c.take<int>(1) : nullptr;
        first = probe ? nullptr : c.take<int>(rows);
    }
};

// counts -> offsets within each chunk and each chunk's base; chunk_base[nchunks] = the total
int ordered_offsets(const OrderedLayout& w, cudaStream_t st) {
    if (int rc = count_offsets<uint32_t>(w.counts, w.nchunks, ORDER_CHUNK, w.offsets, w.chunk_tot, st)) return rc;
    return count_offsets<int64_t>(w.chunk_tot, 1, w.nchunks, w.chunk_base, w.chunk_base + w.nchunks, st);
}

}  // namespace
}  // namespace qk

using namespace qk;

extern "C" size_t qk_join_table_bytes(int64_t capacity) { return capacity > 0 ? (size_t)capacity * sizeof(Slot) : 0; }

extern "C" int qk_join_init(void* table, int64_t capacity, void* stream) {
    if (!table || !pow2(capacity)) QK_FAIL(QK_ERR_INVALID, "qk_join_init: table null or capacity %lld not a power of two", (long long)capacity);
    if (((uintptr_t)table & 15) != 0) QK_FAIL(QK_ERR_INVALID, "qk_join_init: table must be 16-byte aligned");
    k_join_init<<<grid_size(capacity, 16), 256, 0, (cudaStream_t)stream>>>((Slot*)table, capacity);
    QK_LAUNCH_CHECK("k_join_init");
    return QK_OK;
}

extern "C" int qk_join_build(void* table, int64_t capacity, const qk_column* key, int32_t row_base, int32_t* flags, void* stream) {
    const char* who = "qk_join_build";
    if (!table || !pow2(capacity)) QK_FAIL(QK_ERR_INVALID, "%s: bad table / capacity", who);
    if (int rc = check_col(key, who)) return rc;
    if (!dtype_is_int(key->dtype)) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: join keys must be integer columns", who);
    if (row_base < 0 || (int64_t)row_base + key->length > 0x7fffffffLL) QK_FAIL(QK_ERR_INVALID, "%s: build row numbers exceed int32", who);
    if (key->length == 0) return QK_OK;
    k_join_build<<<grid_size(key->length, 16), 256, 0, (cudaStream_t)stream>>>((Slot*)table, (uint64_t)capacity - 1, key->data, key->dtype, key->length, row_base, flags);
    QK_LAUNCH_CHECK("k_join_build");
    return QK_OK;
}

extern "C" int qk_join_probe(const void* table, int64_t capacity, const qk_column* key, int32_t how, int32_t* out_probe_idx,
                             int32_t* out_build_idx, int64_t out_capacity, int64_t* out_count, void* stream) {
    const char* who = "qk_join_probe";
    if (!table || !pow2(capacity)) QK_FAIL(QK_ERR_INVALID, "%s: bad table / capacity", who);
    if (int rc = check_col(key, who)) return rc;
    if (!dtype_is_int(key->dtype)) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: join keys must be integer columns", who);
    if (how < QK_JOIN_INNER || how > QK_JOIN_ANTI) QK_FAIL(QK_ERR_INVALID, "%s: bad join type %d", who, how);
    if (!out_count || out_capacity < 0 || (out_capacity > 0 && !out_probe_idx)) QK_FAIL(QK_ERR_INVALID, "%s: bad output arguments", who);
    if ((how == QK_JOIN_INNER || how == QK_JOIN_LEFT) && out_capacity > 0 && !out_build_idx) QK_FAIL(QK_ERR_INVALID, "%s: inner/left joins need out_build_idx", who);
    cudaStream_t st = (cudaStream_t)stream;
    QK_CUDA(cudaMemsetAsync(out_count, 0, sizeof(int64_t), st));
    if (key->length == 0) return QK_OK;
    k_join_probe<<<grid_size(key->length, 16), 256, 0, st>>>((const Slot*)table, (uint64_t)capacity - 1, key->data, key->dtype, key->length, how,
                                               out_probe_idx, out_build_idx, out_capacity, (unsigned long long*)out_count);
    QK_LAUNCH_CHECK("k_join_probe");
    return QK_OK;
}

extern "C" size_t qk_join_probe_ordered_workspace_bytes(int64_t nrows) {
    if (nrows < 0) return 0;
    Carve c(nullptr);
    OrderedLayout(c, nrows, true);
    return c.bytes;
}

extern "C" int qk_join_probe_ordered(const void* table, int64_t capacity, const qk_column* key, int32_t how, int32_t* out_probe_idx,
                                     int32_t* out_build_idx, int64_t out_capacity, int64_t* out_count, void* workspace,
                                     size_t ws_bytes, void* stream) {
    const char* who = "qk_join_probe_ordered";
    if (!table || !pow2(capacity)) QK_FAIL(QK_ERR_INVALID, "%s: bad table / capacity", who);
    if (int rc = check_col(key, who)) return rc;
    if (!dtype_is_int(key->dtype)) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: join keys must be integer columns", who);
    if (how < QK_JOIN_INNER || how > QK_JOIN_ANTI) QK_FAIL(QK_ERR_INVALID, "%s: bad join type %d", who, how);
    if (!out_count || out_capacity < 0 || (out_capacity > 0 && !out_probe_idx)) QK_FAIL(QK_ERR_INVALID, "%s: bad output arguments", who);
    if ((how == QK_JOIN_INNER || how == QK_JOIN_LEFT) && out_capacity > 0 && !out_build_idx) QK_FAIL(QK_ERR_INVALID, "%s: inner/left joins need out_build_idx", who);
    const int64_t n = key->length;
    if (ws_bytes < qk_join_probe_ordered_workspace_bytes(n) || (n > 0 && !workspace))
        QK_FAIL(QK_ERR_CAPACITY, "%s: workspace of %zu bytes, %zu needed", who, ws_bytes, qk_join_probe_ordered_workspace_bytes(n));
    cudaStream_t st = (cudaStream_t)stream;
    QK_CUDA(cudaMemsetAsync(out_count, 0, sizeof(int64_t), st));
    if (n == 0) return QK_OK;
    Carve c(workspace);
    const OrderedLayout w(c, n, true);
    const uint64_t mask = (uint64_t)capacity - 1;
    QK_CUDA(cudaMemsetAsync(w.nbig, 0, sizeof(int), st));
    k_join_count<<<grid_size(w.npad, 16), 256, 0, st>>>((const Slot*)table, mask, key->data, key->dtype, n, w.npad, how, w.counts, w.big, w.nbig);
    QK_LAUNCH_CHECK("k_join_count");
    if (int rc = ordered_offsets(w, st)) return rc;
    QK_CUDA(cudaMemcpyAsync(out_count, w.chunk_base + w.nchunks, sizeof(int64_t), cudaMemcpyDeviceToDevice, st));
    if (out_capacity == 0) return QK_OK;
    k_join_write<<<grid_size(n, 16), 256, 0, st>>>((const Slot*)table, mask, key->data, key->dtype, n, how, w.counts, w.offsets,
                                                   w.chunk_base, out_probe_idx, out_build_idx, out_capacity);
    QK_LAUNCH_CHECK("k_join_write");
    if (how <= QK_JOIN_LEFT) {
        k_join_sort_big<<<(unsigned)sm_count() * 2, 512, 0, st>>>(w.counts, w.offsets, w.chunk_base, w.big, w.nbig, out_build_idx, out_capacity);
        QK_LAUNCH_CHECK("k_join_sort_big");
    }
    return QK_OK;
}

extern "C" size_t qk_join_place_workspace_bytes(int64_t nleft) {
    if (nleft < 0) return 0;
    Carve c(nullptr);
    OrderedLayout(c, nleft, false);
    return c.bytes;
}

extern "C" int qk_join_place(const int32_t* pos, int64_t nrecv, int64_t nleft, int32_t* out_src, int32_t* out_left, void* workspace,
                             size_t ws_bytes, void* stream) {
    const char* who = "qk_join_place";
    if (nrecv < 0 || nrecv > 0x7fffffffLL || nleft < 0 || nleft > 0x7fffffffLL) QK_FAIL(QK_ERR_INVALID, "%s: row counts out of range", who);
    if (nrecv > 0 && (!pos || !out_src)) QK_FAIL(QK_ERR_INVALID, "%s: null positions or output", who);
    if (ws_bytes < qk_join_place_workspace_bytes(nleft) || (nleft > 0 && !workspace))
        QK_FAIL(QK_ERR_CAPACITY, "%s: workspace of %zu bytes, %zu needed", who, ws_bytes, qk_join_place_workspace_bytes(nleft));
    if (nrecv == 0 || nleft == 0) return QK_OK;
    cudaStream_t st = (cudaStream_t)stream;
    Carve c(workspace);
    const OrderedLayout w(c, nleft, false);
    QK_CUDA(cudaMemsetAsync(w.counts, 0, (size_t)w.npad * sizeof(uint32_t), st));
    k_place_count<<<grid_size(nrecv, 16), 256, 0, st>>>(pos, nrecv, nleft, w.counts, w.first);
    QK_LAUNCH_CHECK("k_place_count");
    if (int rc = ordered_offsets(w, st)) return rc;
    k_place_write<<<grid_size(nrecv, 16), 256, 0, st>>>(pos, nrecv, nleft, w.offsets, w.chunk_base, w.first, out_src, out_left);
    QK_LAUNCH_CHECK("k_place_write");
    return QK_OK;
}
