// quantile.cu -- mergeable quantile sketch for DataStream.approximate_quantile / approximate_median
// (pyquokka/datastream.py:905-1031, where a host t-digest plugin does it per channel and the channel answers are averaged).
//
// Every value is widened to fp64 and mapped to its order-preserving 64-bit image (NaN first made the canonical quiet NaN,
// so it sorts last).  The sketch keeps, per (column, bucket = image >> QK_QSKETCH_SHIFT): the row count and the smallest
// and largest image.  The state is a function of the multiset of values only, so batch splits, channels and ranks merge
// into bit-identical sketches.  It lives in an open-addressed device table of qk_qslot (key = column << 22 | bucket).
//
//   k_qsketch_update  persistent CTAs over tiles of QK_QSKETCH_TILE rows of one column.  A tile is read with 16-byte
//                     streaming loads (scalar loads for a masked, misaligned or short tile) while the previous one is
//                     processed; lanes that share a bucket are aggregated with __match_any_sync / __reduce_*_sync, and the
//                     group leader folds (count, min, max) into a CTA-private shared-memory table.  The tile's distinct
//                     buckets are then looked up in the global table; room for the absent ones is reserved in ctrl[0]
//                     before anything is written.  A tile that would push the load past 1/2 is deferred whole to a device
//                     list (ctrl[1] entries), so growth never counts a row twice: the host grows the table and re-runs
//                     exactly the deferred tiles.  Otherwise one atomicAdd / atomicMin / atomicMax per distinct bucket.
//   k_qsketch_merge   one thread per entry: inserts compacted (key, count, min, max) entries -- growth and the final merge.
#include "common.cuh"
#include <algorithm>
#include <vector>

namespace qk {
namespace {

constexpr int QT = QK_QSKETCH_TILE;     // rows per tile
constexpr int NT = 256;                 // threads per CTA
constexpr int PER = QT / NT;            // values per thread per tile
constexpr int SH = 2 * QT;              // shared-table slots: load <= 1/2 for any tile
constexpr unsigned SEMPTY = 0xFFFFFFFFu;
constexpr unsigned NOSLOT = 0xFFFFFFFFu;
constexpr unsigned long long GEMPTY = QK_QSKETCH_EMPTY;
constexpr int CTAS_PER_SM = 2;          // 108 KB of shared memory each
static_assert(PER == 8, "tile loads assume 8 values per thread");

struct QCol { const void* data; const uint8_t* valid; int32_t dtype; int32_t pad; };

struct UpdArgs {
    const QCol* cols;
    int64_t nrows;
    int64_t tiles_per_col;
    const int32_t* tiles;               // NULL: tile i is i
    int64_t ntiles;
    qk_qslot* table;
    unsigned long long mask;            // capacity - 1
    unsigned long long half;            // capacity / 2: the load limit
    unsigned long long* ctrl;
    int32_t* deferred;
};

struct Smem {
    unsigned key[SH];
    unsigned cnt[SH];
    unsigned long long mn[SH];
    unsigned long long mx[SH];
    unsigned short list[QT];            // claimed slots of the current tile
    unsigned gslot[QT];                 // their global slot, NOSLOT = absent at lookup
    int nlist, nabs, nnew, defer;
};

struct Raw { unsigned long long v[PER]; unsigned act; int dt; int col; int tile; };

__device__ __forceinline__ unsigned long long qimage(double d) {
    const unsigned long long b = d != d ? 0x7FF8000000000000ULL : (unsigned long long)__double_as_longlong(d);
    return (b >> 63) ? ~b : (b | 0x8000000000000000ULL);
}

__device__ __forceinline__ double widen(unsigned long long raw, int dt) {
    switch (dt) {
        case QK_F64: return __longlong_as_double((long long)raw);
        case QK_F32: return (double)__int_as_float((int)(unsigned)raw);
        case QK_I64: return (double)(long long)raw;
        case QK_I32: return (double)(int)(unsigned)raw;
        default: return (double)(unsigned)raw;
    }
}

__device__ __forceinline__ int esize(int dt) { return dt == QK_F64 || dt == QK_I64 ? 8 : dt == QK_U8 ? 1 : 4; }

__device__ __forceinline__ unsigned long long ld_relaxed(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}

__device__ __forceinline__ unsigned shash(unsigned key) { return (key * 0x9E3779B1u) >> (32 - 12); }
static_assert(SH == 1 << 12, "shash yields 12 bits");

__device__ __forceinline__ void load_tile(Raw& r, const UpdArgs& a, int64_t i) {
    const int t = a.tiles ? a.tiles[i] : (int)i;
    const int c = (int)(t / a.tiles_per_col);
    const int64_t r0 = (t - (int64_t)c * a.tiles_per_col) * QT;
    const int64_t n = a.nrows - r0 < QT ? a.nrows - r0 : QT;
    const QCol col = a.cols[c];
    r.tile = t; r.col = c; r.dt = col.dtype;
    const int es = esize(col.dtype);
    const char* base = (const char*)col.data + r0 * es;
    const unsigned tid = threadIdx.x;
    if (n == QT && col.valid == nullptr && es >= 4 && ((uintptr_t)base & 15) == 0) {
        const uint4* q = (const uint4*)base;
        if (es == 8) {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const uint4 w = __ldcs(q + j * NT + tid);
                r.v[2 * j] = w.x | ((unsigned long long)w.y << 32);
                r.v[2 * j + 1] = w.z | ((unsigned long long)w.w << 32);
            }
        } else {
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                const uint4 w = __ldcs(q + j * NT + tid);
                r.v[4 * j] = w.x; r.v[4 * j + 1] = w.y; r.v[4 * j + 2] = w.z; r.v[4 * j + 3] = w.w;
            }
        }
        r.act = 0xFFu;
        return;
    }
    r.act = 0;
#pragma unroll
    for (int j = 0; j < PER; ++j) {
        const int64_t e = r0 + j * NT + tid;
        r.v[j] = 0;
        if (e < r0 + n && (col.valid == nullptr || __ldcs(col.valid + e))) {
            r.act |= 1u << j;
            switch (es) {
                case 8: r.v[j] = (unsigned long long)__ldcs((const long long*)col.data + e); break;
                case 4: r.v[j] = (unsigned)__ldcs((const int*)col.data + e); break;
                default: r.v[j] = ((const uint8_t*)col.data)[e]; break;
            }
        }
    }
}

// one value per lane into the shared table: lanes of a bucket are folded first, their leader inserts
__device__ __forceinline__ void add_value(Smem& s, bool act, unsigned long long img) {
    const unsigned key = act ? (unsigned)(img >> QK_QSKETCH_SHIFT) : SEMPTY;
    const unsigned g = __match_any_sync(0xFFFFFFFFu, key);
    const unsigned hi = (unsigned)(img >> 32), lo = (unsigned)img;
    const unsigned mnhi = __reduce_min_sync(g, hi);
    const unsigned mnlo = __reduce_min_sync(g, hi == mnhi ? lo : 0xFFFFFFFFu);
    const unsigned mxhi = __reduce_max_sync(g, hi);
    const unsigned mxlo = __reduce_max_sync(g, hi == mxhi ? lo : 0u);
    if (key == SEMPTY || lane_id() != (unsigned)(__ffs(g) - 1)) return;
    unsigned h = shash(key);
    while (true) {
        const unsigned cur = *(volatile unsigned*)&s.key[h];
        if (cur == key) break;
        if (cur == SEMPTY) {
            const unsigned old = atomicCAS(&s.key[h], SEMPTY, key);
            if (old == SEMPTY) { s.list[atomicAdd(&s.nlist, 1)] = (unsigned short)h; break; }
            if (old == key) break;
        }
        h = (h + 1) & (SH - 1);
    }
    atomicAdd(&s.cnt[h], (unsigned)__popc(g));
    // 64-bit shared min / max are compare-and-swap loops: skip them unless they would change the slot (bounds only move
    // one way, so a stale read costs at most one needless atomic)
    const unsigned long long mn = ((unsigned long long)mnhi << 32) | mnlo, mx = ((unsigned long long)mxhi << 32) | mxlo;
    if (mn < *(volatile unsigned long long*)&s.mn[h]) atomicMin(&s.mn[h], mn);
    if (mx > *(volatile unsigned long long*)&s.mx[h]) atomicMax(&s.mx[h], mx);
}

// slot of `key` in the global table, claiming an empty one; NOSLOT when the probe runs through the whole table (the
// caller broke the load limit: flagged in ctrl[2])
__device__ __forceinline__ unsigned long long ginsert(qk_qslot* table, unsigned long long mask, unsigned long long key, bool& claimed,
                                                      unsigned long long* ctrl) {
    unsigned long long h = mix64(key) & mask;
    claimed = false;
    for (unsigned long long step = 0; step <= mask; ++step) {
        const unsigned long long cur = ld_relaxed((const unsigned long long*)&table[h].key);
        if (cur == key) return h;
        if (cur == GEMPTY) {
            const unsigned long long old = atomicCAS((unsigned long long*)&table[h].key, GEMPTY, key);
            if (old == GEMPTY) { claimed = true; return h; }
            if (old == key) return h;
        }
        h = (h + 1) & mask;
    }
    atomicExch(&ctrl[2], 1ull);
    return ~0ull;
}

__device__ __forceinline__ void gfold(qk_qslot* sl, unsigned long long cnt, unsigned long long mn, unsigned long long mx) {
    atomicAdd((unsigned long long*)&sl->count, cnt);
    atomicMin((unsigned long long*)&sl->min_image, mn);
    atomicMax((unsigned long long*)&sl->max_image, mx);
}

__device__ void flush_tile(Smem& s, const UpdArgs& a, int col, int tile) {
    const unsigned tid = threadIdx.x;
    const int nd = s.nlist;
    const unsigned long long colkey = (unsigned long long)col << 22;
    // 1. which of the tile's buckets the global table lacks
    int nabs = 0;
    for (int i = tid; i < nd; i += NT) {
        const unsigned long long key = colkey | s.key[s.list[i]];
        unsigned long long h = mix64(key) & a.mask;
        unsigned found = NOSLOT;
        for (unsigned long long step = 0; step <= a.mask; ++step) {
            const unsigned long long cur = ld_relaxed((const unsigned long long*)&a.table[h].key);
            if (cur == key) { found = (unsigned)h; break; }
            if (cur == GEMPTY) break;
            h = (h + 1) & a.mask;
        }
        s.gslot[i] = found;
        nabs += found == NOSLOT;
    }
    if (nabs) atomicAdd(&s.nabs, nabs);
    __syncthreads();
    // 2. reserve room for them, or defer the whole tile
    if (tid == 0) {
        const unsigned long long want = (unsigned long long)s.nabs;
        s.defer = 0;
        if (want) {
            const unsigned long long old = atomicAdd(a.ctrl, want);
            if (old + want > a.half) {
                atomicAdd(a.ctrl, (unsigned long long)(-(long long)want));
                a.deferred[atomicAdd(&a.ctrl[1], 1ull)] = tile;
                s.defer = 1;
            }
        }
    }
    __syncthreads();
    // 3. one atomic per field per distinct bucket; reset the shared slots either way
    const bool defer = s.defer;
    int nnew = 0;
    for (int i = tid; i < nd; i += NT) {
        const unsigned sl = s.list[i];
        if (!defer) {
            unsigned long long h = s.gslot[i];
            if (h == NOSLOT) {
                bool claimed;
                h = ginsert(a.table, a.mask, colkey | s.key[sl], claimed, a.ctrl);
                nnew += claimed;
            }
            if (h != ~0ull) gfold(&a.table[h], s.cnt[sl], s.mn[sl], s.mx[sl]);
        }
        s.key[sl] = SEMPTY; s.cnt[sl] = 0; s.mn[sl] = ~0ull; s.mx[sl] = 0;
    }
    if (nnew) atomicAdd(&s.nnew, nnew);
    __syncthreads();
    if (tid == 0) {
        if (!defer && s.nabs > s.nnew)            // buckets another tile claimed first: give their reservation back
            atomicAdd(a.ctrl, (unsigned long long)(-(long long)(s.nabs - s.nnew)));
        s.nlist = 0; s.nabs = 0; s.nnew = 0;
    }
    __syncthreads();
}

__global__ void __launch_bounds__(NT, CTAS_PER_SM) k_qsketch_update(UpdArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    Smem& s = *reinterpret_cast<Smem*>(smem_raw);
    for (int i = threadIdx.x; i < SH; i += NT) { s.key[i] = SEMPTY; s.cnt[i] = 0; s.mn[i] = ~0ull; s.mx[i] = 0; }
    if (threadIdx.x == 0) { s.nlist = 0; s.nabs = 0; s.nnew = 0; s.defer = 0; }
    __syncthreads();
    int64_t i = blockIdx.x;
    if (i >= a.ntiles) return;
    Raw cur, nxt;
    load_tile(cur, a, i);
    for (; i < a.ntiles; i += gridDim.x) {
        if (i + gridDim.x < a.ntiles) load_tile(nxt, a, i + gridDim.x);       // in flight while this tile is folded
#pragma unroll
        for (int j = 0; j < PER; ++j) add_value(s, (cur.act >> j) & 1u, qimage(widen(cur.v[j], cur.dt)));
        __syncthreads();
        flush_tile(s, a, cur.col, cur.tile);
        cur = nxt;
    }
}

__global__ void __launch_bounds__(256) k_qsketch_merge(const unsigned long long* keys, const unsigned long long* counts,
                                                       const unsigned long long* mins, const unsigned long long* maxs, int64_t n,
                                                       qk_qslot* table, unsigned long long mask, unsigned long long* ctrl) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    bool claimed = false;
    if (i < n && keys[i] != GEMPTY) {
        const unsigned long long h = ginsert(table, mask, keys[i], claimed, ctrl);
        if (h != ~0ull) gfold(&table[h], counts[i], mins[i], maxs[i]);
    }
    const unsigned b = __ballot_sync(0xFFFFFFFFu, claimed);
    if (lane_id() == 0 && b) atomicAdd(ctrl, (unsigned long long)__popc(b));
}

int check_capacity(int64_t capacity, const char* who) {
    if (capacity < QK_QSKETCH_MIN_CAPACITY || capacity > (1LL << 31) || (capacity & (capacity - 1)))
        QK_FAIL(QK_ERR_INVALID, "%s: capacity %lld must be a power of two in [%d, 2^31]", who, (long long)capacity,
                QK_QSKETCH_MIN_CAPACITY);
    return 0;
}

}  // namespace
}  // namespace qk

using namespace qk;

extern "C" size_t qk_qsketch_workspace_bytes(int32_t k) {
    return k < 1 ? 0 : align_up((size_t)k * sizeof(QCol), 256);
}

extern "C" int qk_qsketch_update(const qk_column* cols, const uint8_t* const* valid, int32_t k, int64_t nrows, qk_qslot* table,
                                 int64_t capacity, uint64_t* ctrl, const int32_t* tiles, int64_t ntiles, int32_t* deferred,
                                 void* workspace, size_t ws_bytes, void* stream) {
    const char* who = "qk_qsketch_update";
    if (k < 1) QK_FAIL(QK_ERR_INVALID, "%s: k must be >= 1", who);
    if (!cols) QK_FAIL(QK_ERR_INVALID, "%s: null column table", who);
    if (nrows < 0) QK_FAIL(QK_ERR_INVALID, "%s: negative nrows", who);
    for (int32_t i = 0; i < k; ++i) {
        if (int rc = check_col(&cols[i], who)) return rc;
        if (cols[i].length != nrows) QK_FAIL(QK_ERR_INVALID, "%s: column %d has %lld rows, expected %lld", who, i,
                                             (long long)cols[i].length, (long long)nrows);
    }
    if (int rc = check_capacity(capacity, who)) return rc;
    if (!table || !ctrl) QK_FAIL(QK_ERR_INVALID, "%s: null table or control words", who);
    const int64_t tpc = (nrows + QT - 1) / QT;
    if (tpc * k > 0x7fffffffLL) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: %lld tiles in one call (at most 2^31 - 1)", who, (long long)(tpc * k));
    if (tiles ? (ntiles < 0 || ntiles > tpc * k) : ntiles != tpc * k)
        QK_FAIL(QK_ERR_INVALID, "%s: ntiles %lld does not match the tile list (%lld tiles of %d rows x %d columns)", who,
                (long long)ntiles, (long long)(tpc * k), QT, k);
    if (ntiles > 0 && !deferred) QK_FAIL(QK_ERR_INVALID, "%s: null deferred-tile list", who);
    if (!workspace || ws_bytes < qk_qsketch_workspace_bytes(k))
        QK_FAIL(QK_ERR_CAPACITY, "%s: workspace too small (%zu < %zu)", who, ws_bytes, qk_qsketch_workspace_bytes(k));
    cudaStream_t st = (cudaStream_t)stream;
    QK_CUDA(cudaMemsetAsync(ctrl + 1, 0, sizeof(uint64_t), st));
    if (ntiles == 0) return QK_OK;
    std::vector<QCol> host((size_t)k);
    for (int32_t i = 0; i < k; ++i) host[i] = QCol{cols[i].data, valid ? valid[i] : nullptr, cols[i].dtype, 0};
    QK_CUDA(cudaMemcpyAsync(workspace, host.data(), (size_t)k * sizeof(QCol), cudaMemcpyHostToDevice, st));
    UpdArgs a;
    a.cols = (const QCol*)workspace;
    a.nrows = nrows; a.tiles_per_col = tpc; a.tiles = tiles; a.ntiles = ntiles;
    a.table = table; a.mask = (unsigned long long)capacity - 1; a.half = (unsigned long long)capacity / 2;
    a.ctrl = (unsigned long long*)ctrl; a.deferred = deferred;
    const size_t smem = sizeof(Smem);
    QK_CUDA(cudaFuncSetAttribute(k_qsketch_update, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int64_t grid = std::min<int64_t>(ntiles, (int64_t)CTAS_PER_SM * sm_count());
    k_qsketch_update<<<(unsigned)grid, NT, smem, st>>>(a);
    QK_LAUNCH_CHECK("k_qsketch_update");
    return QK_OK;
}

extern "C" int qk_qsketch_merge(const uint64_t* keys, const uint64_t* counts, const uint64_t* mins, const uint64_t* maxs, int64_t n,
                                qk_qslot* table, int64_t capacity, uint64_t* ctrl, void* stream) {
    const char* who = "qk_qsketch_merge";
    if (n < 0) QK_FAIL(QK_ERR_INVALID, "%s: negative entry count", who);
    if (n > 0 && (!keys || !counts || !mins || !maxs)) QK_FAIL(QK_ERR_INVALID, "%s: null entry arrays", who);
    if (int rc = check_capacity(capacity, who)) return rc;
    if (!table || !ctrl) QK_FAIL(QK_ERR_INVALID, "%s: null table or control words", who);
    if (n > capacity / 2) QK_FAIL(QK_ERR_CAPACITY, "%s: %lld entries exceed half the capacity %lld", who, (long long)n,
                                  (long long)capacity);
    if (n == 0) return QK_OK;
    k_qsketch_merge<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        (const unsigned long long*)keys, (const unsigned long long*)counts, (const unsigned long long*)mins,
        (const unsigned long long*)maxs, n, table, (unsigned long long)capacity - 1, (unsigned long long*)ctrl);
    QK_LAUNCH_CHECK("k_qsketch_merge");
    return QK_OK;
}
