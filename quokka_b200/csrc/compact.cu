// compact.cu -- fast path of K1 for the shape every pushed-down TPC-H scan has:
//     predicate = one integer / date / dictionary-code column against a constant (any of < <= > >= = !=),
//     projection = verbatim columns (keys, measures, dates, codes).
// i.e. "filter by a range on one column and compact k columns" -- no expression evaluation at all.
//
// Two passes, no atomics, STABLE output (input row order is kept, so sorted streams stay sorted):
//   pass 1  k_compact_count: every CTA counts the survivors of its contiguous chunk of rows (reads the
//           predicate column only) -> k_compact_scan turns the counts into output offsets;
//   pass 2  k_filter_compact_tma: column tiles of the chunk are staged into shared memory by the TMA
//           engine (cp.async.bulk + mbarrier complete_tx, 3-stage ring, one elected producer thread); the
//           CTA evaluates the predicate from shared memory, ranks the survivors of a tile with warp ballots
//           + one small warp scan and writes them, column by column, at its running output offset.
//
// HBM-bound: reads (2 x pred + payload) bytes/row, writes payload bytes per surviving row.
// Q3 lineitem scan at SF-100: 600 M x (28 + 4) B read + 324 M x 24 B written = 27.0 GB algorithmic.
#include <stdlib.h>
#include "common.cuh"
#include "tma.cuh"

namespace qk {
namespace {

constexpr int C_NT = 256;
constexpr int C_STAGES = 3;
constexpr int C_MAXCOLS = 8;

struct CompactArgs {
    const unsigned char* src[C_MAXCOLS];   // payload columns
    unsigned char* dst[C_MAXCOLS];
    int32_t width[C_MAXCOLS];
    int32_t off[C_MAXCOLS];                // byte offset of the column's tile inside a stage
    int32_t ncols;
    const unsigned char* pred_col;         // nullptr = no predicate
    int32_t pred_width, pred_off;
    int32_t pred_neg;
    long long pred_lo, pred_hi;
    int32_t tile_rows, stage_bytes;
    // optional semi-join reduction: survivors must also hit the Bloom filter of the partition their key goes to
    const unsigned* bloom;                 // nullptr = off; nparts filters of bloom_words 32-bit words each
    long long bloom_words;
    int32_t bloom_nparts, bloom_col;       // bloom_col = payload column holding the (int64 / int32) join key
};

// Blocked Bloom filter: one 32-byte block (a DRAM sector) per key, 3 bits inside it.
// Blocked Bloom filter, one 64-bit word per key: the key picks a 32-byte block (a DRAM sector) of its partition's filter, one of
// the block's four 64-bit words and three bits inside that word, so a test is ONE 8-byte load + one mask compare.  The hash is
// two rounds of 32-bit multiply-xorshift (the mask kernel is instruction-bound: a 64-bit mix + three 4-byte probes cost
// ~170 instructions per row).
__device__ __forceinline__ void bloom_slots(long long key, long long words_per_part, int nparts, long long* word64, unsigned long long* mask) {
    const unsigned p = part_mod(key, (unsigned)nparts);
    unsigned h = ((unsigned)key ^ ((unsigned)((unsigned long long)key >> 32) * 0x9E3779B1u)) * 0x85EBCA6Bu;
    h ^= h >> 15; h *= 0xC2B2AE35u; h ^= h >> 16;
    const unsigned block = __umulhi(h, (unsigned)(words_per_part >> 3));              // < words_per_part / 8 blocks of 32 bytes
    const unsigned h2 = h * 0x9E3779B1u;
    *word64 = (((long long)p * words_per_part) >> 1) + ((long long)block << 2) + (h2 >> 30);
    *mask = (1ull << ((h2 >> 24) & 63u)) | (1ull << ((h2 >> 18) & 63u)) | (1ull << ((h2 >> 12) & 63u));
}
__device__ __forceinline__ unsigned long long ld_u64_hint(const void* p, unsigned long long pol) {
    unsigned long long v; asm volatile("ld.global.nc.L2::cache_hint.u64 %0, [%1], %2;" : "=l"(v) : "l"(p), "l"(pol)); return v;
}
__global__ void __launch_bounds__(256) k_bloom_build(const void* key, int dt, int64_t n, unsigned* bits, long long words_per_part, int nparts) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        long long w; unsigned long long m;
        bloom_slots(load_i64(key, dt, i), words_per_part, nparts, &w, &m);
        atomicOr((unsigned long long*)bits + w, m);
    }
}

__device__ __forceinline__ void issue_tile(const CompactArgs& A, int64_t tile, unsigned char* stage, unsigned bar) {
    const int64_t base = tile * A.tile_rows;
    mbar_expect_tx(bar, (unsigned)A.stage_bytes);
    for (int c = 0; c < A.ncols; ++c)
        bulk_g2s(smem_u32(stage + A.off[c]), A.src[c] + base * A.width[c], (unsigned)(A.tile_rows * A.width[c]), bar);
}

__device__ __forceinline__ bool eval_pred(const CompactArgs& A, const unsigned char* p, int64_t i) {
    if (!A.pred_col) return true;
    long long x;
    switch (A.pred_width) {
        case 1: x = p[i]; break;
        case 4: x = ((const int*)p)[i]; break;
        default: x = ((const long long*)p)[i]; break;
    }
    return ((x >= A.pred_lo) & (x <= A.pred_hi)) != (A.pred_neg != 0);
}
// the same test on a column that is streamed once from global memory (pass 1): bypass L1, first to leave L2
__device__ __forceinline__ bool eval_pred_stream(const CompactArgs& A, int64_t i, unsigned long long pol) {
    if (!A.pred_col) return true;
    long long x;
    switch (A.pred_width) {
        case 1: x = ld_u8_stream(A.pred_col + i, pol); break;
        case 4: x = ld_i32_stream(A.pred_col + 4 * i, pol); break;
        default: x = ld_i64_stream(A.pred_col + 8 * i, pol); break;
    }
    return ((x >= A.pred_lo) & (x <= A.pred_hi)) != (A.pred_neg != 0);
}

__device__ __forceinline__ void copy_row(const CompactArgs& A, const unsigned char* const* src, int64_t from, int64_t to) {
    for (int c = 0; c < A.ncols; ++c) {
        switch (A.width[c]) {
            case 1: A.dst[c][to] = src[c][from]; break;
            case 4: ((unsigned*)A.dst[c])[to] = ((const unsigned*)src[c])[from]; break;
            default: ((unsigned long long*)A.dst[c])[to] = ((const unsigned long long*)src[c])[from]; break;
        }
    }
}

constexpr int C_MAXSLABS = 16;             // tile_rows / C_NT

// pass 1: evaluate predicate (+ Bloom test) once per row; write one bit per row and the survivor count of every chunk
// (chunk b = rows [b * chunk_rows, (b + 1) * chunk_rows), chunk_rows a multiple of 256).  Every lane owns 8 CONSECUTIVE rows:
// the predicate and key columns arrive as 128-bit loads (6 load instructions for 8 rows of a date32 + int64 pair), the 8 Bloom
// words are requested together, and 4 lanes assemble one bitmap word with two shuffles.  PW / KW = byte width of the predicate /
// Bloom key column (0 = absent).
constexpr int M_NT = 512;
constexpr int M_R = 8;
template <int W> struct Row8 { long long v[8]; };
template <int W> __device__ __forceinline__ void load8(const unsigned char* col, int64_t row0, long long* v, unsigned long long pol) {
    if constexpr (W == 8) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            long long a, b;
            asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.s64 {%0,%1}, [%2], %3;" : "=l"(a), "=l"(b) : "l"(col + 8 * row0 + 16 * q), "l"(pol));
            v[2 * q] = a; v[2 * q + 1] = b;
        }
    } else if constexpr (W == 4) {
#pragma unroll
        for (int q = 0; q < 2; ++q) {
            int a, b, c, d;
            asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.s32 {%0,%1,%2,%3}, [%4], %5;" : "=r"(a), "=r"(b), "=r"(c), "=r"(d) : "l"(col + 4 * row0 + 16 * q), "l"(pol));
            v[4 * q] = a; v[4 * q + 1] = b; v[4 * q + 2] = c; v[4 * q + 3] = d;
        }
    } else if constexpr (W == 1) {
        unsigned long long x;
        asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.u64 %0, [%1], %2;" : "=l"(x) : "l"(col + row0), "l"(pol));
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = (long long)((x >> (8 * j)) & 0xffull);
    }
}
template <int PW, int KW>
__global__ void __launch_bounds__(M_NT, 2) k_compact_mask(const __grid_constant__ CompactArgs A, int64_t nrows, int64_t chunk_rows,
                                                          unsigned* bitmap, long long* counts) {
    __shared__ int wsum[M_NT / 32];
    const int warp = threadIdx.x >> 5, lane = lane_id();
    const int64_t lo = blockIdx.x * chunk_rows;
    const int64_t hi = lo + chunk_rows < nrows ? lo + chunk_rows : nrows;
    const unsigned char* keycol = KW ? A.src[A.bloom_col] : nullptr;
    const unsigned long long stream_pol = l2_policy_evict_first(), keep_pol = l2_policy_evict_last();
    int cnt = 0;
    for (int64_t base = lo + warp * (32 * M_R); base < hi; base += (M_NT / 32) * (32 * M_R)) {
        const int64_t row0 = base + lane * M_R;
        long long x[M_R], k[M_R];
        unsigned m = 0;                                           // bit j = row row0 + j survives
        if (base + 32 * M_R <= hi) {                              // whole group inside the chunk: vector loads
            if constexpr (PW != 0) load8<PW>(A.pred_col, row0, x, stream_pol);
            if constexpr (KW != 0) load8<KW>(keycol, row0, k, stream_pol);
#pragma unroll
            for (int j = 0; j < M_R; ++j) {
                bool pass = true;
                if constexpr (PW != 0) pass = ((x[j] >= A.pred_lo) & (x[j] <= A.pred_hi)) != (A.pred_neg != 0);
                m |= (pass ? 1u : 0u) << j;
            }
        } else {                                                  // ragged end of the chunk
#pragma unroll
            for (int j = 0; j < M_R; ++j) {
                const int64_t row = row0 + j;
                bool pass = row < hi;
                k[j] = 0;
                if (pass) {
                    if constexpr (PW != 0) {
                        const long long xv = PW == 1 ? (long long)A.pred_col[row] : PW == 4 ? (long long)((const int*)A.pred_col)[row] : ((const long long*)A.pred_col)[row];
                        pass = ((xv >= A.pred_lo) & (xv <= A.pred_hi)) != (A.pred_neg != 0);
                    }
                    if constexpr (KW != 0) k[j] = KW == 8 ? ((const long long*)keycol)[row] : (long long)((const int*)keycol)[row];
                }
                m |= (pass ? 1u : 0u) << j;
            }
        }
        if constexpr (KW != 0) {
            unsigned long long word[M_R], want[M_R];
#pragma unroll
            for (int j = 0; j < M_R; ++j) {
                long long w;
                bloom_slots(k[j], A.bloom_words, A.bloom_nparts, &w, &want[j]);
                word[j] = ((m >> j) & 1u) ? ld_u64_hint((const unsigned long long*)A.bloom + w, keep_pol) : 0ull;     // the filter stays in L2
            }
#pragma unroll
            for (int j = 0; j < M_R; ++j) if ((word[j] & want[j]) != want[j]) m &= ~(1u << j);
        }
        cnt += __popc(m);
        // rows row0 .. row0 + 7 are byte (lane & 3) of bitmap word (base >> 5) + (lane >> 2)
        unsigned v = m << (8 * (lane & 3));
        v |= __shfl_xor_sync(0xffffffffu, v, 1);
        v |= __shfl_xor_sync(0xffffffffu, v, 2);
        if ((lane & 3) == 0 && base + (int64_t)(lane >> 2) * 32 < hi) bitmap[(base >> 5) + (lane >> 2)] = v;
    }
    for (int o = 16; o; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    if (lane == 0) wsum[warp] = cnt;
    __syncthreads();
    if (threadIdx.x == 0) {
        long long t = 0;
        for (int w = 0; w < M_NT / 32; ++w) t += wsum[w];
        counts[blockIdx.x] = t;
    }
}
// exclusive scan of up to 1024 chunk counts; offsets[n] = total, also stored to *out_rows
__global__ void __launch_bounds__(1024) k_compact_scan(const long long* counts, int n, long long* offsets, long long* out_rows) {
    __shared__ long long wtot[32];
    const int i = threadIdx.x;
    long long v = i < n ? counts[i] : 0, x = v;
    for (int o = 1; o < 32; o <<= 1) {
        const long long y = __shfl_up_sync(0xffffffffu, x, o);
        if ((int)lane_id() >= o) x += y;
    }
    if (lane_id() == 31) wtot[i >> 5] = x;
    __syncthreads();
    if (i < 32) {
        long long w = wtot[i], t = w;
        for (int o = 1; o < 32; o <<= 1) {
            const long long y = __shfl_up_sync(0xffffffffu, t, o);
            if ((int)lane_id() >= o) t += y;
        }
        wtot[i] = t - w;
    }
    __syncthreads();
    const long long excl = wtot[i >> 5] + x - v;
    if (i < n) offsets[i] = excl;
    if (i == n - 1) { offsets[n] = excl + v; *out_rows = excl + v; }
}

template <typename T>
__device__ __forceinline__ void copy_col(const unsigned char* src, unsigned char* dst, int slabs, unsigned my, const int* wcount,
                                         long long base, int warp, int lane) {
    for (int r = 0; r < slabs; ++r) {
        const bool pass = (my >> r) & 1u;
        const unsigned bal = __ballot_sync(0xffffffffu, pass);
        if (pass) {
            const long long pos = base + wcount[r * (C_NT / 32) + warp] + __popc(bal & ((1u << lane) - 1u));
            ((T*)dst)[pos] = ((const T*)src)[r * C_NT + threadIdx.x];
        }
    }
}

// pass 2
__global__ void __launch_bounds__(C_NT, 3) k_filter_compact_tma(const __grid_constant__ CompactArgs A, int64_t nrows, int64_t chunk_rows,
                                                                const long long* offsets, const unsigned* __restrict__ bitmap) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    __shared__ __align__(8) unsigned long long bars[C_STAGES];
    __shared__ int wcount[C_MAXSLABS * (C_NT / 32) + 1];   // survivors per (slab, warp) -> exclusive prefix; [n] = tile total
    const int slabs = A.tile_rows / C_NT;
    const int nw = slabs * (C_NT / 32);
    const int warp = threadIdx.x >> 5, lane = lane_id();
    const int64_t lo = blockIdx.x * chunk_rows;
    const int64_t hi = lo + chunk_rows < nrows ? lo + chunk_rows : nrows;
    const int64_t my_n = hi > lo ? (hi - lo) / A.tile_rows : 0;          // full tiles of my chunk
    const int64_t tile0 = lo / A.tile_rows;                                // chunk_rows is a multiple of tile_rows
    // Sparse chunk (fewer than 1 row in 8 survives, e.g. after the Bloom filter): do not stage whole tiles;
    // walk the bitmap and fetch only the surviving rows from global memory (one 32-byte sector per row
    // and column instead of the full column width for all rows).  Same output order.
    if (hi > lo && (offsets[blockIdx.x + 1] - offsets[blockIdx.x]) * 8 < (hi - lo)) {
        __shared__ int wtot[C_NT / 32];
        long long run = offsets[blockIdx.x];
        const int64_t w_lo = lo >> 5, w_hi = (hi + 31) >> 5;
        int* list = (int*)smem_raw;                              // the tile ring is idle on this path: survivor row numbers
        const bool listed = (size_t)C_STAGES * A.stage_bytes >= (size_t)C_NT * 32 * sizeof(int);
        for (int64_t wb = w_lo; wb < w_hi; wb += C_NT) {        // 256 bitmap words = 8192 rows per step
            const int64_t wi = wb + threadIdx.x;
            unsigned m = wi < w_hi ? __ldg(&bitmap[wi]) : 0u;
            // exclusive scan of popc over the 256 threads
            int v = __popc(m), x = v;
            for (int o = 1; o < 32; o <<= 1) {
                const int y = __shfl_up_sync(0xffffffffu, x, o);
                if (lane >= o) x += y;
            }
            if (lane == 31) wtot[warp] = x;
            __syncthreads();
            int before = 0, total = 0;
            for (int w = 0; w < C_NT / 32; ++w) { if (w < warp) before += wtot[w]; total += wtot[w]; }
            if (listed) {
                // 1. every thread lists its survivors' row numbers (relative to the step) in output order
                int slot = before + x - v;
                while (m) {
                    const int j = __ffs(m) - 1;
                    list[slot++] = (int)(threadIdx.x * 32 + j);
                    m &= m - 1;
                }
                __syncthreads();
                // 2. one survivor per thread and round: the loads of all columns and of all threads are independent, so
                //    the gather runs at memory-level parallelism instead of one row at a time per thread
                const int64_t row0 = wb << 5;
                for (int e = threadIdx.x; e < total; e += C_NT) {
                    const int64_t from = row0 + list[e];
                    const long long to = run + e;
                    unsigned long long val[C_MAXCOLS];
#pragma unroll
                    for (int c = 0; c < C_MAXCOLS; ++c) {
                        if (c < A.ncols) {
                            switch (A.width[c]) {
                                case 1: val[c] = A.src[c][from]; break;
                                case 4: val[c] = ((const unsigned*)A.src[c])[from]; break;
                                default: val[c] = ((const unsigned long long*)A.src[c])[from]; break;
                            }
                        }
                    }
#pragma unroll
                    for (int c = 0; c < C_MAXCOLS; ++c) {
                        if (c < A.ncols) {
                            switch (A.width[c]) {
                                case 1: A.dst[c][to] = (unsigned char)val[c]; break;
                                case 4: ((unsigned*)A.dst[c])[to] = (unsigned)val[c]; break;
                                default: ((unsigned long long*)A.dst[c])[to] = val[c]; break;
                            }
                        }
                    }
                }
            } else {
                long long pos = run + before + x - v;
                while (m) {
                    const int j = __ffs(m) - 1;
                    copy_row(A, A.src, (wi << 5) + j, pos++);
                    m &= m - 1;
                }
            }
            run += total;
            __syncthreads();
        }
        return;
    }
    if (threadIdx.x == 0) {
        for (int s = 0; s < C_STAGES; ++s) mbar_init(smem_u32(&bars[s]), 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (threadIdx.x == 0)
        for (int s = 0; s < C_STAGES && s < my_n; ++s)
            issue_tile(A, tile0 + s, smem_raw + (size_t)s * A.stage_bytes, smem_u32(&bars[s]));
    long long running = hi > lo ? offsets[blockIdx.x] : 0;
    int s = 0;
    unsigned parity = 0;
    for (int64_t it = 0; it < my_n; ++it) {
        mbar_wait(smem_u32(&bars[s]), parity);
        const unsigned char* st = smem_raw + (size_t)s * A.stage_bytes;
        // 1. my pass bits + survivors per (slab, warp), from the bitmap of pass 1 (one word per warp and slab)
        unsigned my = 0;
        const int64_t word0 = ((tile0 + it) * A.tile_rows) >> 5;
        for (int r = 0; r < slabs; ++r) {
            const unsigned bal = __ldg(&bitmap[word0 + r * (C_NT / 32) + warp]);
            if (lane == 0) wcount[r * (C_NT / 32) + warp] = __popc(bal);
            my |= ((bal >> lane) & 1u) << r;
        }
        __syncthreads();
        // 2. exclusive scan of the slabs x 8 counts by warp 0
        if (warp == 0) {
            int carry = 0;
            for (int b = 0; b < nw; b += 32) {
                const int i = b + lane;
                int v = i < nw ? wcount[i] : 0, x = v;
                for (int o = 1; o < 32; o <<= 1) {
                    const int y = __shfl_up_sync(0xffffffffu, x, o);
                    if (lane >= o) x += y;
                }
                if (i < nw) wcount[i] = carry + x - v;
                carry += __shfl_sync(0xffffffffu, x, 31);
            }
            if (lane == 0) wcount[nw] = carry;
        }
        __syncthreads();
        // 3. survivors, in row order, column by column (the width switch is outside the row loop)
        for (int c = 0; c < A.ncols; ++c) {
            const unsigned char* src = st + A.off[c];
            switch (A.width[c]) {
                case 1: copy_col<unsigned char>(src, A.dst[c], slabs, my, wcount, running, warp, lane); break;
                case 4: copy_col<unsigned>(src, A.dst[c], slabs, my, wcount, running, warp, lane); break;
                default: copy_col<unsigned long long>(src, A.dst[c], slabs, my, wcount, running, warp, lane); break;
            }
        }
        running += wcount[nw];
        __syncthreads();                                   // stage s and wcount are free again
        if (threadIdx.x == 0 && it + C_STAGES < my_n)
            issue_tile(A, tile0 + it + C_STAGES, smem_raw + (size_t)s * A.stage_bytes, smem_u32(&bars[s]));
        if (++s == C_STAGES) { s = 0; parity ^= 1u; }
    }
    // ragged tail of the chunk (< tile_rows rows, only the last chunk has one): straight from global memory
    const int64_t t0 = lo + my_n * A.tile_rows;
    if (t0 < hi) {
        __shared__ int tsum[C_NT / 32];
        for (int64_t k0 = t0; k0 < hi; k0 += C_NT) {
            const int64_t row = k0 + threadIdx.x;
            const unsigned bal = k0 + warp * 32 < hi ? __ldg(&bitmap[(k0 >> 5) + warp]) : 0u;     // bits past `hi` are 0
            const bool pass = (bal >> lane) & 1u;
            if (lane == 0) tsum[warp] = __popc(bal);
            __syncthreads();
            int before = 0, total = 0;
            for (int w = 0; w < C_NT / 32; ++w) { if (w < warp) before += tsum[w]; total += tsum[w]; }
            if (pass) copy_row(A, A.src, row, running + before + __popc(bal & lanemask_lt()));
            running += total;
            __syncthreads();
        }
    }
}

}  // namespace

int try_filter_compact_tma(const qk_column* cols, int ncols, int64_t nrows, const qk_expr* pred, const qk_expr* proj, int nproj,
                           qk_column* out, int64_t* out_rows, void* workspace, size_t ws_bytes, const qk_bloom* bloom, cudaStream_t st) {
    if (nproj < 1 || nproj > C_MAXCOLS) return 1;
    CompactArgs A{};
    if (bloom && bloom->bits) {
        if (bloom->key_proj < 0 || bloom->key_proj >= nproj || bloom->nparts < 1 || bloom->words_per_part < 8 || (bloom->words_per_part & 7))
            QK_FAIL(QK_ERR_INVALID, "qk_scan_filter_project_sj: bad Bloom descriptor");
        A.bloom = (const unsigned*)bloom->bits; A.bloom_words = bloom->words_per_part; A.bloom_nparts = bloom->nparts; A.bloom_col = bloom->key_proj;
    }
    const int npred = pred ? pred->n_nodes : 0;
    int row_bytes = 0;
    auto al16 = [](const void* p) { return ((uintptr_t)p & 15) == 0; };
    for (int j = 0; j < nproj; ++j) {
        if (proj[j].n_nodes != 1 || proj[j].nodes[0].op != QK_OP_COL) return 1;       // expressions: interpreter path
        const qk_column& c = cols[proj[j].nodes[0].a0];
        if (!al16(c.data) || !al16(out[j].data)) return 1;
        A.src[j] = (const unsigned char*)c.data; A.dst[j] = (unsigned char*)out[j].data; A.width[j] = dtype_size(c.dtype);
        row_bytes += A.width[j];
    }
    A.ncols = nproj;
    if (npred == 0) {
        A.pred_col = nullptr; A.pred_width = 0;
    } else {
        if (npred != 1 || (pred->nodes[0].op != QK_OP_CMP_COL_IMM && pred->nodes[0].op != QK_OP_RANGE_COL_IMM)) return 1;
        const qk_expr_node& nd = pred->nodes[0];
        const qk_column& c = cols[nd.a0];
        if (!al16(c.data)) return 1;
        A.pred_col = (const unsigned char*)c.data; A.pred_width = dtype_size(c.dtype);
        const long long imm = nd.imm_i;
        long long lo = INT64_MIN, hi = INT64_MAX;
        bool empty = false;
        A.pred_neg = 0;
        if (nd.op == QK_OP_RANGE_COL_IMM) { lo = nd.imm_i; hi = (long long)nd.imm; A.pred_neg = nd.a1 != 0; empty = lo > hi; }
        else switch (nd.a1) {
            case QK_CMP_LT: if (imm == INT64_MIN) empty = true; else hi = imm - 1; break;
            case QK_CMP_LE: hi = imm; break;
            case QK_CMP_GT: if (imm == INT64_MAX) empty = true; else lo = imm + 1; break;
            case QK_CMP_GE: lo = imm; break;
            case QK_CMP_EQ: lo = hi = imm; break;
            default: lo = hi = imm; A.pred_neg = 1; break;
        }
        if (empty) { lo = 1; hi = 0; }
        A.pred_lo = lo; A.pred_hi = hi;
    }
    // tile size: 3 CTAs per SM (so one CTA's output-reservation atomic overlaps the others' work), each with a
    // 3-stage ring inside ~72 KB; QK_COMPACT_CTAS overrides the CTAs-per-SM target for experiments
    static int ctas_per_sm = [] { const char* e = getenv("QK_COMPACT_CTAS"); int v = e ? atoi(e) : 3; return v < 1 ? 1 : (v > 4 ? 4 : v); }();
    int tile = ((216 * 1024 / ctas_per_sm - 1024) / C_STAGES / row_bytes) / C_NT * C_NT;
    if (tile > C_MAXSLABS * C_NT) tile = C_MAXSLABS * C_NT;
    if (tile < C_NT) return 1;
    A.tile_rows = tile;
    int off = 0;
    // widest columns first keeps every sub-array 16-byte aligned (tile is a multiple of 256 rows)
    for (int w : {8, 4, 1}) {
        for (int j = 0; j < nproj; ++j) if (A.width[j] == w) { A.off[j] = off; off += w * tile; }
    }
    A.stage_bytes = off;
    const size_t smem = (size_t)C_STAGES * A.stage_bytes;
    QK_CUDA(cudaFuncSetAttribute(k_filter_compact_tma, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int sms = sm_count();
    // contiguous chunks of whole tiles, one per CTA
    const int64_t ntiles = (nrows + tile - 1) / tile;
    int64_t want = (int64_t)sms * ctas_per_sm;
    if (want > 1024) want = 1024;
    const int64_t tiles_per_chunk = (ntiles + want - 1) / want;
    const int64_t chunk_rows = tiles_per_chunk * tile;
    const int nb = (int)((nrows + chunk_rows - 1) / chunk_rows);
    const size_t bitmap_bytes = align_up((size_t)((nrows + 31) / 32 + 8) * 4, 256);
    if (ws_bytes < (size_t)(2 * 1024 + 8) * 8 + bitmap_bytes || !workspace) return 1;
    long long* counts = (long long*)workspace;
    long long* offsets = counts + 1024;
    unsigned* bitmap = (unsigned*)((char*)workspace + (size_t)(2 * 1024 + 8) * 8);
    if (A.bloom) {
        const int kd = cols[proj[A.bloom_col].nodes[0].a0].dtype;
        if (kd != QK_I64 && kd != QK_I32) QK_FAIL(QK_ERR_UNSUPPORTED, "qk_scan_filter_project_sj: the join key must be int64 / int32");
    }
    {
        const int pw = A.pred_col ? A.pred_width : 0, kw = A.bloom ? A.width[A.bloom_col] : 0;
#define QK_MASK(PW, KW) k_compact_mask<PW, KW><<<nb, M_NT, 0, st>>>(A, nrows, chunk_rows, bitmap, counts)
        if (kw == 0) { if (pw == 0) QK_MASK(0, 0); else if (pw == 1) QK_MASK(1, 0); else if (pw == 4) QK_MASK(4, 0); else QK_MASK(8, 0); }
        else if (kw == 4) { if (pw == 0) QK_MASK(0, 4); else if (pw == 1) QK_MASK(1, 4); else if (pw == 4) QK_MASK(4, 4); else QK_MASK(8, 4); }
        else { if (pw == 0) QK_MASK(0, 8); else if (pw == 1) QK_MASK(1, 8); else if (pw == 4) QK_MASK(4, 8); else QK_MASK(8, 8); }
#undef QK_MASK
    }
    QK_LAUNCH_CHECK("k_compact_mask");
    k_compact_scan<<<1, 1024, 0, st>>>(counts, nb, offsets, (long long*)out_rows);
    QK_LAUNCH_CHECK("k_compact_scan");
    k_filter_compact_tma<<<nb, C_NT, smem, st>>>(A, nrows, chunk_rows, offsets, bitmap);
    QK_LAUNCH_CHECK("k_filter_compact_tma");
    return 0;
}

int bloom_build(const qk_column* key, unsigned* bits, long long words_per_part, int nparts, cudaStream_t st) {
    if (key->length == 0) return QK_OK;
    int64_t nb = (key->length + 255) / 256;
    if (nb > (int64_t)sm_count() * 16) nb = (int64_t)sm_count() * 16;
    k_bloom_build<<<(unsigned)nb, 256, 0, st>>>(key->data, key->dtype, key->length, bits, words_per_part, nparts);
    QK_LAUNCH_CHECK("k_bloom_build");
    return QK_OK;
}

}  // namespace qk
