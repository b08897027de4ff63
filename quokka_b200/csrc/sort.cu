// sort.cu -- K13 stable LSD radix sort to a permutation (DataStream.sort; sql_executors.py:88-187 SuperFastSortExecutor).
//
// The key is mapped once to its 64-bit order image (common.cuh order_image, complemented for descending order) and the
// (image, row number) pairs are sorted by 8-bit digits, least significant first, between two buffers.  Payload columns
// never travel: the caller moves them once with qk_gather(perm).  Per live pass the algorithm moves
//   count   8 B/row read  (the image array; 4 B/row for the NULL pass, which reads the row numbers)
//   scatter 12 B/row read + 12 B/row written
// and pass 0 reads the key (through perm_in when given) and writes 12 B/row.  The host never reads a histogram: pass 0
// accumulates all digit histograms at once, k_sort_plan turns them into per-digit bin bases and marks the digits in
// which every valid row agrees, and the kernels of such a digit return at once (the source buffer of every pass is part of
// that plan, in device memory).  The last live pass writes straight to perm_out / image_out.
// NULL rows (valid == 0) carry bit 31 of their row number through the passes (row numbers are < 2^31) and one image, so
// they tie; a final 1-bit pass on that flag puts them last.  Every position is a sum of counts: no atomic decides one.
#include "common.cuh"

namespace qk {
namespace {

constexpr int S_NT = 512;                       // threads of the count and scatter CTAs
constexpr int S_ITEMS = 8;                      // rows per thread and tile
constexpr int S_TILE = S_NT * S_ITEMS;          // 4096 rows ranked and reordered in shared memory at a time
constexpr int S_WARPS = S_NT / 32;
constexpr int S_DIGITS = 9;                     // the image's eight bytes, least significant first, then the NULL flag
constexpr int S_MAX_CHUNKS = 1024;              // one chunk of whole tiles per CTA of the persistent grid
constexpr unsigned S_NULL = 0x80000000u;
constexpr size_t S_SCATTER_SMEM = (size_t)S_TILE * 12 + 256 * 20 + S_WARPS * 4 + (size_t)S_WARPS * 256 * 2;

struct SortState {
    unsigned hist[S_DIGITS][256];
    long long base[S_DIGITS][256];              // first output position of every bin
    int live[S_DIGITS];                         // 0: every row has the same digit, the pass is skipped
    int src[S_DIGITS];                          // the buffer (0 / 1) pass d reads
    int last_live;                              // -1: no pass runs and k_sort_finish copies buffer 0
};

__device__ int g_sort_plan[2];                  // live image passes and live NULL pass of the last sort (qk_sort_last_plan)

__device__ __forceinline__ int digit_of(unsigned long long im, unsigned rw, int d) {
    return d < 8 ? (int)((im >> (8 * d)) & 0xff) : (int)(rw >> 31);
}

// pass 0: image + row number of every row, and the histograms of digits [d_lo, d_hi) (one shared-memory atomic per
// warp, digit and distinct value; one global add per CTA and bin)
__global__ void __launch_bounds__(256) k_sort_image_hist(const void* key, int dt, const uint8_t* valid, int descending,
                                                         const int32_t* perm_in, int64_t n, int d_lo, int d_hi,
                                                         unsigned long long* img, unsigned* row, SortState* S) {
    __shared__ unsigned sh[S_DIGITS][256];
    for (int j = threadIdx.x; j < S_DIGITS * 256; j += 256) (&sh[0][0])[j] = 0;
    __syncthreads();
    const unsigned long long flip = descending ? ~0ull : 0ull;
    const int64_t nround = (n + 31) / 32 * 32;
    for (int64_t i = blockIdx.x * 256ll + threadIdx.x; i < nround; i += gridDim.x * 256ll) {
        const bool in = i < n;
        unsigned long long im = 0;
        unsigned rw = 0;
        if (in) {
            const int32_t s = perm_in ? perm_in[i] : (int32_t)i;
            const bool null = valid && valid[s] == 0;
            im = (null ? 0ull : order_image(key, dt, s)) ^ flip;        // NULLs share one image
            rw = (unsigned)s | (null ? S_NULL : 0u);
            img[i] = im;
            row[i] = rw;
        }
        for (int d = d_lo; d < d_hi; ++d) {
            const int dg = in ? digit_of(im, rw, d) : -1;
            const unsigned peers = __match_any_sync(0xffffffffu, dg);
            if (in && (peers & lanemask_lt()) == 0) atomicAdd(&sh[d][dg], (unsigned)__popc(peers));
        }
    }
    __syncthreads();
    for (int d = d_lo; d < d_hi; ++d)
        if (sh[d][threadIdx.x]) atomicAdd(&S->hist[d][threadIdx.x], sh[d][threadIdx.x]);
}

// one CTA: bin bases of every digit, the digits worth a pass, and the buffer each pass reads
__global__ void __launch_bounds__(256) k_sort_plan(SortState* S, long long n, int d_lo, int d_hi, int null_digit) {
    __shared__ long long wsum[8];
    // the NULL rows tie whatever their image, so an image digit is worth a pass only when the VALID rows differ in it:
    // the NULLs (all in bin null_digit of every image digit) are taken out of the counts that are tested
    const long long nnull = d_hi == S_DIGITS ? (long long)S->hist[8][1] : 0;
    for (int d = 0; d < S_DIGITS; ++d) {
        const bool on = d >= d_lo && d < d_hi;
        const long long c = on ? (long long)S->hist[d][threadIdx.x] : 0;
        long long total;
        S->base[d][threadIdx.x] = cta_exclusive_scan<256>(c, wsum, total);
        const bool all = d < 8 ? c - ((int)threadIdx.x == null_digit ? nnull : 0) == n - nnull : c == n;
        const int uniform = __syncthreads_or(all);                     // also the barrier before wsum is used again
        if (threadIdx.x == 0) S->live[d] = on && !uniform;
    }
    if (threadIdx.x == 0) {
        int par = 0, last = -1, nlive = 0;
        for (int d = 0; d < S_DIGITS; ++d) {
            S->src[d] = par;
            if (S->live[d]) { par ^= 1; last = d; nlive += d < 8; }
        }
        S->last_live = last;
        g_sort_plan[0] = nlive;
        g_sort_plan[1] = S->live[8];
    }
}

// counts[bin * nchunks + chunk] = rows of the chunk whose digit d is `bin`
__global__ void __launch_bounds__(S_NT) k_sort_count(const SortState* S, int d, const unsigned long long* img0,
                                                     const unsigned long long* img1, const unsigned* row0, const unsigned* row1,
                                                     int64_t n, int64_t chunk_rows, int64_t nchunks, unsigned* counts) {
    if (!S->live[d]) return;
    __shared__ unsigned sh[256];
    if (threadIdx.x < 256) sh[threadIdx.x] = 0;
    __syncthreads();
    const unsigned long long* img = S->src[d] ? img1 : img0;
    const unsigned* row = S->src[d] ? row1 : row0;
    const int64_t start = blockIdx.x * chunk_rows, end = start + chunk_rows < n ? start + chunk_rows : n;
    for (int64_t i = start + threadIdx.x; i < start + chunk_rows; i += S_NT) {          // chunk_rows is a multiple of S_NT
        const bool in = i < end;
        const int dg = !in ? -1 : d < 8 ? digit_of(img[i], 0u, d) : digit_of(0ull, row[i], d);
        const unsigned peers = __match_any_sync(0xffffffffu, dg);
        if (in && (peers & lanemask_lt()) == 0) atomicAdd(&sh[dg], (unsigned)__popc(peers));
    }
    __syncthreads();
    if (threadIdx.x < 256) counts[(size_t)threadIdx.x * nchunks + blockIdx.x] = sh[threadIdx.x];
}

// One chunk per CTA, tile by tile.  A warp owns 256 consecutive rows of the tile and visits them 32 at a time in row
// order: the rank of a row among the warp's earlier rows of its bin is the warp's running count of the bin plus its rank
// among the peers of a match_any.  The warps' counts are then scanned per bin and the bins across the tile, the tile is
// reordered in shared memory, and every bin's run leaves as consecutive stores behind the chunk's running bin offsets.
__global__ void __launch_bounds__(S_NT, 2) k_sort_scatter(const SortState* S, int d, unsigned long long* img0,
                                                          unsigned long long* img1, unsigned* row0, unsigned* row1,
                                                          int32_t* perm_out, unsigned long long* image_out, int64_t n,
                                                          int64_t chunk_rows, int64_t nchunks, const int64_t* offsets) {
    if (!S->live[d]) return;
    extern __shared__ __align__(16) unsigned char smem[];
    unsigned long long* simg = (unsigned long long*)smem;
    long long* sdelta = (long long*)(simg + S_TILE);            // global position of a bin's run minus its place in the tile
    long long* running = sdelta + 256;                          // next global position of every bin
    unsigned* srow = (unsigned*)(running + 256);
    int* sbin = (int*)(srow + S_TILE);                          // first place of every bin in the reordered tile
    int* wsum = sbin + 256;
    uint16_t* wc = (uint16_t*)(wsum + S_WARPS);                 // wc[warp][bin]: the warp's count, then its offset in the bin
    const int warp = threadIdx.x >> 5, lane = lane_id();
    const int sb = S->src[d];
    const bool last = S->last_live == d;
    const unsigned long long* img = sb ? img1 : img0;
    const unsigned* row = sb ? row1 : row0;
    unsigned long long* oimg = last ? image_out : (sb ? img0 : img1);
    unsigned* orow = last ? (unsigned*)perm_out : (sb ? row0 : row1);
    const unsigned keep = last ? ~S_NULL : ~0u;
    const int64_t start = blockIdx.x * chunk_rows, end = start + chunk_rows < n ? start + chunk_rows : n;
    if (threadIdx.x < 256) running[threadIdx.x] = S->base[d][threadIdx.x] + offsets[(size_t)threadIdx.x * nchunks + blockIdx.x];
    uint16_t* mywc = wc + warp * 256;
    for (int64_t tbase = start; tbase < end; tbase += S_TILE) {
        for (int j = threadIdx.x; j < S_WARPS * 128; j += S_NT) ((unsigned*)wc)[j] = 0;
        __syncthreads();
        unsigned long long im[S_ITEMS];
        unsigned rw[S_ITEMS];
        int rk[S_ITEMS];                                        // digit << 16 | rank in the warp's rows of the bin, -1 past the end
        const int64_t wbase = tbase + warp * (32 * S_ITEMS) + lane;
#pragma unroll
        for (int r = 0; r < S_ITEMS; ++r) {
            const int64_t i = wbase + r * 32;
            const bool in = i < end;
            im[r] = in ? img[i] : 0ull;
            rw[r] = in ? row[i] : 0u;
        }
#pragma unroll
        for (int r = 0; r < S_ITEMS; ++r) {
            const bool in = wbase + r * 32 < end;
            const int dg = in ? digit_of(im[r], rw[r], d) : -1;
            const unsigned peers = __match_any_sync(0xffffffffu, dg);
            const int before = in ? mywc[dg] : 0;
            __syncwarp();
            if (in && (peers & lanemask_lt()) == 0) mywc[dg] = (uint16_t)(before + __popc(peers));
            __syncwarp();
            rk[r] = in ? (dg << 16 | (before + __popc(peers & lanemask_lt()))) : -1;
        }
        __syncthreads();
        int cnt = 0;
        if (threadIdx.x < 256)
            for (int w = 0; w < S_WARPS; ++w) {
                const int t = wc[w * 256 + threadIdx.x];
                wc[w * 256 + threadIdx.x] = (uint16_t)cnt;
                cnt += t;
            }
        int total;
        const int first = cta_exclusive_scan<S_NT>(cnt, wsum, total);
        if (threadIdx.x < 256) {
            sbin[threadIdx.x] = first;
            sdelta[threadIdx.x] = running[threadIdx.x] - first;
            running[threadIdx.x] += cnt;
        }
        __syncthreads();
#pragma unroll
        for (int r = 0; r < S_ITEMS; ++r) {
            if (rk[r] < 0) continue;
            const int dg = rk[r] >> 16, pos = sbin[dg] + mywc[dg] + (rk[r] & 0xffff);
            simg[pos] = im[r];
            srow[pos] = rw[r];
        }
        __syncthreads();
        for (int p = threadIdx.x; p < total; p += S_NT) {
            const unsigned long long v = simg[p];
            const unsigned w = srow[p];
            const long long g = p + sdelta[digit_of(v, w, d)];
            if (oimg) oimg[g] = v;
            orow[g] = w & keep;
        }
        __syncthreads();
    }
}

// every row agreed in every digit: the order is the input order
__global__ void __launch_bounds__(256) k_sort_finish(const SortState* S, const unsigned long long* img0, const unsigned* row0,
                                                     int32_t* perm_out, unsigned long long* image_out, int64_t n) {
    if (S->last_live >= 0) return;
    for (int64_t i = blockIdx.x * 256ll + threadIdx.x; i < n; i += gridDim.x * 256ll) {
        perm_out[i] = (int32_t)(row0[i] & ~S_NULL);
        if (image_out) image_out[i] = img0[i];
    }
}

// the workspace: both (image, row number) buffers, the plan, then the per-chunk bin counts, their offsets and the bin totals
struct SortWs {
    unsigned long long* img[2]; unsigned* row[2]; SortState* S; unsigned* counts; int64_t* offsets; int64_t* totals; size_t bytes;
    SortWs(int64_t n, void* base) {
        Carve c(base);
        for (int b = 0; b < 2; ++b) img[b] = c.take<unsigned long long>(n);
        for (int b = 0; b < 2; ++b) row[b] = c.take<unsigned>(n);
        S = c.take<SortState>(1);
        counts = c.take<unsigned>((size_t)S_MAX_CHUNKS * 256);
        offsets = c.take<int64_t>((size_t)S_MAX_CHUNKS * 256);
        totals = c.take<int64_t>(256);
        bytes = c.bytes;
    }
};

thread_local char g_sort_plan_text[48] = "";
thread_local int g_sort_device = -1;

}  // namespace
}  // namespace qk

using namespace qk;

static int64_t sort_chunk_rows(int64_t n) {
    const int64_t tiles = (n + S_TILE - 1) / S_TILE;
    int64_t grid = (int64_t)sm_count() * 2;                        // two resident scatter CTAs per SM
    if (grid > S_MAX_CHUNKS) grid = S_MAX_CHUNKS;
    return (tiles + grid - 1) / grid * S_TILE;
}

extern "C" size_t qk_sort_workspace_bytes(int64_t nrows) {
    return nrows < 0 ? 0 : SortWs(nrows, nullptr).bytes;
}

extern "C" int qk_sort_perm(const qk_column* key, const uint8_t* valid, int32_t descending, const int32_t* perm_in,
                            int32_t* perm_out, uint64_t* image_out, int64_t nrows, void* workspace, size_t ws_bytes, void* stream) {
    const char* who = "qk_sort_perm";
    if (nrows > 0x7fffffffLL) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: %lld rows; row numbers are int32", who, (long long)nrows);
    if (int rc = check_col(key, who)) return rc;
    if (nrows < 0 || key->length != nrows) QK_FAIL(QK_ERR_INVALID, "%s: the key holds %lld rows, nrows is %lld", who, (long long)key->length, (long long)nrows);
    const int64_t n = nrows;
    if (n == 0) return QK_OK;
    if (!perm_out) QK_FAIL(QK_ERR_INVALID, "%s: null perm_out", who);
    const SortWs w(n, workspace);
    if (!workspace || ws_bytes < w.bytes) QK_FAIL(QK_ERR_CAPACITY, "%s: workspace too small", who);
    cudaStream_t st = (cudaStream_t)stream;
    // the digits below the key's width are the same in every image; the NULL digit exists only with a mask
    const int d_lo = 8 - dtype_size(key->dtype), d_hi = valid ? 9 : 8;
    QK_CUDA(cudaMemsetAsync(w.S->hist, 0, sizeof(w.S->hist), st));
    k_sort_image_hist<<<grid_size(n, 8), 256, 0, st>>>(key->data, key->dtype, valid, descending, perm_in, n, d_lo, d_hi, w.img[0], w.row[0], w.S);
    QK_LAUNCH_CHECK("k_sort_image_hist");
    k_sort_plan<<<1, 256, 0, st>>>(w.S, n, d_lo, d_hi, descending ? 0xff : 0);
    QK_LAUNCH_CHECK("k_sort_plan");
    const int64_t chunk_rows = sort_chunk_rows(n), nchunks = (n + chunk_rows - 1) / chunk_rows;
    QK_CUDA(qk::raise_smem_limit((const void*)k_sort_scatter, (size_t)S_SCATTER_SMEM));
    for (int d = d_lo; d < d_hi; ++d) {
        k_sort_count<<<(unsigned)nchunks, S_NT, 0, st>>>(w.S, d, w.img[0], w.img[1], w.row[0], w.row[1], n, chunk_rows, nchunks, w.counts);
        QK_LAUNCH_CHECK("k_sort_count");
        if (int rc = count_offsets(w.counts, 256, nchunks, w.offsets, w.totals, st)) return rc;
        k_sort_scatter<<<(unsigned)nchunks, S_NT, S_SCATTER_SMEM, st>>>(w.S, d, w.img[0], w.img[1], w.row[0], w.row[1], perm_out,
                                                                       (unsigned long long*)image_out, n, chunk_rows, nchunks, w.offsets);
        QK_LAUNCH_CHECK("k_sort_scatter");
    }
    k_sort_finish<<<grid_size(n, 8), 256, 0, st>>>(w.S, w.img[0], w.row[0], perm_out, (unsigned long long*)image_out, n);
    QK_LAUNCH_CHECK("k_sort_finish");
    cudaGetDevice(&g_sort_device);
    return QK_OK;
}

// reads the plan of the last qk_sort_perm of this thread back from its device (waits for the device)
extern "C" const char* qk_sort_last_plan(void) {
    if (g_sort_device < 0) return g_sort_plan_text;
    int cur = 0, plan[2] = {0, 0};
    cudaGetDevice(&cur);
    cudaSetDevice(g_sort_device);
    const cudaError_t e = cudaDeviceSynchronize() == cudaSuccess ? cudaMemcpyFromSymbol(plan, g_sort_plan, sizeof(plan)) : cudaErrorUnknown;
    cudaSetDevice(cur);
    if (e != cudaSuccess) { set_err("qk_sort_last_plan: %s", cudaGetErrorString(e)); return ""; }
    snprintf(g_sort_plan_text, sizeof(g_sort_plan_text), "d8 passes=%d/8 nulls=%d", plan[0], plan[1]);
    return g_sort_plan_text;
}
