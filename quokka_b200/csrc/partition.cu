// partition.cu -- K3 stable multi-way partition (hash-partition shuffle input, segment-by-symbol),
// plus the scatter / gather movers that materialise columns.  All HBM-bound:
//   plan    reads the key column twice (histogram + rank): 2 x key bytes, writes 4 B/row (dest)
//   scatter reads + writes every payload byte once (+ 4 B/row of dest)
// Stability (rows keep their order inside a partition) is what lets the as-of path partition by
// symbol without re-sorting by time, and matches Polars partition_by (quokka_runtime.py:222).
#include "common.cuh"

namespace qk {
namespace {

constexpr int P_NT = 256;
constexpr int P_CHUNK_MIN = 4096;        // rows per CTA-chunk (grows with nparts so that the count matrix stays small)
constexpr int P_SMEM_PARTS = 16384;      // partitions whose per-chunk histogram lives in shared memory

__device__ __forceinline__ int part_of(const void* key, int dt, int64_t row, int nparts, int mode) {
    const int64_t k = load_i64(key, dt, row);
    if (mode == QK_PART_CODE) return (int)(k < 0 ? 0 : (k >= nparts ? nparts - 1 : k));   // codes are clamped (memory safety)
    return (int)part_mod(k, (unsigned)nparts);      // reference: key % num_target_channels (quokka_runtime.py:222), without a 64-bit division
}

// pass 1: per-chunk histogram, stored partition-major: hist[p * nchunks + chunk]
// rows per chunk: keeps nchunks * nparts (the count matrix) under ~4 M entries and a partition's row of it short
// enough for one CTA to scan in a few steps, while leaving several chunks per CTA of the persistent grids
static int64_t chunk_rows_for(int64_t n, int nparts) {
    int64_t max_chunks = (int64_t)(1 << 22) / (nparts > 0 ? nparts : 1);
    if (max_chunks < 1) max_chunks = 1;
    if (max_chunks > 8192) max_chunks = 8192;
    int64_t c = (n + max_chunks - 1) / max_chunks;
    if (c < P_CHUNK_MIN) c = P_CHUNK_MIN;
    return (c + P_NT - 1) / P_NT * P_NT;
}

__global__ void __launch_bounds__(P_NT) k_part_hist(const void* key, int dt, int64_t n, int nparts, int mode,
                                                    int64_t nchunks, int64_t chunk_rows, unsigned* hist) {
    extern __shared__ __align__(16) unsigned sh[];
    for (int64_t chunk = blockIdx.x; chunk < nchunks; chunk += gridDim.x) {
        for (int p = threadIdx.x; p < nparts; p += P_NT) sh[p] = 0;
        __syncthreads();
        const int64_t base = chunk * chunk_rows;
        for (int64_t t = threadIdx.x; t < chunk_rows; t += P_NT) {
            const int64_t row = base + t;
            const int p = row < n ? part_of(key, dt, row, nparts, mode) : -1;
            const unsigned peers = __match_any_sync(0xffffffffu, p);       // one shared-memory atomic per
            if (p >= 0 && (peers & lanemask_lt()) == 0) atomicAdd(&sh[p], (unsigned)__popc(peers));  // (warp, partition)
        }
        __syncthreads();
        for (int p = threadIdx.x; p < nparts; p += P_NT) hist[(size_t)p * nchunks + chunk] = sh[p];
        __syncthreads();
    }
}

// pass 2a: one CTA per partition scans that partition's per-chunk counts (a contiguous row of the partition-major
// histogram) -> offsets RELATIVE to the partition's start, and the partition's row total.
__global__ void __launch_bounds__(P_NT) k_part_scan_rows(const unsigned* hist, int64_t nchunks, int64_t* offsets, int64_t* totals) {
    __shared__ int64_t wtot[P_NT / 32];
    const int64_t row = (int64_t)blockIdx.x * nchunks;
    const int warp = threadIdx.x >> 5;
    int64_t carry = 0;
    for (int64_t base = 0; base < nchunks; base += P_NT) {
        const int64_t i = base + threadIdx.x;
        const int64_t v = i < nchunks ? hist[row + i] : 0;
        int64_t x = v;
        for (int o = 1; o < 32; o <<= 1) {
            const int64_t y = __shfl_up_sync(0xffffffffu, x, o);
            if ((int)lane_id() >= o) x += y;
        }
        if (lane_id() == 31) wtot[warp] = x;
        __syncthreads();
        int64_t before = 0, total = 0;
        for (int w = 0; w < P_NT / 32; ++w) { if (w < warp) before += wtot[w]; total += wtot[w]; }
        if (i < nchunks) offsets[row + i] = carry + before + x - v;
        carry += total;
        __syncthreads();
    }
    if (threadIdx.x == 0) totals[blockIdx.x] = carry;
}
// pass 2b: exclusive scan of the nparts totals (single CTA; nparts <= 16384) -> part_offsets[nparts + 1]
__global__ void __launch_bounds__(1024) k_part_scan_totals(const int64_t* totals, int nparts, int64_t* part_offsets) {
    __shared__ int64_t wtot[32];
    __shared__ int64_t carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (int base = 0; base < nparts; base += 1024) {
        const int i = base + threadIdx.x;
        int64_t v = i < nparts ? totals[i] : 0, x = v;
        for (int o = 1; o < 32; o <<= 1) {
            int64_t y = __shfl_up_sync(0xffffffffu, x, o);
            if ((int)lane_id() >= o) x += y;
        }
        if (lane_id() == 31) wtot[threadIdx.x >> 5] = x;
        __syncthreads();
        if (threadIdx.x < 32) {
            int64_t w = wtot[threadIdx.x], t = w;
            for (int o = 1; o < 32; o <<= 1) {
                int64_t y = __shfl_up_sync(0xffffffffu, t, o);
                if ((int)lane_id() >= o) t += y;
            }
            wtot[threadIdx.x] = t - w;
        }
        __syncthreads();
        const int64_t excl = carry + wtot[threadIdx.x >> 5] + x - v;
        if (i < nparts) part_offsets[i] = excl;
        __syncthreads();
        if (threadIdx.x == 1023) carry = excl + v;
        __syncthreads();
    }
    if (threadIdx.x == 0) part_offsets[nparts] = carry;
}

// pass 3: stable rank of every row inside its chunk -> dest.  Rows are visited in order, one 256-row
// slab at a time.  Inside a warp the rank among equal partitions comes from match_any + popc (peer
// ballot); across warps from a per-warp count table in shared memory, so all 8 warps work in parallel
// and a slab costs three CTA barriers.
__global__ void __launch_bounds__(P_NT) k_part_dest(const void* key, int dt, int64_t n, int nparts, int mode,
                                                    int64_t nchunks, int64_t chunk_rows, const int64_t* offsets,
                                                    const int64_t* part_offsets, int32_t* dest) {
    extern __shared__ __align__(16) unsigned sh[];   // wcount[nparts][8] (u8) first (8-byte aligned), then running[nparts] (u32)
    uint8_t* wcount = (uint8_t*)sh;                  // 8 bytes per partition: one count per warp (<= 32)
    unsigned* running = sh + 2 * nparts;
    const int warp = threadIdx.x >> 5;
    static_assert(P_NT / 32 == 8, "one byte per warp in a 64-bit word");
    for (int p = threadIdx.x; p < nparts * 2; p += P_NT) ((unsigned*)wcount)[p] = 0;
    for (int64_t chunk = blockIdx.x; chunk < nchunks; chunk += gridDim.x) {
        for (int p = threadIdx.x; p < nparts; p += P_NT) running[p] = 0;
        __syncthreads();
        const int64_t base = chunk * chunk_rows;
        for (int64_t t0 = 0; t0 < chunk_rows && base + t0 < n; t0 += P_NT) {
            const int64_t row = base + t0 + threadIdx.x;
            const bool valid = row < n;
            const int p = valid ? part_of(key, dt, row, nparts, mode) : -1;
            const unsigned peers = __match_any_sync(0xffffffffu, p);
            const int rank = __popc(peers & lanemask_lt());
            const int npeers = __popc(peers);
            if (valid && rank == 0) wcount[p * 8 + warp] = (uint8_t)npeers;
            __syncthreads();
            if (valid) {
                // counts of the warps before mine: low `warp` bytes of the 64-bit word, summed by a multiply
                const unsigned long long wc = *(const unsigned long long*)(wcount + p * 8);
                const unsigned long long lowmask = warp == 0 ? 0ull : (~0ull >> (64 - 8 * warp));
                const unsigned before = running[p] + (unsigned)(((wc & lowmask) * 0x0101010101010101ull) >> 56);
                dest[row] = (int32_t)(part_offsets[p] + offsets[(size_t)p * nchunks + chunk] + before + rank);
            }
            __syncthreads();
            if (valid && rank == 0) {
                atomicAdd(&running[p], (unsigned)npeers);
                wcount[p * 8 + warp] = 0;
            }
            __syncthreads();
        }
    }
}

// ---------------------------------------------------------------- CODE mode over more than P_SMEM_PARTS partitions
// LSD radix: the clamped code is split into 14-bit digits and every digit gets one stable pass of the kernels above (a
// P_SMEM_PARTS-way CODE partition of the digit column).  Stable passes from the low digit up leave the rows sorted by the
// whole code, in input order within a code.
constexpr int P_DIGIT_BITS = 14;
static_assert((1 << P_DIGIT_BITS) == P_SMEM_PARTS, "one digit = one shared-memory partition pass");

__device__ __forceinline__ int32_t clamped_code(const void* key, int dt, int64_t row, int nparts) {
    const int64_t k = load_i64(key, dt, row);
    return (int32_t)(k < 0 ? 0 : (k >= nparts ? nparts - 1 : k));
}

// digit[r] = (clamped code of row r >> shift) & (P_SMEM_PARTS - 1)
__global__ void __launch_bounds__(256) k_radix_digit(const void* key, int dt, int64_t n, int nparts, int shift, int32_t* digit) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        digit[i] = (clamped_code(key, dt, i, nparts) >> shift) & (P_SMEM_PARTS - 1);
}

// after a pass with destination `pass_dest`: the codes move to their new positions, and the final destination of every
// original row follows one more step (dest[i] = pass_dest[dest[i]]; skipped after the first pass, which wrote dest itself)
__global__ void __launch_bounds__(256) k_radix_move(const void* key, int dt, int64_t n, int nparts, const int32_t* pass_dest,
                                                    int32_t* moved, int32_t* dest, int compose) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        moved[pass_dest[i]] = clamped_code(key, dt, i, nparts);
        if (compose) dest[i] = pass_dest[dest[i]];
    }
}

// part_offsets[p] = first position whose code is >= p, over the fully sorted codes (p = nparts gives n)
__global__ void __launch_bounds__(256) k_radix_offsets(const int32_t* sorted, int64_t n, int nparts, int64_t* part_offsets) {
    for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p <= nparts; p += (int64_t)gridDim.x * blockDim.x) {
        int64_t lo = 0, hi = n;
        while (lo < hi) {
            const int64_t mid = (lo + hi) >> 1;
            if (sorted[mid] < p) lo = mid + 1; else hi = mid;
        }
        part_offsets[p] = lo;
    }
}

// ---------------------------------------------------------------- scatter / gather
struct MoveArgs {
    const void* src[QK_MAX_COLS];
    void* dst[QK_MAX_COLS];
    int8_t width[QK_MAX_COLS];
    int32_t ncols;
};

__global__ void __launch_bounds__(256) k_scatter(const __grid_constant__ MoveArgs M, const int32_t* dest, int64_t n) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t d = dest[i];
        for (int c = 0; c < M.ncols; ++c) {
            switch (M.width[c]) {
                case 1: ((uint8_t*)M.dst[c])[d] = ((const uint8_t*)M.src[c])[i]; break;
                case 4: ((uint32_t*)M.dst[c])[d] = ((const uint32_t*)M.src[c])[i]; break;
                default: ((uint64_t*)M.dst[c])[d] = ((const uint64_t*)M.src[c])[i]; break;
            }
        }
    }
}

__global__ void __launch_bounds__(256) k_gather(const __grid_constant__ MoveArgs M, const int32_t* idx, int64_t n) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t s = idx[i];
        for (int c = 0; c < M.ncols; ++c) {
            switch (M.width[c]) {
                case 1: ((uint8_t*)M.dst[c])[i] = s < 0 ? (uint8_t)0 : ((const uint8_t*)M.src[c])[s]; break;
                case 4: ((uint32_t*)M.dst[c])[i] = s < 0 ? 0u : ((const uint32_t*)M.src[c])[s]; break;
                default: ((uint64_t*)M.dst[c])[i] = s < 0 ? 0ull : ((const uint64_t*)M.src[c])[s]; break;
            }
        }
    }
}

// Scatter straight into the receivers' memory: row i of this rank goes to partition p (found from its
// position `dest[i]` in the partition-ordered output), i.e. to peer p, at row peer_row_off[p] + rank-in-partition
// of that peer's receive column.  One pass over the payload does the local re-ordering AND the transfer: the
// stores travel over NVLink (or stay local for p == my rank).  Replaces qk_scatter + an NCCL all-to-all.
struct PeerArgs {
    const void* src[QK_MAX_COLS];
    unsigned long long dst[QK_MAX_PEERS][QK_MAX_COLS];   // device-mapped pointers into every peer's mailbox
    long long row_off[QK_MAX_PEERS];
    int8_t width[QK_MAX_COLS];
    int32_t ncols, nparts;
};

__global__ void __launch_bounds__(256) k_scatter_peer(const __grid_constant__ PeerArgs P, const int32_t* dest, const int64_t* part_offsets, int64_t n) {
    __shared__ long long off[QK_MAX_PEERS + 1];
    if (threadIdx.x <= P.nparts) off[threadIdx.x] = part_offsets[threadIdx.x];
    __syncthreads();
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const long long d = dest[i];
        int p = 0;
        while (p + 1 < P.nparts && d >= off[p + 1]) ++p;
        const long long r = d - off[p] + P.row_off[p];
        for (int c = 0; c < P.ncols; ++c) {
            switch (P.width[c]) {
                case 1: ((uint8_t*)P.dst[p][c])[r] = ((const uint8_t*)P.src[c])[i]; break;
                case 4: ((uint32_t*)P.dst[p][c])[r] = ((const uint32_t*)P.src[c])[i]; break;
                default: ((uint64_t*)P.dst[p][c])[r] = ((const uint64_t*)P.src[c])[i]; break;
            }
        }
    }
}

int fill_move(MoveArgs& M, const qk_column* cols, int ncols, qk_column* out, int64_t n_src, int64_t n_dst, const char* who) {
    if (ncols < 0 || ncols > QK_MAX_COLS) QK_FAIL(QK_ERR_INVALID, "%s: ncols out of range", who);
    M.ncols = ncols;
    for (int c = 0; c < ncols; ++c) {
        if (int rc = check_col(&cols[c], who)) return rc;
        if (int rc = check_col(&out[c], who)) return rc;
        if (cols[c].dtype != out[c].dtype) QK_FAIL(QK_ERR_INVALID, "%s: dtype mismatch on column %d", who, c);
        if (n_src >= 0 && cols[c].length != n_src) QK_FAIL(QK_ERR_INVALID, "%s: column %d length mismatch", who, c);
        if (out[c].length < n_dst) QK_FAIL(QK_ERR_CAPACITY, "%s: output %d too small", who, c);
        M.src[c] = cols[c].data; M.dst[c] = (void*)out[c].data; M.width[c] = (int8_t)dtype_size(cols[c].dtype);
    }
    return 0;
}

}  // namespace
}  // namespace qk

using namespace qk;

// workspace of one shared-memory partition (nparts <= P_SMEM_PARTS)
static size_t smem_plan_bytes(int64_t nrows, int32_t nparts) {
    const int64_t cr = chunk_rows_for(nrows, nparts);
    const int64_t nchunks = (nrows + cr - 1) / cr + 1;
    return align_up((size_t)nchunks * nparts * 4, 256) + align_up((size_t)nchunks * nparts * 8, 256) + align_up((size_t)nparts * 8, 256);
}

// partitions of the radix pass that handles the digit at `shift` (the top digit needs fewer than P_SMEM_PARTS)
static int radix_pass_parts(int32_t nparts, int shift) {
    const int32_t top = (nparts - 1) >> shift;
    return top >= P_SMEM_PARTS - 1 ? P_SMEM_PARTS : top + 1;
}

static int radix_passes(int32_t nparts) {
    int bits = 0;
    while (bits < 31 && ((int64_t)(nparts - 1) >> bits) != 0) ++bits;
    return (bits + P_DIGIT_BITS - 1) / P_DIGIT_BITS;
}

// radix path: digit, pass destination, two code buffers (n x int32 each), the pass's part_offsets, then one
// shared-memory partition's workspace
static size_t radix_plan_bytes(int64_t nrows, int32_t nparts) {
    size_t inner = 0;
    for (int d = 0; d < radix_passes(nparts); ++d) {
        const size_t b = smem_plan_bytes(nrows, radix_pass_parts(nparts, d * P_DIGIT_BITS));
        inner = b > inner ? b : inner;
    }
    return 4 * align_up((size_t)nrows * 4, 256) + align_up((size_t)(P_SMEM_PARTS + 1) * 8, 256) + inner;
}

extern "C" size_t qk_partition_workspace_bytes(int64_t nrows, int32_t nparts) {
    if (nrows < 0 || nparts <= 0) return 0;
    return nparts <= P_SMEM_PARTS ? smem_plan_bytes(nrows, nparts) : radix_plan_bytes(nrows, nparts);
}

// one stable partition with its per-chunk histograms in shared memory (nparts <= P_SMEM_PARTS)
static int smem_plan(const qk_column* key, int32_t nparts, int32_t mode, int32_t* dest, int64_t* part_offsets, void* workspace,
                     cudaStream_t st) {
    const int64_t n = key->length;
    const int64_t chunk_rows = chunk_rows_for(n, nparts);
    const int64_t nchunks = (n + chunk_rows - 1) / chunk_rows;
    unsigned* hist = (unsigned*)workspace;
    int64_t* offsets = (int64_t*)((char*)workspace + align_up((size_t)(nchunks + 1) * nparts * 4, 256));
    int64_t* totals = (int64_t*)((char*)offsets + align_up((size_t)(nchunks + 1) * nparts * 8, 256));
    const int sms = sm_count();
    const int64_t nb = nchunks < (int64_t)sms * 8 ? nchunks : (int64_t)sms * 8;
    const size_t smem = (size_t)nparts * 4;
    QK_CUDA(cudaFuncSetAttribute(k_part_hist, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_part_hist<<<(unsigned)nb, P_NT, smem, st>>>(key->data, key->dtype, n, nparts, mode, nchunks, chunk_rows, hist);
    QK_LAUNCH_CHECK("k_part_hist");
    k_part_scan_rows<<<(unsigned)nparts, P_NT, 0, st>>>(hist, nchunks, offsets, totals);
    QK_LAUNCH_CHECK("k_part_scan_rows");
    k_part_scan_totals<<<1, 1024, 0, st>>>(totals, nparts, part_offsets);
    QK_LAUNCH_CHECK("k_part_scan_totals");
    const size_t smem_dest = (size_t)nparts * 12;
    QK_CUDA(cudaFuncSetAttribute(k_part_dest, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_dest));
    k_part_dest<<<(unsigned)nb, P_NT, smem_dest, st>>>(key->data, key->dtype, n, nparts, mode, nchunks, chunk_rows, offsets, part_offsets, dest);
    QK_LAUNCH_CHECK("k_part_dest");
    return QK_OK;
}

static unsigned grid_of(int64_t n) {            // grid-stride kernels: 256 threads per block, at most 16 blocks per SM
    const int64_t nb = (n + 255) / 256, cap = (int64_t)sm_count() * 16;
    return (unsigned)(nb < 1 ? 1 : (nb > cap ? cap : nb));
}

// CODE partition with more than P_SMEM_PARTS parts: one stable shared-memory pass per 14-bit digit of the clamped code,
// low digit first, then part_offsets by binary search in the sorted codes
static int radix_plan(const qk_column* key, int32_t nparts, int32_t* dest, int64_t* part_offsets, void* workspace, cudaStream_t st) {
    const int64_t n = key->length;
    char* w = (char*)workspace;
    const size_t col_bytes = align_up((size_t)n * 4, 256);
    int32_t* digit = (int32_t*)w; w += col_bytes;
    int32_t* pass_dest = (int32_t*)w; w += col_bytes;
    int32_t* codes[2] = {(int32_t*)w, (int32_t*)(w + col_bytes)}; w += 2 * col_bytes;
    int64_t* pass_offsets = (int64_t*)w; w += align_up((size_t)(P_SMEM_PARTS + 1) * 8, 256);
    const unsigned grid = grid_of(n);
    const void* src = key->data;
    int src_dt = key->dtype;
    const int passes = radix_passes(nparts);
    for (int d = 0; d < passes; ++d) {
        const int shift = d * P_DIGIT_BITS;
        k_radix_digit<<<grid, 256, 0, st>>>(src, src_dt, n, nparts, shift, digit);
        QK_LAUNCH_CHECK("k_radix_digit");
        qk_column dcol = *key;
        dcol.data = digit; dcol.dtype = QK_I32;
        int32_t* out = d == 0 ? dest : pass_dest;
        if (int rc = smem_plan(&dcol, radix_pass_parts(nparts, shift), QK_PART_CODE, out, pass_offsets, w, st)) return rc;
        k_radix_move<<<grid, 256, 0, st>>>(src, src_dt, n, nparts, out, codes[d & 1], dest, d > 0);
        QK_LAUNCH_CHECK("k_radix_move");
        src = codes[d & 1]; src_dt = QK_I32;
    }
    k_radix_offsets<<<grid_of((int64_t)nparts + 1), 256, 0, st>>>((const int32_t*)src, n, nparts, part_offsets);
    QK_LAUNCH_CHECK("k_radix_offsets");
    return QK_OK;
}

extern "C" int qk_partition_plan(const qk_column* key, int32_t nparts, int32_t mode, int32_t* dest,
                                 int64_t* part_offsets, void* workspace, size_t ws_bytes, void* stream) {
    const char* who = "qk_partition_plan";
    if (int rc = check_col(key, who)) return rc;
    if (!dtype_is_int(key->dtype)) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: only integer keys are supported (the reference pins `key %% n` for ints only)", who);
    if (mode != QK_PART_MOD && mode != QK_PART_CODE) QK_FAIL(QK_ERR_INVALID, "%s: bad mode", who);
    if (nparts <= 0 || (mode == QK_PART_MOD && nparts > P_SMEM_PARTS))
        QK_FAIL(QK_ERR_UNSUPPORTED, "%s: nparts must be in [1, %d]%s", who, P_SMEM_PARTS, mode == QK_PART_MOD ? " in MOD mode" : "");
    if (!part_offsets || (key->length > 0 && !dest)) QK_FAIL(QK_ERR_INVALID, "%s: null output", who);
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t n = key->length;
    if (n == 0) {
        QK_CUDA(cudaMemsetAsync(part_offsets, 0, sizeof(int64_t) * ((size_t)nparts + 1), st));
        return QK_OK;
    }
    if (!workspace || ws_bytes < qk_partition_workspace_bytes(n, nparts)) QK_FAIL(QK_ERR_CAPACITY, "%s: workspace too small", who);
    if (nparts > P_SMEM_PARTS) return radix_plan(key, nparts, dest, part_offsets, workspace, st);
    return smem_plan(key, nparts, mode, dest, part_offsets, workspace, st);
}

extern "C" int qk_scatter(const qk_column* cols, int32_t ncols, const int32_t* dest, qk_column* out, void* stream) {
    MoveArgs M;
    if (ncols == 0) return QK_OK;
    if (!cols || !out) QK_FAIL(QK_ERR_INVALID, "qk_scatter: null arguments");
    const int64_t n = cols[0].length;
    if (int rc = fill_move(M, cols, ncols, out, n, n, "qk_scatter")) return rc;
    if (n == 0) return QK_OK;
    if (!dest) QK_FAIL(QK_ERR_INVALID, "qk_scatter: null dest");
    int64_t nb = (n + 255) / 256;
    if (nb > (int64_t)sm_count() * 16) nb = (int64_t)sm_count() * 16;
    k_scatter<<<(unsigned)nb, 256, 0, (cudaStream_t)stream>>>(M, dest, n);
    QK_LAUNCH_CHECK("k_scatter");
    return QK_OK;
}

extern "C" int qk_gather(const qk_column* cols, int32_t ncols, const int32_t* idx, int64_t n_idx, qk_column* out, void* stream) {
    MoveArgs M;
    if (ncols == 0 || n_idx == 0) return QK_OK;
    if (!cols || !out || !idx || n_idx < 0) QK_FAIL(QK_ERR_INVALID, "qk_gather: bad arguments");
    if (int rc = fill_move(M, cols, ncols, out, -1, n_idx, "qk_gather")) return rc;
    int64_t nb = (n_idx + 255) / 256;
    if (nb > (int64_t)sm_count() * 16) nb = (int64_t)sm_count() * 16;
    k_gather<<<(unsigned)nb, 256, 0, (cudaStream_t)stream>>>(M, idx, n_idx);
    QK_LAUNCH_CHECK("k_gather");
    return QK_OK;
}

extern "C" int qk_scatter_peer(const qk_column* cols, int32_t ncols, const int32_t* dest, const int64_t* part_offsets, int32_t nparts,
                               const uint64_t* peer_col_ptrs, const int64_t* peer_row_off, void* stream) {
    const char* who = "qk_scatter_peer";
    if (ncols < 1 || ncols > QK_MAX_COLS || nparts < 1 || nparts > QK_MAX_PEERS) QK_FAIL(QK_ERR_INVALID, "%s: ncols / nparts out of range", who);
    if (!cols || !part_offsets || !peer_col_ptrs || !peer_row_off) QK_FAIL(QK_ERR_INVALID, "%s: null arguments", who);
    static thread_local PeerArgs P;
    const int64_t n = cols[0].length;
    for (int c = 0; c < ncols; ++c) {
        if (int rc = check_col(&cols[c], who)) return rc;
        if (cols[c].length != n) QK_FAIL(QK_ERR_INVALID, "%s: column %d length mismatch", who, c);
        P.src[c] = cols[c].data; P.width[c] = (int8_t)dtype_size(cols[c].dtype);
    }
    for (int p = 0; p < nparts; ++p) {
        P.row_off[p] = peer_row_off[p];
        for (int c = 0; c < ncols; ++c) P.dst[p][c] = peer_col_ptrs[(size_t)p * ncols + c];
    }
    P.ncols = ncols; P.nparts = nparts;
    if (n == 0) return QK_OK;
    if (!dest) QK_FAIL(QK_ERR_INVALID, "%s: null dest", who);
    int64_t nb = (n + 255) / 256;
    if (nb > (int64_t)sm_count() * 16) nb = (int64_t)sm_count() * 16;
    k_scatter_peer<<<(unsigned)nb, 256, 0, (cudaStream_t)stream>>>(P, dest, part_offsets, n);
    QK_LAUNCH_CHECK("k_scatter_peer");
    return QK_OK;
}
