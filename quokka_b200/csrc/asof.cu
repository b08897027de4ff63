// asof.cu -- K7 backward as-of join by key (SortedAsofExecutor, ts_executors.py:324-383).
//
// Both inputs are time-sorted.  The right side is segmented by its `by` code with the STABLE partition
// of partition.cu (time order survives inside a segment, so no sort is needed), then every left row does
// an upper-bound binary search inside its key's segment: the LAST right row with r_time <= l_time, the
// tie rule of Polars / pandas.  HBM-bound: right side read + written once (time 8 B + index 4 B per row),
// left side 12 B/row read + 4 B/row written, plus ~log2(segment) cached probes per left row; neighbouring
// left rows of one key search neighbouring positions, so the probes hit L2.
#include "common.cuh"

namespace qk {
namespace {

__global__ void __launch_bounds__(256) k_asof_prepare(const long long* r_time, const int32_t* dest, int64_t n,
                                                      long long* sorted_time, int32_t* sorted_idx) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int32_t d = dest[i];
        sorted_time[d] = r_time[i];
        sorted_idx[d] = (int32_t)i;
    }
}

__global__ void __launch_bounds__(256) k_asof_search(const long long* l_time, const int32_t* l_by, int64_t n_left, int n_by,
                                                     const long long* sorted_time, const int32_t* sorted_idx,
                                                     const int64_t* seg, int32_t* out) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n_left; i += (int64_t)gridDim.x * blockDim.x) {
        const int b = l_by[i];
        int32_t r = -1;
        if (b >= 0 && b < n_by) {
            const long long t = l_time[i];
            int64_t lo = seg[b], hi = seg[b + 1];
            const int64_t first = lo;
            while (lo < hi) {                       // upper bound: first position with time > t
                const int64_t mid = (lo + hi) >> 1;
                if (sorted_time[mid] <= t) lo = mid + 1; else hi = mid;
            }
            if (lo > first) r = sorted_idx[lo - 1];
        }
        out[i] = r;
    }
}


// ================================================================================================================
// Sorted-merge as-of (the default when the per-key table fits shared memory).  Both inputs are time-sorted, so the
// join is one sweep over the merged timeline carrying last[key] = row of the newest right row of every key:
// a right row updates its entry, a left row reads it.  The timeline is cut into WINDOWS of AS_W merged rows
// (merge-path diagonals, right rows first on ties: r_time <= l_time matches); a CTA owns a contiguous run of windows (a
// chunk) and keeps its table in shared memory:
//   1  k_asof_bounds   one diagonal per window -> (right, left) split points
//   2  k_asof_local    every CTA folds its chunk's RIGHT keys -> newest right row per key inside the chunk (atomicMax: row
//                      numbers grow with time)
//   3  k_asof_carry    one thread per key folds the chunk tables front to back -> the table valid at each chunk's start
//   4  k_asof_sweep    every CTA walks its windows.  Per window, all 256 threads at once:
//                        a  the window's rows (right rows first, then left rows) go to shared memory, the next window's
//                           loads are already in flight in registers
//                        b  every left row reads table[key] (= newest row BEFORE the window) and ranks itself among the window's
//                           right rows (binary search in shared memory): `lim` = how many of them precede it
//                        c  every right row does atomicMax(table[key], row)
//                        d  every left row reads table[key] again: unchanged -> no right row of its key in this window, the
//                           old value is the answer; changed and the new row ranks below `lim` -> that row; else (the key's
//                           newest row of the window comes AFTER this left row, ~1 % of left rows) the warp scans the
//                           window's keys backwards from `lim`, 128 at a time, for an earlier one
// The first version of this sweep gave every WARP a chunk and a private table: 6 warps per SM, 12 shuffles of binary search
// and a serial loop over the left rows per 32-row step -- latency-bound.
// No sort, no scatter: reads 12 B per right row + 4 B again in step 2, 12 B per left row, writes 4 B per left row.
// Row numbers in the table are the caller's (local row + r_base); carry_in must hold rows below r_base (older rows).
constexpr int AS_NT = 256, AS_K = 4, AS_W = AS_NT * AS_K;

__global__ void __launch_bounds__(128) k_asof_bounds(const long long* r_time, long long nr, const long long* l_time, long long nl,
                                                     long long nwin, long long* wr, long long* wl) {
    const long long w = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (w > nwin) return;
    const long long total = nr + nl;
    const long long d = w * AS_W < total ? w * AS_W : total;
    long long lo = d > nl ? d - nl : 0, hi = d < nr ? d : nr;
    while (lo < hi) {                                   // merge path: right rows first on ties
        const long long mid = (lo + hi) >> 1;
        if (r_time[mid] <= l_time[d - 1 - mid]) lo = mid + 1; else hi = mid;
    }
    wr[w] = lo; wl[w] = d - lo;
}

__global__ void __launch_bounds__(AS_NT) k_asof_local(const int32_t* r_by, const long long* wr, long long nwin, long long wpc, int n_by,
                                                      int32_t* tables) {
    extern __shared__ int32_t tab[];
    const int tid = threadIdx.x;
    for (int s = tid; s < n_by; s += AS_NT) tab[s] = -1;
    __syncthreads();
    long long w0 = (long long)blockIdx.x * wpc; if (w0 > nwin) w0 = nwin;
    long long w1 = w0 + wpc; if (w1 > nwin) w1 = nwin;
    const long long qa = wr[w0], qb = wr[w1];
    for (long long q0 = qa + tid; q0 < qb; q0 += AS_NT * 8) {          // 8 independent loads per thread in flight
        int sym[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) { const long long q = q0 + u * AS_NT; sym[u] = q < qb ? r_by[q] : -1; }
#pragma unroll
        for (int u = 0; u < 8; ++u)
            if ((unsigned)sym[u] < (unsigned)n_by) atomicMax(&tab[sym[u]], (int32_t)(q0 + u * AS_NT));
    }
    __syncthreads();
    int32_t* out = tables + (size_t)blockIdx.x * n_by;
    for (int s = tid; s < n_by; s += AS_NT) out[s] = tab[s];
}

// tables[c][s]: in = newest right row of key s inside chunk c (-1 none); out = newest right row of key s BEFORE chunk c,
// as the caller will see it (local rows + r_base, older rows = carry_in's value)
__global__ void __launch_bounds__(256) k_asof_carry(int32_t* tables, int P, int n_by, const int32_t* carry_in, int32_t r_base, int32_t* carry_out) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_by) return;
    int32_t run = carry_in ? carry_in[s] : -1;
    for (int c0 = 0; c0 < P; c0 += 8) {                  // 8 loads in flight per thread, then the 8 dependent stores
        int32_t v[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) v[u] = c0 + u < P ? tables[(size_t)(c0 + u) * n_by + s] : -1;
#pragma unroll
        for (int u = 0; u < 8; ++u)
            if (c0 + u < P) {
                tables[(size_t)(c0 + u) * n_by + s] = run;
                if (v[u] >= 0) run = v[u] + r_base;
            }
    }
    if (carry_out) carry_out[s] = run;
}

__global__ void __launch_bounds__(AS_NT) k_asof_sweep(const long long* __restrict__ r_time, const int32_t* __restrict__ r_by,
                                                      const long long* __restrict__ l_time, const int32_t* __restrict__ l_by,
                                                      const long long* __restrict__ wr, const long long* __restrict__ wl, long long nwin,
                                                      long long wpc, int n_by, const int32_t* __restrict__ tables, int32_t r_base,
                                                      int32_t* __restrict__ out) {
    extern __shared__ __align__(16) unsigned char as_smem[];
    long long* wtime = (long long*)as_smem;                              // [2][AS_W] the window's times: right rows, then left rows
    int32_t* wsym = (int32_t*)(as_smem + 2 * AS_W * 8);                  // [2][AS_W] their keys
    int32_t* tab = (int32_t*)(as_smem + 2 * AS_W * 12);                  // [n_by]
    const int tid = threadIdx.x, lane = tid & 31;
    const int32_t* before = tables + (size_t)blockIdx.x * n_by;
    for (int s = tid; s < n_by; s += AS_NT) tab[s] = before[s];
    long long w0 = (long long)blockIdx.x * wpc; if (w0 > nwin) w0 = nwin;
    long long w1 = w0 + wpc; if (w1 > nwin) w1 = nwin;
    if (w0 >= w1) return;                                                // (uniform over the CTA)
    // window w spans right rows [qi0, qi1) and left rows [ti0, ti1); (qi2, ti2) ends window w + 1 -- read one window ahead
    long long qi0 = wr[w0], ti0 = wl[w0], qi1 = wr[w0 + 1], ti1 = wl[w0 + 1];
    long long qi2 = w0 + 2 <= nwin ? wr[w0 + 2] : qi1, ti2 = w0 + 2 <= nwin ? wl[w0 + 2] : ti1;
    long long nt_[AS_K];
    int ns_[AS_K];
    auto fetch = [&](long long qa, long long qb, long long ta, long long tb) {     // slot i: right row qa + i, then left row ta + (i - nq)
        const int nq = (int)(qb - qa), n = nq + (int)(tb - ta);
#pragma unroll
        for (int k = 0; k < AS_K; ++k) {
            const int i = tid + k * AS_NT;
            nt_[k] = 0; ns_[k] = -1;
            if (i < nq) { nt_[k] = r_time[qa + i]; ns_[k] = r_by[qa + i]; }
            else if (i < n) { nt_[k] = l_time[ta + (i - nq)]; ns_[k] = l_by[ta + (i - nq)]; }
        }
    };
    fetch(qi0, qi1, ti0, ti1);
    __syncthreads();                                                     // the table is loaded
    for (long long w = w0; w < w1; ++w) {
        const int nq = (int)(qi1 - qi0), n = nq + (int)(ti1 - ti0);
        const int buf = (int)((w - w0) & 1);
        long long* bt = wtime + buf * AS_W;
        int32_t* bs = wsym + buf * AS_W;
        long long ct[AS_K];
        int cs[AS_K];
#pragma unroll
        for (int k = 0; k < AS_K; ++k) {
            const int i = tid + k * AS_NT;
            ct[k] = nt_[k]; cs[k] = ns_[k];
            if (i < n) { bt[i] = ct[k]; bs[i] = cs[k]; }
        }
        long long qi3 = qi2, ti3 = ti2;
        if (w + 1 < w1) {                                                // the next window's rows start their way now
            if (w + 3 <= nwin) { qi3 = wr[w + 3]; ti3 = wl[w + 3]; }
            fetch(qi1, qi2, ti1, ti2);
        }
        __syncthreads();                                                 // window staged
        int a0[AS_K], lim[AS_K];
#pragma unroll
        for (int k = 0; k < AS_K; ++k) {
            const int i = tid + k * AS_NT;
            a0[k] = -1; lim[k] = 0;
            if (i >= nq && i < n && (unsigned)cs[k] < (unsigned)n_by) {
                a0[k] = tab[cs[k]];
                int lo = 0, hi = nq;
                const long long T = ct[k];
                while (lo < hi) { const int mid = (lo + hi) >> 1; if (bt[mid] <= T) lo = mid + 1; else hi = mid; }
                lim[k] = lo;
            }
        }
        __syncthreads();                                                 // every left row has read the table of before the window
#pragma unroll
        for (int k = 0; k < AS_K; ++k) {
            const int i = tid + k * AS_NT;
            if (i < nq && (unsigned)cs[k] < (unsigned)n_by) atomicMax(&tab[cs[k]], (int32_t)(qi0 + i) + r_base);
        }
        __syncthreads();                                                 // the table of after the window
#pragma unroll
        for (int k = 0; k < AS_K; ++k) {
            const int i = tid + k * AS_NT;
            const bool left = i >= nq && i < n;
            int ans = -1;
            bool slow = false;
            if (left && (unsigned)cs[k] < (unsigned)n_by) {
                const int a1 = tab[cs[k]];
                ans = a0[k];
                if (a1 != a0[k]) {                                       // a right row of this key inside the window
                    if (a1 - r_base - (int32_t)qi0 < lim[k]) ans = a1;   // ... its newest one precedes this left row
                    else slow = true;                                    // ... it follows: is there an earlier one?
                }
            }
            unsigned todo = __ballot_sync(0xffffffffu, slow);
            while (todo) {
                const int src = __ffs(todo) - 1;
                todo &= todo - 1;
                const int key = __shfl_sync(0xffffffffu, cs[k], src);
                const int top = __shfl_sync(0xffffffffu, lim[k], src);
                int found = -1;
                for (int b = (top - 1) >> 7; b >= 0 && found < 0; --b) {      // 128 keys per step (one 16-byte read per lane), newest block first
                    const int i0 = (b << 7) + (lane << 2);
                    const int4 v = *reinterpret_cast<const int4*>(bs + i0);   // slots past the window's right rows are masked by `top`
                    int best = -1;
                    if (v.x == key && i0 < top) best = i0;
                    if (v.y == key && i0 + 1 < top) best = i0 + 1;
                    if (v.z == key && i0 + 2 < top) best = i0 + 2;
                    if (v.w == key && i0 + 3 < top) best = i0 + 3;
                    found = __reduce_max_sync(0xffffffffu, best);
                }
                if (lane == src && found >= 0) ans = (int32_t)qi0 + found + r_base;
            }
            if (left) out[ti0 + (i - nq)] = ans;
        }
        qi0 = qi1; ti0 = ti1; qi1 = qi2; ti1 = ti2; qi2 = qi3; ti2 = ti3;
    }
}

}  // namespace
}  // namespace qk

using namespace qk;

static size_t asof_fixed_bytes(int64_t n_right, int32_t n_by) {
    return align_up((size_t)n_right * 4, 256)            // dest
         + align_up((size_t)(n_by + 1) * 8, 256)         // segment offsets
         + align_up((size_t)n_right * 8, 256)            // sorted_time
         + align_up((size_t)n_right * 4, 256);           // sorted_idx
}

extern "C" size_t qk_asof_workspace_bytes(int64_t n_right, int32_t n_by) {
    if (n_right < 0 || n_by <= 0) return 0;
    return asof_fixed_bytes(n_right, n_by) + qk_partition_workspace_bytes(n_right, n_by);
}

extern "C" int qk_asof_backward(const qk_column* l_time, const qk_column* l_by, const qk_column* r_time,
                                const qk_column* r_by, int32_t n_by, int32_t* out_ridx, void* workspace,
                                size_t ws_bytes, void* stream) {
    const char* who = "qk_asof_backward";
    if (int rc = check_col(l_time, who)) return rc;
    if (int rc = check_col(l_by, who)) return rc;
    if (int rc = check_col(r_time, who)) return rc;
    if (int rc = check_col(r_by, who)) return rc;
    if (l_time->dtype != QK_I64 || r_time->dtype != QK_I64) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: time columns must be int64", who);
    if (l_by->dtype != QK_I32 || r_by->dtype != QK_I32) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: by columns must be dense int32 codes", who);
    if (l_time->length != l_by->length || r_time->length != r_by->length) QK_FAIL(QK_ERR_INVALID, "%s: time / by length mismatch", who);
    if (n_by <= 0) QK_FAIL(QK_ERR_INVALID, "%s: n_by must be positive", who);
    const int64_t nl = l_time->length, nr = r_time->length;
    if (nl == 0) return QK_OK;
    if (!out_ridx) QK_FAIL(QK_ERR_INVALID, "%s: null output", who);
    if (!workspace || ws_bytes < qk_asof_workspace_bytes(nr, n_by)) QK_FAIL(QK_ERR_CAPACITY, "%s: workspace too small", who);
    char* w = (char*)workspace;
    int32_t* dest = (int32_t*)w; w += align_up((size_t)nr * 4, 256);
    int64_t* seg = (int64_t*)w; w += align_up((size_t)(n_by + 1) * 8, 256);
    long long* sorted_time = (long long*)w; w += align_up((size_t)nr * 8, 256);
    int32_t* sorted_idx = (int32_t*)w; w += align_up((size_t)nr * 4, 256);
    if (int rc = qk_partition_plan(r_by, n_by, QK_PART_CODE, dest, seg, w, ws_bytes - asof_fixed_bytes(nr, n_by), stream)) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    const int cap = sm_count() * 16;
    if (nr > 0) {
        int64_t nb = (nr + 255) / 256; if (nb > cap) nb = cap;
        k_asof_prepare<<<(unsigned)nb, 256, 0, st>>>((const long long*)r_time->data, dest, nr, sorted_time, sorted_idx);
        QK_LAUNCH_CHECK("k_asof_prepare");
    }
    int64_t nb = (nl + 255) / 256; if (nb > cap) nb = cap;
    k_asof_search<<<(unsigned)nb, 256, 0, st>>>((const long long*)l_time->data, (const int32_t*)l_by->data, nl, n_by,
                                                sorted_time, sorted_idx, seg, out_ridx);
    QK_LAUNCH_CHECK("k_asof_search");
    return QK_OK;
}

// ---- sorted-merge as-of ------------------------------------------------------------------------------------------
static int asof_merge_chunks(int32_t n_by, size_t* smem_out) {
    const size_t table = align_up((size_t)n_by * 4, 16);
    if (table > 160 * 1024) return 0;                              // table too large for shared memory: partition path
    const size_t smem = (size_t)2 * AS_W * 12 + table;
    int per_sm = (int)((228 * 1024) / (smem + 1024));
    if (per_sm > 8) per_sm = 8;
    if (per_sm < 1) per_sm = 1;
    *smem_out = smem;
    return sm_count() * per_sm;
}
static int64_t asof_windows(int64_t total) { return total > 0 ? (total + AS_W - 1) / AS_W : 1; }

extern "C" size_t qk_asof_merge_workspace_bytes(int64_t n_left, int64_t n_right, int32_t n_by) {
    size_t smem;
    const int P = n_by > 0 ? asof_merge_chunks(n_by, &smem) : 0;
    if (P == 0 || n_left < 0 || n_right < 0) return 0;
    return align_up((size_t)(asof_windows(n_left + n_right) + 1) * 16, 256) + align_up((size_t)P * n_by * 4, 256);
}

extern "C" int qk_asof_merge(const qk_column* l_time, const qk_column* l_by, const qk_column* r_time, const qk_column* r_by,
                             int32_t n_by, const int32_t* carry_in, int32_t r_base, int32_t* carry_out, int32_t* out_ridx,
                             void* workspace, size_t ws_bytes, void* stream) {
    const char* who = "qk_asof_merge";
    if (int rc = check_col(l_time, who)) return rc;
    if (int rc = check_col(l_by, who)) return rc;
    if (int rc = check_col(r_time, who)) return rc;
    if (int rc = check_col(r_by, who)) return rc;
    if (l_time->dtype != QK_I64 || r_time->dtype != QK_I64) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: time columns must be int64", who);
    if (l_by->dtype != QK_I32 || r_by->dtype != QK_I32) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: by columns must be dense int32 codes", who);
    if (l_time->length != l_by->length || r_time->length != r_by->length) QK_FAIL(QK_ERR_INVALID, "%s: time / by length mismatch", who);
    if (n_by <= 0) QK_FAIL(QK_ERR_INVALID, "%s: n_by must be positive", who);
    const int64_t nl = l_time->length, nr = r_time->length;
    if (r_base < 0 || (int64_t)r_base + nr > 0x7fffffffLL) QK_FAIL(QK_ERR_INVALID, "%s: right row numbers exceed int32", who);
    size_t smem = 0;
    const int P0 = asof_merge_chunks(n_by, &smem);
    if (P0 == 0) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: %d keys do not fit a shared-memory table; use qk_asof_backward", who, n_by);
    if (nl > 0 && !out_ridx) QK_FAIL(QK_ERR_INVALID, "%s: null output", who);
    if (!workspace || ws_bytes < qk_asof_merge_workspace_bytes(nl, nr, n_by)) QK_FAIL(QK_ERR_CAPACITY, "%s: workspace too small", who);
    const int64_t nwin = asof_windows(nl + nr);
    const int64_t wpc = (nwin + P0 - 1) / P0;                      // windows per chunk (CTA)
    const int P = (int)((nwin + wpc - 1) / wpc);                   // chunks that have a window: <= P0
    cudaStream_t st = (cudaStream_t)stream;
    long long* wr = (long long*)workspace;
    long long* wl = wr + (nwin + 1);
    int32_t* tables = (int32_t*)((char*)workspace + align_up((size_t)(nwin + 1) * 16, 256));
    k_asof_bounds<<<(unsigned)((nwin + 1 + 127) / 128), 128, 0, st>>>((const long long*)r_time->data, nr, (const long long*)l_time->data, nl, nwin, wr, wl);
    QK_LAUNCH_CHECK("k_asof_bounds");
    const size_t table_bytes = align_up((size_t)n_by * 4, 16);
    QK_CUDA(cudaFuncSetAttribute(k_asof_local, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)table_bytes));
    QK_CUDA(cudaFuncSetAttribute(k_asof_sweep, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_asof_local<<<P, AS_NT, table_bytes, st>>>((const int32_t*)r_by->data, wr, nwin, wpc, n_by, tables);
    QK_LAUNCH_CHECK("k_asof_local");
    k_asof_carry<<<(n_by + 255) / 256, 256, 0, st>>>(tables, P, n_by, carry_in, r_base, carry_out);
    QK_LAUNCH_CHECK("k_asof_carry");
    if (nl == 0) return QK_OK;                                      // no left rows: the caller wanted the table only (carry_out)
    k_asof_sweep<<<P, AS_NT, smem, st>>>((const long long*)r_time->data, (const int32_t*)r_by->data, (const long long*)l_time->data,
                                         (const int32_t*)l_by->data, wr, wl, nwin, wpc, n_by, tables, r_base, out_ridx);
    QK_LAUNCH_CHECK("k_asof_sweep");
    return QK_OK;
}
