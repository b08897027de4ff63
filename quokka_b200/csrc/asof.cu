// asof.cu -- K7 as-of join by key (SortedAsofExecutor, ts_executors.py:324-383): backward, forward and nearest, with an
// optional tolerance.
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

// What the strategy entry points (qk_asof_join, qk_asof_search_join) do where an answer is written: the nearest pick between
// the backward and the forward candidate (a distance tie goes to the backward one) and the tolerance, |r_time - l_time| <= tol.
// Local right rows are numbered r_base + i; a row below r_base is the backward carry of its key, a row at or past r_base + nr
// the forward carry, and their times come from back_time / fwd_time (int64[n_by]).
struct Pick {
    const long long* r_time; const long long* back_time; const long long* fwd_time;
    long long tol;               // < 0: no tolerance
    int32_t r_base, nr;
    bool nearest;
};
__device__ __forceinline__ unsigned long long time_dist(long long a, long long b) {
    return a < b ? (unsigned long long)b - (unsigned long long)a : (unsigned long long)a - (unsigned long long)b;
}
__device__ __forceinline__ long long row_time(const Pick& p, int32_t row, int key) {
    const int32_t loc = row - p.r_base;
    if ((unsigned)loc < (unsigned)p.nr) return p.r_time[loc];
    return row < p.r_base ? p.back_time[key] : p.fwd_time[key];
}
// back / fwd = the two candidates as rows (-1 none), tb / tf their times
__device__ __forceinline__ int32_t pick_answer(long long t, int32_t back, long long tb, int32_t fwd, long long tf, long long tol) {
    const bool take_back = back >= 0 && (fwd < 0 || time_dist(tb, t) <= time_dist(tf, t));
    const int32_t ans = take_back ? back : fwd;
    if (ans < 0 || tol < 0) return ans;
    return time_dist(take_back ? tb : tf, t) <= (unsigned long long)tol ? ans : -1;
}

// MODE = QK_ASOF_BACKWARD: the LAST right row of the key with r_time <= l_time (upper bound); QK_ASOF_FORWARD: the FIRST one
// with r_time >= l_time (lower bound); QK_ASOF_NEAREST: both neighbours of the upper bound.  PICK: the nearest pick and the
// tolerance `tol` at the write (the backward join of qk_asof_backward has neither).
template <int MODE, bool PICK>
__global__ void __launch_bounds__(256) k_asof_search(const long long* l_time, const int32_t* l_by, int64_t n_left, int n_by,
                                                     const long long* sorted_time, const int32_t* sorted_idx,
                                                     const int64_t* seg, int32_t* out, long long tol) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n_left; i += (int64_t)gridDim.x * blockDim.x) {
        const int b = l_by[i];
        int32_t r = -1;
        if (b >= 0 && b < n_by) {
            const long long t = l_time[i];
            int64_t lo = seg[b], hi = seg[b + 1];
            const int64_t first = lo;
            if constexpr (MODE == QK_ASOF_FORWARD) {
                const int64_t end = hi;
                while (lo < hi) {                   // lower bound: first position with time >= t
                    const int64_t mid = (lo + hi) >> 1;
                    if (sorted_time[mid] < t) lo = mid + 1; else hi = mid;
                }
                if (lo < end) r = PICK ? pick_answer(t, -1, 0, sorted_idx[lo], sorted_time[lo], tol) : sorted_idx[lo];
            } else {
                const int64_t end = hi;
                while (lo < hi) {                   // upper bound: first position with time > t
                    const int64_t mid = (lo + hi) >> 1;
                    if (sorted_time[mid] <= t) lo = mid + 1; else hi = mid;
                }
                if constexpr (!PICK) {
                    if (lo > first) r = sorted_idx[lo - 1];
                } else {
                    // nearest: no right row at t -> the upper bound is also the lower bound; one at t -> the backward one wins
                    const bool nb = lo > first, nf = MODE == QK_ASOF_NEAREST && lo < end;
                    r = pick_answer(t, nb ? sorted_idx[lo - 1] : -1, nb ? sorted_time[lo - 1] : 0,
                                    nf ? sorted_idx[lo] : -1, nf ? sorted_time[lo] : 0, tol);
                }
            }
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
//
// FWD (the forward join) is the mirror: left rows first on merge-path ties (r_time >= l_time matches), table =
// first[key] = the OLDEST right row at or after the current point, folded with atomicMin (none = INT32_MAX inside the
// kernels), the chunk tables carried back to front, and every CTA walks its windows from the last one.  A left row ranks
// itself by lower bound (`lim` = the window's right rows before it); the slow scan runs forwards from `lim`.  carry_in
// rows must be numbered at or past r_base + nr (newer rows).
constexpr int AS_NT = 256, AS_K = 4, AS_W = AS_NT * AS_K;
constexpr int32_t AS_NONE_FWD = 0x7fffffff;

template <bool FWD>
__global__ void __launch_bounds__(128) k_asof_bounds(const long long* r_time, long long nr, const long long* l_time, long long nl,
                                                     long long nwin, long long* wr, long long* wl) {
    const long long w = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (w > nwin) return;
    const long long total = nr + nl;
    const long long d = w * AS_W < total ? w * AS_W : total;
    long long lo = d > nl ? d - nl : 0, hi = d < nr ? d : nr;
    while (lo < hi) {                                   // merge path: right rows first on ties (FWD: left rows first)
        const long long mid = (lo + hi) >> 1;
        if (FWD ? r_time[mid] < l_time[d - 1 - mid] : r_time[mid] <= l_time[d - 1 - mid]) lo = mid + 1; else hi = mid;
    }
    wr[w] = lo; wl[w] = d - lo;
}

template <bool FWD>
__global__ void __launch_bounds__(AS_NT) k_asof_local(const int32_t* r_by, const long long* wr, long long nwin, long long wpc, int n_by,
                                                      int32_t* tables) {
    extern __shared__ int32_t tab[];
    const int tid = threadIdx.x;
    for (int s = tid; s < n_by; s += AS_NT) tab[s] = FWD ? AS_NONE_FWD : -1;
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
            if ((unsigned)sym[u] < (unsigned)n_by) {
                if constexpr (FWD) atomicMin(&tab[sym[u]], (int32_t)(q0 + u * AS_NT));
                else atomicMax(&tab[sym[u]], (int32_t)(q0 + u * AS_NT));
            }
    }
    __syncthreads();
    int32_t* out = tables + (size_t)blockIdx.x * n_by;
    for (int s = tid; s < n_by; s += AS_NT) out[s] = tab[s];
}

// tables[c][s]: in = newest right row of key s inside chunk c (-1 none); out = newest right row of key s BEFORE chunk c,
// as the caller will see it (local rows + r_base, older rows = carry_in's value).
// FWD: in = oldest right row inside chunk c (AS_NONE_FWD none); out = oldest right row AFTER chunk c, newer rows = carry_in's
// value; chunks from the last to the first; carry_out = the oldest right row of every key (-1 none).
template <bool FWD>
__global__ void __launch_bounds__(256) k_asof_carry(int32_t* tables, int P, int n_by, const int32_t* carry_in, int32_t r_base, int32_t* carry_out) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_by) return;
    int32_t run = carry_in ? carry_in[s] : -1;
    if (FWD && run < 0) run = AS_NONE_FWD;
    for (int c0 = 0; c0 < P; c0 += 8) {                  // 8 loads in flight per thread, then the 8 dependent stores
        int32_t v[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) v[u] = c0 + u < P ? tables[(size_t)(FWD ? P - 1 - (c0 + u) : c0 + u) * n_by + s] : -1;
#pragma unroll
        for (int u = 0; u < 8; ++u)
            if (c0 + u < P) {
                tables[(size_t)(FWD ? P - 1 - (c0 + u) : c0 + u) * n_by + s] = run;
                if (FWD ? v[u] != AS_NONE_FWD : v[u] >= 0) run = v[u] + r_base;
            }
    }
    if (FWD && run == AS_NONE_FWD) run = -1;
    if (carry_out) carry_out[s] = run;
}

// PICK: the answer goes through Pick at the write (tolerance; p.nearest: this is the forward sweep of a nearest join and
// out[] already holds the backward sweep's answers).  The kernel of qk_asof_merge is <false, false>.
template <bool FWD, bool PICK>
__global__ void __launch_bounds__(AS_NT) k_asof_sweep(const long long* __restrict__ r_time, const int32_t* __restrict__ r_by,
                                                      const long long* __restrict__ l_time, const int32_t* __restrict__ l_by,
                                                      const long long* __restrict__ wr, const long long* __restrict__ wl, long long nwin,
                                                      long long wpc, int n_by, const int32_t* __restrict__ tables, int32_t r_base,
                                                      int32_t* __restrict__ out, Pick pk) {
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
    // the window bounds in walking order: (qi0, ti0) and (qi1, ti1) end the current window, (qi2, ti2) ends the next one --
    // read one window ahead.  Backward window w spans right rows [qi0, qi1) and left rows [ti0, ti1); FWD walks from the last
    // window down, so window w spans [qi1, qi0) and [ti1, ti0)
    const long long wa = FWD ? w1 : w0;
    long long qi0 = wr[wa], ti0 = wl[wa], qi1 = wr[FWD ? wa - 1 : wa + 1], ti1 = wl[FWD ? wa - 1 : wa + 1];
    long long qi2 = FWD ? (wa - 2 >= 0 ? wr[wa - 2] : qi1) : (w0 + 2 <= nwin ? wr[w0 + 2] : qi1);
    long long ti2 = FWD ? (wa - 2 >= 0 ? wl[wa - 2] : ti1) : (w0 + 2 <= nwin ? wl[w0 + 2] : ti1);
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
    if (FWD) fetch(qi1, qi0, ti1, ti0); else fetch(qi0, qi1, ti0, ti1);
    __syncthreads();                                                     // the table is loaded
    for (long long w = FWD ? w1 - 1 : w0; FWD ? w >= w0 : w < w1; w += FWD ? -1 : 1) {
        const long long qa = FWD ? qi1 : qi0, ta = FWD ? ti1 : ti0;      // the window's first right and left rows
        const int nq = (int)(FWD ? qi0 - qi1 : qi1 - qi0), n = nq + (int)(FWD ? ti0 - ti1 : ti1 - ti0);
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
        if (FWD ? w - 1 >= w0 : w + 1 < w1) {                            // the next window's rows start their way now
            if (FWD ? w - 2 >= 0 : w + 3 <= nwin) { qi3 = wr[FWD ? w - 2 : w + 3]; ti3 = wl[FWD ? w - 2 : w + 3]; }
            if (FWD) fetch(qi2, qi1, ti2, ti1); else fetch(qi1, qi2, ti1, ti2);
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
                while (lo < hi) { const int mid = (lo + hi) >> 1; if (FWD ? bt[mid] < T : bt[mid] <= T) lo = mid + 1; else hi = mid; }
                lim[k] = lo;
            }
        }
        __syncthreads();                                                 // every left row has read the table of before the window
#pragma unroll
        for (int k = 0; k < AS_K; ++k) {
            const int i = tid + k * AS_NT;
            if (i < nq && (unsigned)cs[k] < (unsigned)n_by) {
                if constexpr (FWD) atomicMin(&tab[cs[k]], (int32_t)(qa + i) + r_base);
                else atomicMax(&tab[cs[k]], (int32_t)(qa + i) + r_base);
            }
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
                    // ... its newest one precedes this left row (FWD: its oldest one follows it)
                    if (FWD ? a1 - r_base - (int32_t)qa >= lim[k] : a1 - r_base - (int32_t)qa < lim[k]) ans = a1;
                    else slow = true;                                    // ... it does not: is there another one?
                }
            }
            unsigned todo = __ballot_sync(0xffffffffu, slow);
            while (todo) {
                const int src = __ffs(todo) - 1;
                todo &= todo - 1;
                const int key = __shfl_sync(0xffffffffu, cs[k], src);
                const int top = __shfl_sync(0xffffffffu, lim[k], src);
                if constexpr (FWD) {
                    int found = AS_NONE_FWD;
                    for (int b = top >> 7; (b << 7) < nq && found == AS_NONE_FWD; ++b) {   // 128 keys per step, oldest block first
                        const int i0 = (b << 7) + (lane << 2);
                        const int4 v = *reinterpret_cast<const int4*>(bs + i0);      // slots outside [top, nq) are masked
                        int best = AS_NONE_FWD;
                        if (v.w == key && i0 + 3 >= top && i0 + 3 < nq) best = i0 + 3;
                        if (v.z == key && i0 + 2 >= top && i0 + 2 < nq) best = i0 + 2;
                        if (v.y == key && i0 + 1 >= top && i0 + 1 < nq) best = i0 + 1;
                        if (v.x == key && i0 >= top && i0 < nq) best = i0;
                        found = __reduce_min_sync(0xffffffffu, best);
                    }
                    if (lane == src && found != AS_NONE_FWD) ans = (int32_t)qa + found + r_base;
                } else {
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
                    if (lane == src && found >= 0) ans = (int32_t)qa + found + r_base;
                }
            }
            if (FWD && ans == AS_NONE_FWD) ans = -1;
            if (left) {
                int32_t* o = out + ta + (i - nq);
                if constexpr (PICK) {
                    const int kk = cs[k];
                    const long long T = ct[k];
                    const int32_t back = FWD ? (pk.nearest ? *o : -1) : ans, fwd = FWD ? ans : -1;
                    ans = pick_answer(T, back, back >= 0 ? row_time(pk, back, kk) : 0, fwd, fwd >= 0 ? row_time(pk, fwd, kk) : 0, pk.tol);
                }
                *o = ans;
            }
        }
        qi0 = qi1; ti0 = ti1; qi1 = qi2; ti1 = ti2; qi2 = qi3; ti2 = ti3;
    }
}

// the backward path's workspace: the right rows' partition destinations, the key segments, the right rows in key order
// (time, row number), then the partition's own workspace
struct AsofWs {
    int32_t* dest; int64_t* seg; long long* sorted_time; int32_t* sorted_idx; void* part; size_t part_bytes, bytes;
    AsofWs(int64_t n_right, int32_t n_by, void* base) : part_bytes(qk_partition_workspace_bytes(n_right, n_by)) {
        Carve c(base);
        dest = c.take<int32_t>(n_right);
        seg = c.take<int64_t>((size_t)(n_by + 1));
        sorted_time = c.take<long long>(n_right);
        sorted_idx = c.take<int32_t>(n_right);
        part = c.take<char>(part_bytes);
        bytes = c.bytes;
    }
};

// the merge's workspace: the bounds of every window (wr[nwin + 1], then wl[nwin + 1]), then one key table per chunk
struct AsofMergeWs {
    long long* bounds; int32_t* tables; size_t bytes;
    AsofMergeWs(int64_t nwin, int P, int32_t n_by, void* base) {
        Carve c(base);
        bounds = c.take<long long>((size_t)(nwin + 1) * 2);
        tables = c.take<int32_t>((size_t)P * n_by);
        bytes = c.bytes;
    }
};

}  // namespace
}  // namespace qk

using namespace qk;

static int check_asof_inputs(const qk_column* l_time, const qk_column* l_by, const qk_column* r_time, const qk_column* r_by,
                             int32_t n_by, const char* who) {
    if (int rc = check_col(l_time, who)) return rc;
    if (int rc = check_col(l_by, who)) return rc;
    if (int rc = check_col(r_time, who)) return rc;
    if (int rc = check_col(r_by, who)) return rc;
    if (l_time->dtype != QK_I64 || r_time->dtype != QK_I64) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: time columns must be int64", who);
    if (l_by->dtype != QK_I32 || r_by->dtype != QK_I32) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: by columns must be dense int32 codes", who);
    if (l_time->length != l_by->length || r_time->length != r_by->length) QK_FAIL(QK_ERR_INVALID, "%s: time / by length mismatch", who);
    if (n_by <= 0) QK_FAIL(QK_ERR_INVALID, "%s: n_by must be positive", who);
    return QK_OK;
}

static bool valid_strategy(int32_t s) { return s == QK_ASOF_BACKWARD || s == QK_ASOF_FORWARD || s == QK_ASOF_NEAREST; }

extern "C" size_t qk_asof_workspace_bytes(int64_t n_right, int32_t n_by) {
    if (n_right < 0 || n_by <= 0) return 0;
    return AsofWs(n_right, n_by, nullptr).bytes;
}

// the partition + search join: qk_asof_backward (strategy backward, no pick) and qk_asof_search_join
static int asof_search_join(const qk_column* l_time, const qk_column* l_by, const qk_column* r_time, const qk_column* r_by,
                            int32_t n_by, int32_t strategy, int64_t tolerance, bool pick, int32_t* out_ridx, void* workspace,
                            size_t ws_bytes, void* stream, const char* who) {
    if (int rc = check_asof_inputs(l_time, l_by, r_time, r_by, n_by, who)) return rc;
    const int64_t nl = l_time->length, nr = r_time->length;
    if (nl == 0) return QK_OK;
    if (!out_ridx) QK_FAIL(QK_ERR_INVALID, "%s: null output", who);
    const AsofWs w(nr, n_by, workspace);
    if (!workspace || ws_bytes < w.bytes) QK_FAIL(QK_ERR_CAPACITY, "%s: workspace too small", who);
    if (int rc = qk_partition_plan(r_by, n_by, QK_PART_CODE, w.dest, w.seg, w.part, w.part_bytes, stream)) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    if (nr > 0) {
        k_asof_prepare<<<grid_size(nr, 16), 256, 0, st>>>((const long long*)r_time->data, w.dest, nr, w.sorted_time, w.sorted_idx);
        QK_LAUNCH_CHECK("k_asof_prepare");
    }
    const long long* lt = (const long long*)l_time->data;
    const int32_t* lb = (const int32_t*)l_by->data;
    const unsigned grid = grid_size(nl, 16);
    const long long tol = tolerance;
    if (!pick) k_asof_search<QK_ASOF_BACKWARD, false><<<grid, 256, 0, st>>>(lt, lb, nl, n_by, w.sorted_time, w.sorted_idx, w.seg, out_ridx, tol);
    else if (strategy == QK_ASOF_BACKWARD) k_asof_search<QK_ASOF_BACKWARD, true><<<grid, 256, 0, st>>>(lt, lb, nl, n_by, w.sorted_time, w.sorted_idx, w.seg, out_ridx, tol);
    else if (strategy == QK_ASOF_FORWARD) k_asof_search<QK_ASOF_FORWARD, true><<<grid, 256, 0, st>>>(lt, lb, nl, n_by, w.sorted_time, w.sorted_idx, w.seg, out_ridx, tol);
    else k_asof_search<QK_ASOF_NEAREST, true><<<grid, 256, 0, st>>>(lt, lb, nl, n_by, w.sorted_time, w.sorted_idx, w.seg, out_ridx, tol);
    QK_LAUNCH_CHECK("k_asof_search");
    return QK_OK;
}

extern "C" int qk_asof_backward(const qk_column* l_time, const qk_column* l_by, const qk_column* r_time,
                                const qk_column* r_by, int32_t n_by, int32_t* out_ridx, void* workspace,
                                size_t ws_bytes, void* stream) {
    return asof_search_join(l_time, l_by, r_time, r_by, n_by, QK_ASOF_BACKWARD, -1, false, out_ridx, workspace, ws_bytes, stream,
                            "qk_asof_backward");
}

extern "C" int qk_asof_search_join(const qk_column* l_time, const qk_column* l_by, const qk_column* r_time, const qk_column* r_by,
                                   int32_t n_by, int32_t strategy, int64_t tolerance, int32_t* out_ridx, void* workspace,
                                   size_t ws_bytes, void* stream) {
    const char* who = "qk_asof_search_join";
    if (!valid_strategy(strategy)) QK_FAIL(QK_ERR_INVALID, "%s: unknown strategy %d", who, strategy);
    return asof_search_join(l_time, l_by, r_time, r_by, n_by, strategy, tolerance < 0 ? -1 : tolerance, true, out_ridx, workspace,
                            ws_bytes, stream, who);
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
    return AsofMergeWs(asof_windows(n_left + n_right), P, n_by, nullptr).bytes;
}

// One direction of the merge join over a laid-out workspace: bounds, chunk tables, carry, sweep.  Nearest runs it twice over
// the same workspace (on one stream): backward into out_ridx, then forward, which picks between the two at the write.
template <bool FWD, bool PICK>
static int asof_merge_pass(const qk_column* l_time, const qk_column* l_by, const qk_column* r_time, const qk_column* r_by,
                           int32_t n_by, const int32_t* carry_in, int32_t r_base, int32_t* carry_out, int32_t* out_ridx,
                           const AsofMergeWs& w, int64_t nwin, int P0, size_t smem, const Pick& pk, cudaStream_t st) {
    const int64_t nl = l_time->length, nr = r_time->length;
    const int64_t wpc = (nwin + P0 - 1) / P0;                      // windows per chunk (CTA)
    const int P = (int)((nwin + wpc - 1) / wpc);                   // chunks that have a window: <= P0
    long long* wr = w.bounds;
    long long* wl = wr + (nwin + 1);
    int32_t* tables = w.tables;
    k_asof_bounds<FWD><<<(unsigned)((nwin + 1 + 127) / 128), 128, 0, st>>>((const long long*)r_time->data, nr, (const long long*)l_time->data, nl, nwin, wr, wl);
    QK_LAUNCH_CHECK("k_asof_bounds");
    const size_t table_bytes = align_up((size_t)n_by * 4, 16);
    QK_CUDA(qk::raise_smem_limit((const void*)k_asof_local<FWD>, (size_t)table_bytes));
    QK_CUDA(qk::raise_smem_limit((const void*)k_asof_sweep<FWD, PICK>, (size_t)smem));
    k_asof_local<FWD><<<P, AS_NT, table_bytes, st>>>((const int32_t*)r_by->data, wr, nwin, wpc, n_by, tables);
    QK_LAUNCH_CHECK("k_asof_local");
    k_asof_carry<FWD><<<(n_by + 255) / 256, 256, 0, st>>>(tables, P, n_by, carry_in, r_base, carry_out);
    QK_LAUNCH_CHECK("k_asof_carry");
    if (nl == 0) return QK_OK;                                      // no left rows: the caller wanted the table only (carry_out)
    k_asof_sweep<FWD, PICK><<<P, AS_NT, smem, st>>>((const long long*)r_time->data, (const int32_t*)r_by->data, (const long long*)l_time->data,
                                                   (const int32_t*)l_by->data, wr, wl, nwin, wpc, n_by, tables, r_base, out_ridx, pk);
    QK_LAUNCH_CHECK("k_asof_sweep");
    return QK_OK;
}

// checks and workspace of the merge join; P0 = 0 when the keys do not fit the shared-memory table
static int asof_merge_setup(const qk_column* l_time, const qk_column* l_by, const qk_column* r_time, const qk_column* r_by,
                            int32_t n_by, int32_t r_base, int32_t* out_ridx, void* workspace, size_t ws_bytes, const char* who,
                            AsofMergeWs* w, int64_t* nwin, int* P0, size_t* smem) {
    if (int rc = check_asof_inputs(l_time, l_by, r_time, r_by, n_by, who)) return rc;
    const int64_t nl = l_time->length, nr = r_time->length;
    if (r_base < 0 || (int64_t)r_base + nr > 0x7fffffffLL) QK_FAIL(QK_ERR_INVALID, "%s: right row numbers exceed int32", who);
    *P0 = asof_merge_chunks(n_by, smem);
    if (*P0 == 0) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: %d keys do not fit a shared-memory table; use the search join", who, n_by);
    if (nl > 0 && !out_ridx) QK_FAIL(QK_ERR_INVALID, "%s: null output", who);
    *nwin = asof_windows(nl + nr);
    *w = AsofMergeWs(*nwin, *P0, n_by, workspace);
    if (!workspace || ws_bytes < w->bytes) QK_FAIL(QK_ERR_CAPACITY, "%s: workspace too small", who);
    return QK_OK;
}

extern "C" int qk_asof_merge(const qk_column* l_time, const qk_column* l_by, const qk_column* r_time, const qk_column* r_by,
                             int32_t n_by, const int32_t* carry_in, int32_t r_base, int32_t* carry_out, int32_t* out_ridx,
                             void* workspace, size_t ws_bytes, void* stream) {
    AsofMergeWs w(0, 0, 0, nullptr);
    int64_t nwin;
    int P0;
    size_t smem = 0;
    if (int rc = asof_merge_setup(l_time, l_by, r_time, r_by, n_by, r_base, out_ridx, workspace, ws_bytes, "qk_asof_merge", &w, &nwin, &P0, &smem))
        return rc;
    return asof_merge_pass<false, false>(l_time, l_by, r_time, r_by, n_by, carry_in, r_base, carry_out, out_ridx, w, nwin, P0, smem, Pick{},
                                         (cudaStream_t)stream);
}

extern "C" size_t qk_asof_join_workspace_bytes(int64_t n_left, int64_t n_right, int32_t n_by, int32_t strategy) {
    return valid_strategy(strategy) ? qk_asof_merge_workspace_bytes(n_left, n_right, n_by) : 0;
}

extern "C" int qk_asof_join(const qk_column* l_time, const qk_column* l_by, const qk_column* r_time, const qk_column* r_by,
                            int32_t n_by, int32_t strategy, int64_t tolerance, const int32_t* carry_back,
                            const int64_t* carry_back_time, const int32_t* carry_fwd, const int64_t* carry_fwd_time, int32_t r_base,
                            int32_t* carry_out, int32_t* out_ridx, void* workspace, size_t ws_bytes, void* stream) {
    const char* who = "qk_asof_join";
    if (!valid_strategy(strategy)) QK_FAIL(QK_ERR_INVALID, "%s: unknown strategy %d", who, strategy);
    if ((carry_back && !carry_back_time) || (carry_fwd && !carry_fwd_time)) QK_FAIL(QK_ERR_INVALID, "%s: a carry table without its times", who);
    if (strategy == QK_ASOF_NEAREST && carry_out) QK_FAIL(QK_ERR_INVALID, "%s: a nearest join has no carry_out", who);
    if ((strategy == QK_ASOF_BACKWARD && carry_fwd) || (strategy == QK_ASOF_FORWARD && carry_back))
        QK_FAIL(QK_ERR_INVALID, "%s: a carry table of the other direction", who);
    AsofMergeWs w(0, 0, 0, nullptr);
    int64_t nwin;
    int P0;
    size_t smem = 0;
    if (int rc = asof_merge_setup(l_time, l_by, r_time, r_by, n_by, r_base, out_ridx, workspace, ws_bytes, who, &w, &nwin, &P0, &smem))
        return rc;
    const int64_t nr = r_time->length;
    Pick pk{(const long long*)r_time->data, (const long long*)carry_back_time, (const long long*)carry_fwd_time,
            tolerance < 0 ? -1 : (long long)tolerance, r_base, (int32_t)nr, strategy == QK_ASOF_NEAREST};
    cudaStream_t st = (cudaStream_t)stream;
    if (strategy == QK_ASOF_BACKWARD)
        return asof_merge_pass<false, true>(l_time, l_by, r_time, r_by, n_by, carry_back, r_base, carry_out, out_ridx, w, nwin, P0, smem, pk, st);
    if (strategy == QK_ASOF_NEAREST) {
        if (l_time->length == 0) return QK_OK;
        if (int rc = asof_merge_pass<false, false>(l_time, l_by, r_time, r_by, n_by, carry_back, r_base, nullptr, out_ridx, w, nwin, P0, smem,
                                                   pk, st))
            return rc;
    }
    return asof_merge_pass<true, true>(l_time, l_by, r_time, r_by, n_by, carry_fwd, r_base, carry_out, out_ridx, w, nwin, P0, smem, pk, st);
}
