// window.cu -- time-series windows over a key-partitioned, time-sorted stream (pyquokka/executors/ts_executors.py:12-288:
// HoppingWindowExecutor / SlidingWindowExecutor / SessionWindowExecutor; the reference delegates to Polars
// groupby_dynamic / groupby_rolling and DuckDB window SQL).  The rows arrive segmented by key with the stable partition of
// partition.cu (time order survives inside a segment), exactly what the as-of path uses; on top of that:
//   sliding  k_win_sliding: every row aggregates the rows of its key with time in (t - size, t] -- lower bound by binary
//            search inside the key's segment, ties at t included, then one pass over the window (SUM / MIN / MAX / COUNT / AVG);
//   hopping  k_win_hop_expand: every row is assigned to the windows [k * hop, k * hop + size) that contain it (one output
//            slot per window, ceil(size / hop) slots per row; windows that start before the key's first truncated timestamp
//            are not produced, like Polars' start_by = "window"); the (key, window start) pairs then go through the hash
//            aggregate of hashagg.cu;
//   session  k_win_session_flag + a prefix sum: a new session starts at a key's first row and after every gap > timeout;
//            the session ids then go through the hash aggregate;
//   running  k_win_run_*: per-event (OnEventTrigger) tumbling and session windows, every row the running aggregate of its
//            window up to its time (see the section comment below).
// HBM-bound except for wide sliding windows, which re-read their rows from L1 / L2.
#include "common.cuh"

namespace qk {
namespace {

struct WinArgs {
    const double* val[QK_MAX_AGGS];
    double* out[2 * QK_MAX_AGGS];
    int8_t op[2 * QK_MAX_AGGS];       // QK_WIN_*
    int8_t src[2 * QK_MAX_AGGS];      // index into val (ignored for COUNT)
    int32_t nout;
};

__global__ void __launch_bounds__(256) k_win_sliding(const long long* time, const int32_t* by, const int64_t* seg, int n_by, int64_t n,
                                                     long long size, const __grid_constant__ WinArgs W) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int b = by[i];
        int64_t s0 = i, s1 = i + 1;
        if (b >= 0 && b < n_by) { s0 = seg[b]; s1 = seg[b + 1]; }
        const long long t = time[i];
        int64_t lo = s0, hi = i;                       // first row of the segment with time > t - size
        while (lo < hi) {
            const int64_t mid = (lo + hi) >> 1;
            if (time[mid] > t - size) hi = mid; else lo = mid + 1;
        }
        int64_t last = i;                              // rows after i with the same timestamp belong to the window too
        while (last + 1 < s1 && time[last + 1] == t) ++last;
        const double cnt = (double)(last - lo + 1);
        for (int o = 0; o < W.nout; ++o) {
            const int op = W.op[o];
            double r;
            if (op == QK_WIN_COUNT) r = cnt;
            else {
                const double* v = W.val[W.src[o]];
                r = v[lo];
                if (op == QK_WIN_MIN) { for (int64_t j = lo + 1; j <= last; ++j) r = fmin(r, v[j]); }
                else if (op == QK_WIN_MAX) { for (int64_t j = lo + 1; j <= last; ++j) r = fmax(r, v[j]); }
                else {
                    for (int64_t j = lo + 1; j <= last; ++j) r += v[j];
                    if (op == QK_WIN_AVG) r /= cnt;
                }
            }
            W.out[o][i] = r;
        }
    }
}

__device__ __forceinline__ long long floordiv(long long a, long long b) {      // b > 0
    long long q = a / b;
    return (a % b != 0 && a < 0) ? q - 1 : q;
}

__global__ void __launch_bounds__(256) k_win_hop_expand(const long long* time, const int32_t* by, const int64_t* seg, int n_by, int64_t n,
                                                        long long size, long long hop, int slots, long long* wstart, int32_t* key,
                                                        int32_t* src) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int b = by[i];
        const bool ok = b >= 0 && b < n_by;
        const long long t = time[i];
        const long long first = ok ? floordiv(time[seg[b]], hop) * hop : 0;          // the key's first window start
        const long long kmax = floordiv(t, hop), kmin = floordiv(t - size, hop) + 1;  // k * hop <= t < k * hop + size
        for (int q = 0; q < slots; ++q) {
            const long long k = kmax - q;
            const bool valid = ok && k >= kmin && k * hop >= first;
            const int64_t o = i * slots + q;
            wstart[o] = k * hop; key[o] = b; src[o] = valid ? (int32_t)i : -1;
        }
    }
}

// The run boundaries, one rule per window kind, between consecutive rows (prev, t) of one key.  A session breaks after a gap >
// timeout; the times are sorted within a key, so t - prev is taken as an unsigned difference, exact even from -2^62 to +2^62.
// A tumbling window breaks where floor(t / size) changes: the windows [k * size, (k + 1) * size) of k_win_hop_expand.
__device__ __forceinline__ bool session_breaks(long long prev, long long t, long long timeout) {
    return (unsigned long long)t - (unsigned long long)prev > (unsigned long long)timeout;
}
__device__ __forceinline__ bool tumbling_breaks(long long prev, long long t, long long size) {
    return floordiv(prev, size) != floordiv(t, size);
}
template <int KIND>
__device__ __forceinline__ bool run_breaks(long long prev, long long t, long long param) {
    return KIND == QK_WIN_RUN_TUMBLING ? tumbling_breaks(prev, t, param) : session_breaks(prev, t, param);
}

__global__ void __launch_bounds__(256) k_win_session_flag(const long long* time, const int32_t* by, int64_t n, long long timeout, int32_t* flag) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        flag[i] = (i == 0 || by[i] != by[i - 1] || session_breaks(time[i - 1], time[i], timeout)) ? 1 : 0;
}

// ---------------------------------------------------------------- per-event running aggregates (qk_window_running)
// Every row gets the fold of its run's rows with time <= its own (DuckDB's RANGE UNBOUNDED PRECEDING within PARTITION BY
// key, window).  That is the running fold in row order (ROWS semantics) read at the row's peer end, the last row of the run
// with the same time: a peer group never straddles a run boundary.  Reduce-then-scan over tiles of R_TILE rows:
//   k_win_run_reduce  per tile and channel: the fold of the rows after the tile's last run start (or of the whole tile), and
//                     whether a run starts in the tile;
//   k_win_run_carry   one CTA per channel: a segmented scan of those, in tile order, gives each tile the fold of its first
//                     run's rows before the tile;
//   k_win_run_apply   per tile: the running fold again, with the carry, into shared memory; every row whose peer end lies in
//                     the tile reads its value there and writes it;
//   k_win_run_ties    per tile whose last row is not a peer end: one galloping search finds that peer group's end in a later
//                     tile, and the group's rows in this tile copy its values.
// Peer ends: a reverse pass over the rows would be one more scan; instead a row finds its peer end inside its tile from the
// warps' ballots of peer-end flags, and only the one peer group per tile that runs past the tile searches, so a key whose
// rows all share one time costs one O(log n) search per tile, not a walk per row.  The channels are the running count (channel
// 0, exact in fp64, also AVG's divisor) and one per non-COUNT output.  Every fold runs in a fixed order (warp shuffles, warps in
// order, tiles in order), so the result does not depend on the grid or the SM count.
constexpr int R_NT = 256, R_PER = 8, R_WROWS = 32 * R_PER, R_TILE = R_NT * R_PER, RC_NT = 1024;
constexpr int R_NCH = 1 + 2 * QK_MAX_AGGS;

__device__ __forceinline__ double fold(int op, double a, double b) {      // a: the earlier rows
    return op == QK_WIN_MIN ? fmin(a, b) : op == QK_WIN_MAX ? fmax(a, b) : a + b;
}

// the fold (has, c) of the earlier rows followed by a stretch (flag: a run starts in it, tail: its fold after its last start)
__device__ __forceinline__ void fold_stretch(int op, bool& has, double& c, bool flag, double tail) {
    c = (flag || !has) ? tail : fold(op, c, tail);
    has = true;
}

// In-warp segmented inclusive scan of a (one value per lane, S: the ballot of run starts): the fold from the latest run start
// at or before the lane.  Returns whether such a start exists.
__device__ __forceinline__ bool warp_seg_scan(int op, unsigned S, double& a) {
    const int lane = lane_id();
    const unsigned upto = S & (0xffffffffu >> (31 - lane));
    const int s = upto ? 31 - __clz(upto) : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const double y = __shfl_up_sync(0xffffffffu, a, o);
        if (lane - o >= s) a = fold(op, y, a);
    }
    return upto != 0;
}

// Run-start and peer-end ballots of the warp's stretch: rows wbase + 32 j + lane.  Rows past n start a run and end a peer group.
template <int KIND>
__device__ __forceinline__ void run_flags(const long long* time, const int32_t* by, int64_t n, int64_t wbase, long long param,
                                          unsigned* S, unsigned* E) {
    const int lane = lane_id();
#pragma unroll
    for (int j = 0; j < R_PER; ++j) {
        const int64_t i = wbase + 32 * j + lane;
        const bool in = i < n;
        const long long t = in ? time[i] : 0;
        const int b = in ? by[i] : 0;
        long long tp = __shfl_up_sync(0xffffffffu, t, 1), tn = __shfl_down_sync(0xffffffffu, t, 1);
        int bp = __shfl_up_sync(0xffffffffu, b, 1), bn = __shfl_down_sync(0xffffffffu, b, 1);
        if (lane == 0 && in && i > 0) { tp = time[i - 1]; bp = by[i - 1]; }
        if (lane == 31 && i + 1 < n) { tn = time[i + 1]; bn = by[i + 1]; }
        S[j] = __ballot_sync(0xffffffffu, !in || i == 0 || bp != b || run_breaks<KIND>(tp, t, param));
        E[j] = __ballot_sync(0xffffffffu, !in || i + 1 == n || bn != b || tn != t);
    }
}

// The running fold of channel ch over this CTA's tile into x[j] (row wbase + 32 j + lane).  Rows before the tile's first run
// start fold in (has_c, c), the fold of their run's rows before the tile.  Returns the fold at the tile's last row in every
// thread and sets tile_flag (a run starts in the tile).  Ends with a __syncthreads: wflag / wtail can be reused after it.
__device__ __forceinline__ double tile_scan(const WinArgs& W, int ch, int64_t n, int64_t wbase, const unsigned* S, bool has_c, double c,
                                            double* x, int* wflag, double* wtail, bool& tile_flag) {
    const int op = ch == 0 ? QK_WIN_COUNT : W.op[ch - 1];
    const double* v = ch == 0 ? nullptr : W.val[W.src[ch - 1]];
    const int warp = threadIdx.x >> 5;
    bool seen[R_PER];                                     // a run starts in the stretch at or before the row
    bool has = false, any = false;
    double run = 0.0;
#pragma unroll
    for (int j = 0; j < R_PER; ++j) {
        const int64_t i = wbase + 32 * j + lane_id();
        double a = v ? (i < n ? v[i] : 0.0) : 1.0;
        const bool own = warp_seg_scan(op, S[j], a);
        if (!own && has) a = fold(op, run, a);
        seen[j] = own || any;
        any = any || S[j] != 0;
        x[j] = a;
        run = __shfl_sync(0xffffffffu, a, 31);
        has = true;
    }
    if (lane_id() == 31) { wflag[warp] = any; wtail[warp] = run; }
    __syncthreads();
    bool hw = has_c, ht = has_c;
    double cw = c, ct = c;
    tile_flag = false;
    for (int w = 0; w < R_NT / 32; ++w) {
        if (w < warp) fold_stretch(op, hw, cw, wflag[w], wtail[w]);
        fold_stretch(op, ht, ct, wflag[w], wtail[w]);
        tile_flag = tile_flag || wflag[w];
    }
#pragma unroll
    for (int j = 0; j < R_PER; ++j)
        if (!seen[j] && hw) x[j] = fold(op, cw, x[j]);
    __syncthreads();
    return ct;
}

// the workspace: per tile a run-start flag, then per tile and channel the tile's fold and its carry
struct RunWs {
    uint8_t* flag; double* tail; double* carry; size_t bytes;
    RunWs(int64_t n, void* base) {
        const int64_t nb = (n + R_TILE - 1) / R_TILE;
        Carve c(base);
        flag = c.take<uint8_t>(nb);
        tail = c.take<double>(nb * R_NCH);
        carry = c.take<double>(nb * R_NCH);
        bytes = c.bytes;
    }
};

template <int KIND>
__global__ void __launch_bounds__(R_NT) k_win_run_reduce(const long long* time, const int32_t* by, int64_t n, long long param,
                                                         const __grid_constant__ WinArgs W, uint8_t* flag, double* tail) {
    __shared__ int wflag[R_NT / 32];
    __shared__ double wtail[R_NT / 32];
    const int64_t wbase = (int64_t)blockIdx.x * R_TILE + (threadIdx.x >> 5) * R_WROWS;
    unsigned S[R_PER], E[R_PER];
    run_flags<KIND>(time, by, n, wbase, param, S, E);
    double x[R_PER];
    bool tf = false;
    for (int ch = 0; ch <= W.nout; ++ch) {
        if (ch > 0 && W.op[ch - 1] == QK_WIN_COUNT) continue;
        const double t = tile_scan(W, ch, n, wbase, S, false, 0.0, x, wflag, wtail, tf);
        if (threadIdx.x == 0) tail[blockIdx.x * (int64_t)R_NCH + ch] = t;
    }
    if (threadIdx.x == 0) flag[blockIdx.x] = tf;
}

// carry[k] = the fold of tile k's first run over the rows before tile k: a segmented scan of the tile folds, in chunks of RC_NT tiles
__global__ void __launch_bounds__(RC_NT) k_win_run_carry(int64_t nb, const __grid_constant__ WinArgs W, const uint8_t* flag,
                                                         const double* tail, double* carry) {
    const int ch = blockIdx.x;
    if (ch > 0 && W.op[ch - 1] == QK_WIN_COUNT) return;
    const int op = ch == 0 ? QK_WIN_COUNT : W.op[ch - 1];
    __shared__ int wflag[RC_NT / 32];
    __shared__ double wtail[RC_NT / 32];
    __shared__ double chunk;
    const int warp = threadIdx.x >> 5;
    bool has = false;
    double c = 0.0;
    for (int64_t base = 0; base < nb; base += RC_NT) {
        const int64_t k = base + threadIdx.x;
        const bool f = k < nb ? flag[k] != 0 : true;
        double a = k < nb ? tail[k * R_NCH + ch] : 0.0;
        const unsigned S = __ballot_sync(0xffffffffu, f);
        const bool own = warp_seg_scan(op, S, a);
        if (lane_id() == 31) { wflag[warp] = S != 0; wtail[warp] = a; }
        __syncthreads();
        bool hw = has;
        double cw = c;
        for (int w = 0; w < warp; ++w) fold_stretch(op, hw, cw, wflag[w], wtail[w]);
        if (!own && hw) a = fold(op, cw, a);
        if (k + 1 < nb) carry[(k + 1) * R_NCH + ch] = a;
        if (threadIdx.x == RC_NT - 1) chunk = a;
        __syncthreads();
        c = chunk;
        has = true;
        __syncthreads();
    }
}

template <int KIND>
__global__ void __launch_bounds__(R_NT) k_win_run_apply(const long long* time, const int32_t* by, int64_t n, long long param,
                                                        const __grid_constant__ WinArgs W, const double* carry) {
    __shared__ int wflag[R_NT / 32], wend[R_NT / 32];
    __shared__ double wtail[R_NT / 32];
    __shared__ double cnt[R_TILE], val[R_TILE];
    const int warp = threadIdx.x >> 5, lane = lane_id();
    const int64_t tbase = (int64_t)blockIdx.x * R_TILE, wbase = tbase + warp * R_WROWS;
    unsigned S[R_PER], E[R_PER];
    run_flags<KIND>(time, by, n, wbase, param, S, E);
    // the first peer end of every stretch, then each row's peer end as a tile-local index (-1: past the tile)
    int first = -1;
#pragma unroll
    for (int j = R_PER - 1; j >= 0; --j)
        if (E[j]) first = warp * R_WROWS + 32 * j + __ffs(E[j]) - 1;
    if (lane == 0) wend[warp] = first;
    __syncthreads();
    int pe[R_PER];
    int next = -1;
    for (int w = R_NT / 32 - 1; w > warp; --w)
        if (wend[w] >= 0) next = wend[w];
#pragma unroll
    for (int j = R_PER - 1; j >= 0; --j) {
        const unsigned m = E[j] & (0xffffffffu << lane);
        pe[j] = m ? warp * R_WROWS + 32 * j + __ffs(m) - 1 : next;
        if (E[j]) next = warp * R_WROWS + 32 * j + __ffs(E[j]) - 1;
    }
    const bool has_c = blockIdx.x > 0;
    double x[R_PER];
    bool tf;
    for (int ch = 0; ch <= W.nout; ++ch) {
        const int op = ch == 0 ? QK_WIN_COUNT : W.op[ch - 1];
        if (op != QK_WIN_COUNT || ch == 0) {
            tile_scan(W, ch, n, wbase, S, has_c, has_c ? carry[blockIdx.x * (int64_t)R_NCH + ch] : 0.0, x, wflag, wtail, tf);
            double* dst = ch == 0 ? cnt : val;
#pragma unroll
            for (int j = 0; j < R_PER; ++j) dst[warp * R_WROWS + 32 * j + lane] = x[j];
        }
        __syncthreads();
        if (ch > 0) {
            double* out = W.out[ch - 1];
#pragma unroll
            for (int j = 0; j < R_PER; ++j) {
                const int64_t i = wbase + 32 * j + lane;
                if (i < n && pe[j] >= 0)
                    out[i] = op == QK_WIN_COUNT ? cnt[pe[j]] : op == QK_WIN_AVG ? val[pe[j]] / cnt[pe[j]] : val[pe[j]];
            }
        }
        __syncthreads();
    }
}

// rows of the tile's last peer group when it runs past the tile: the values of its peer end, found by a galloping search
__global__ void __launch_bounds__(R_NT) k_win_run_ties(const long long* time, const int32_t* by, int64_t n, const __grid_constant__ WinArgs W) {
    __shared__ int64_t end;
    const int64_t tbase = (int64_t)blockIdx.x * R_TILE, r = min(tbase + R_TILE, n) - 1;
    const long long t = time[r];
    const int b = by[r];
    if (r + 1 >= n || by[r + 1] != b || time[r + 1] != t) return;
    if (threadIdx.x == 0) {
        int64_t lo = r + 1, step = 1;                       // lo is a peer of r
        while (lo + step < n && by[lo + step] == b && time[lo + step] == t) { lo += step; step <<= 1; }
        int64_t hi = min(lo + step, n);                      // hi is not (or is n)
        while (hi - lo > 1) {
            const int64_t mid = lo + (hi - lo) / 2;
            if (by[mid] == b && time[mid] == t) lo = mid; else hi = mid;
        }
        end = lo;
    }
    __syncthreads();
    const int64_t j = end;
    for (int64_t i = r - threadIdx.x; i >= tbase; i -= R_NT) {
        if (by[i] != b || time[i] != t) break;              // the group is contiguous and ends at r
        for (int o = 0; o < W.nout; ++o) W.out[o][i] = W.out[o][j];
    }
}

// inclusive prefix sum int32 -> int64: per-block sums, count_offsets turns them into block offsets, every block adds its offset
constexpr int S_NT = 256, S_PER = 8, S_TILE = S_NT * S_PER;
__global__ void __launch_bounds__(S_NT) k_scan_block_sums(const int32_t* in, int64_t n, int64_t* sums) {
    __shared__ int64_t w[S_NT / 32];
    const int64_t base = (int64_t)blockIdx.x * S_TILE;
    int64_t s = 0;
    for (int j = 0; j < S_PER; ++j) { const int64_t i = base + j * S_NT + threadIdx.x; s += i < n ? in[i] : 0; }
    const int64_t total = cta_sum<S_NT>(s, w);
    if (threadIdx.x == 0) sums[blockIdx.x] = total;
}
__global__ void __launch_bounds__(S_NT) k_scan_apply(const int32_t* in, int64_t n, const int64_t* offsets, long long* out) {
    __shared__ int64_t wtot[S_NT / 32];
    const int64_t base = (int64_t)blockIdx.x * S_TILE;
    int64_t run = offsets[blockIdx.x];
    for (int j = 0; j < S_PER; ++j) {
        const int64_t i = base + j * S_NT + threadIdx.x;
        const int64_t v = i < n ? in[i] : 0;
        int64_t total;
        const int64_t before = cta_exclusive_scan<S_NT>(v, wtot, total);
        if (i < n) out[i] = run + before + v;
        run += total;
        __syncthreads();
    }
}

// the session workspace: one new-session flag per row, then one sum per tile and the total (scanned in place to offsets)
struct SessionWs {
    int32_t* flag; int64_t* sums; size_t bytes;
    SessionWs(int64_t n, void* base) {
        Carve c(base);
        flag = c.take<int32_t>(n);
        sums = c.take<int64_t>((n + S_TILE - 1) / S_TILE + 1);
        bytes = c.bytes;
    }
};

}  // namespace
}  // namespace qk

using namespace qk;

static int check_ts(const qk_column* time, const qk_column* by, const char* who) {
    if (int rc = check_col(time, who)) return rc;
    if (int rc = check_col(by, who)) return rc;
    if (time->dtype != QK_I64 || by->dtype != QK_I32) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: time must be int64 and the key int32 codes", who);
    if (time->length != by->length) QK_FAIL(QK_ERR_INVALID, "%s: time / key length mismatch", who);
    return 0;
}

extern "C" int qk_window_sliding(const qk_column* time, const qk_column* by, const int64_t* seg, int32_t n_by, int64_t size,
                                 const qk_column* vals, int32_t nvals, const int32_t* ops, const int32_t* srcs, int32_t nout,
                                 qk_column* out, void* stream) {
    const char* who = "qk_window_sliding";
    if (int rc = check_ts(time, by, who)) return rc;
    if (!seg || n_by <= 0 || size <= 0) QK_FAIL(QK_ERR_INVALID, "%s: bad segments / window size", who);
    if (nvals < 0 || nvals > QK_MAX_AGGS || nout < 1 || nout > 2 * QK_MAX_AGGS || !ops || !srcs || !out) QK_FAIL(QK_ERR_INVALID, "%s: bad aggregate arguments", who);
    WinArgs W{};
    const int64_t n = time->length;
    for (int v = 0; v < nvals; ++v) {
        if (int rc = check_col(&vals[v], who)) return rc;
        if (vals[v].dtype != QK_F64 || vals[v].length != n) QK_FAIL(QK_ERR_INVALID, "%s: value column %d must be fp64 with %lld rows", who, v, (long long)n);
        W.val[v] = (const double*)vals[v].data;
    }
    for (int o = 0; o < nout; ++o) {
        if (ops[o] < QK_WIN_SUM || ops[o] > QK_WIN_AVG) QK_FAIL(QK_ERR_INVALID, "%s: bad window aggregate %d", who, ops[o]);
        if (ops[o] != QK_WIN_COUNT && (srcs[o] < 0 || srcs[o] >= nvals)) QK_FAIL(QK_ERR_INVALID, "%s: aggregate %d names no value column", who, o);
        if (int rc = check_col(&out[o], who)) return rc;
        if (out[o].dtype != QK_F64 || out[o].length < n) QK_FAIL(QK_ERR_CAPACITY, "%s: output %d must be fp64 with %lld rows", who, o, (long long)n);
        W.out[o] = (double*)out[o].data; W.op[o] = (int8_t)ops[o]; W.src[o] = (int8_t)(ops[o] == QK_WIN_COUNT ? 0 : srcs[o]);
    }
    W.nout = nout;
    if (n == 0) return QK_OK;
    k_win_sliding<<<grid_size(n, 16), 256, 0, (cudaStream_t)stream>>>((const long long*)time->data, (const int32_t*)by->data, seg, n_by, n, size, W);
    QK_LAUNCH_CHECK("k_win_sliding");
    return QK_OK;
}

extern "C" size_t qk_window_running_workspace_bytes(int64_t nrows) {
    return nrows < 0 ? 0 : RunWs(nrows, nullptr).bytes;
}

extern "C" int qk_window_running(const qk_column* time, const qk_column* by, const int64_t* seg, int32_t n_by, int32_t kind, int64_t param,
                                 const qk_column* vals, int32_t nvals, const int32_t* ops, const int32_t* srcs, int32_t nout,
                                 qk_column* out, void* workspace, size_t ws_bytes, void* stream) {
    const char* who = "qk_window_running";
    if (int rc = check_ts(time, by, who)) return rc;
    if (!seg || n_by <= 0) QK_FAIL(QK_ERR_INVALID, "%s: bad segments", who);
    if (kind == QK_WIN_RUN_TUMBLING ? param <= 0 : kind == QK_WIN_RUN_SESSION ? param < 0 : true)
        QK_FAIL(QK_ERR_INVALID, "%s: bad window kind %d / %s %lld", who, kind, kind == QK_WIN_RUN_SESSION ? "timeout" : "size", (long long)param);
    if (nvals < 0 || nvals > QK_MAX_AGGS || nout < 1 || nout > 2 * QK_MAX_AGGS || !ops || !srcs || !out) QK_FAIL(QK_ERR_INVALID, "%s: bad aggregate arguments", who);
    WinArgs W{};
    const int64_t n = time->length;
    for (int v = 0; v < nvals; ++v) {
        if (int rc = check_col(&vals[v], who)) return rc;
        if (vals[v].dtype != QK_F64 || vals[v].length != n) QK_FAIL(QK_ERR_INVALID, "%s: value column %d must be fp64 with %lld rows", who, v, (long long)n);
        W.val[v] = (const double*)vals[v].data;
    }
    for (int o = 0; o < nout; ++o) {
        if (ops[o] < QK_WIN_SUM || ops[o] > QK_WIN_AVG) QK_FAIL(QK_ERR_INVALID, "%s: bad window aggregate %d", who, ops[o]);
        if (ops[o] != QK_WIN_COUNT && (srcs[o] < 0 || srcs[o] >= nvals)) QK_FAIL(QK_ERR_INVALID, "%s: aggregate %d names no value column", who, o);
        if (int rc = check_col(&out[o], who)) return rc;
        if (out[o].dtype != QK_F64 || out[o].length < n) QK_FAIL(QK_ERR_CAPACITY, "%s: output %d must be fp64 with %lld rows", who, o, (long long)n);
        W.out[o] = (double*)out[o].data; W.op[o] = (int8_t)ops[o]; W.src[o] = (int8_t)(ops[o] == QK_WIN_COUNT ? 0 : srcs[o]);
    }
    W.nout = nout;
    if (n == 0) return QK_OK;
    const RunWs w(n, workspace);
    if (!workspace || ws_bytes < w.bytes) QK_FAIL(QK_ERR_CAPACITY, "%s: workspace too small (%zu < %zu bytes)", who, ws_bytes, w.bytes);
    const long long* t = (const long long*)time->data;
    const int32_t* b = (const int32_t*)by->data;
    const unsigned nb = (unsigned)((n + R_TILE - 1) / R_TILE);
    cudaStream_t st = (cudaStream_t)stream;
    if (kind == QK_WIN_RUN_TUMBLING) k_win_run_reduce<QK_WIN_RUN_TUMBLING><<<nb, R_NT, 0, st>>>(t, b, n, param, W, w.flag, w.tail);
    else k_win_run_reduce<QK_WIN_RUN_SESSION><<<nb, R_NT, 0, st>>>(t, b, n, param, W, w.flag, w.tail);
    QK_LAUNCH_CHECK("k_win_run_reduce");
    k_win_run_carry<<<nout + 1, RC_NT, 0, st>>>(nb, W, w.flag, w.tail, w.carry);
    QK_LAUNCH_CHECK("k_win_run_carry");
    if (kind == QK_WIN_RUN_TUMBLING) k_win_run_apply<QK_WIN_RUN_TUMBLING><<<nb, R_NT, 0, st>>>(t, b, n, param, W, w.carry);
    else k_win_run_apply<QK_WIN_RUN_SESSION><<<nb, R_NT, 0, st>>>(t, b, n, param, W, w.carry);
    QK_LAUNCH_CHECK("k_win_run_apply");
    k_win_run_ties<<<nb, R_NT, 0, st>>>(t, b, n, W);
    QK_LAUNCH_CHECK("k_win_run_ties");
    return QK_OK;
}

extern "C" int qk_window_hop_expand(const qk_column* time, const qk_column* by, const int64_t* seg, int32_t n_by, int64_t size, int64_t hop,
                                    int32_t slots, int64_t* wstart, int32_t* key, int32_t* src, void* stream) {
    const char* who = "qk_window_hop_expand";
    if (int rc = check_ts(time, by, who)) return rc;
    if (!seg || n_by <= 0 || size <= 0 || hop <= 0 || slots < 1 || (int64_t)slots * hop < size) QK_FAIL(QK_ERR_INVALID, "%s: bad window geometry", who);
    const int64_t n = time->length;
    if (n * slots > 0x7fffffffLL) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: %lld rows x %d windows exceed int32 row numbers; feed smaller batches", who, (long long)n, slots);
    if (n == 0) return QK_OK;
    if (!wstart || !key || !src) QK_FAIL(QK_ERR_INVALID, "%s: null outputs", who);
    k_win_hop_expand<<<grid_size(n, 16), 256, 0, (cudaStream_t)stream>>>((const long long*)time->data, (const int32_t*)by->data, seg, n_by, n, size, hop,
                                                                     slots, (long long*)wstart, key, src);
    QK_LAUNCH_CHECK("k_win_hop_expand");
    return QK_OK;
}

extern "C" size_t qk_window_session_workspace_bytes(int64_t nrows) {
    return nrows < 0 ? 0 : SessionWs(nrows, nullptr).bytes;
}

extern "C" int qk_window_session_ids(const qk_column* time, const qk_column* by, int64_t timeout, int64_t* ids, void* workspace,
                                     size_t ws_bytes, void* stream) {
    const char* who = "qk_window_session_ids";
    if (int rc = check_ts(time, by, who)) return rc;
    if (timeout < 0) QK_FAIL(QK_ERR_INVALID, "%s: negative timeout", who);
    const int64_t n = time->length;
    if (n == 0) return QK_OK;
    const SessionWs w(n, workspace);
    if (!ids || !workspace || ws_bytes < w.bytes) QK_FAIL(QK_ERR_CAPACITY, "%s: null output / workspace too small", who);
    int32_t* flag = w.flag;
    int64_t* sums = w.sums;                                                           // nb + 1: offsets, then the total
    cudaStream_t st = (cudaStream_t)stream;
    k_win_session_flag<<<grid_size(n, 16), 256, 0, st>>>((const long long*)time->data, (const int32_t*)by->data, n, timeout, flag);
    QK_LAUNCH_CHECK("k_win_session_flag");
    const int64_t nb = (n + S_TILE - 1) / S_TILE;
    k_scan_block_sums<<<(unsigned)nb, S_NT, 0, st>>>(flag, n, sums);
    QK_LAUNCH_CHECK("k_scan_block_sums");
    if (int rc = count_offsets(sums, 1, nb, sums, sums + nb, st)) return rc;      // in place
    k_scan_apply<<<(unsigned)nb, S_NT, 0, st>>>(flag, n, sums, (long long*)ids);
    QK_LAUNCH_CHECK("k_scan_apply");
    return QK_OK;
}
