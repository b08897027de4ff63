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
//            the session ids then go through the hash aggregate.
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

__global__ void __launch_bounds__(256) k_win_session_flag(const long long* time, const int32_t* by, int64_t n, long long timeout, int32_t* flag) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        flag[i] = (i == 0 || by[i] != by[i - 1] || time[i] - time[i - 1] > timeout) ? 1 : 0;
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
