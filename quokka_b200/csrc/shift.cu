// shift.cu -- K14 lag / lead per key over a stream in order (OrderedStream.shift; pyquokka/orderedstream.py:13-35).
//
// qk_shift_plan turns the stable key partition (qk_partition_plan with QK_PART_CODE: dest = a row's place in key-segmented
// order, seg = the segment starts) into one source row per output row.  Row i sits at p = dest[i] inside its key's segment
// [s, e); its source sits at p - n when that is inside the segment, and the inverse permutation (inv[dest[i]] = i, one
// launch) names it.  The same pass flags the rows another rank needs (edge) and counts rows whose time is below their
// predecessor's in the key (the order check).  Without a key the segment is the whole input and no inverse is needed.
// Per row: dest + by + inv (4 B each, read), src written (4 B), edge (1 B) and time (8 B row + 8 B predecessor) when asked.
//
// qk_shift_gather then writes every shifted column in one launch: src < n_a reads the rank's own table A, src >= n_a the
// small boundary table B of other ranks' rows, src == -1 the column's fill value; validity travels with the value.
#include "common.cuh"

namespace qk {
namespace {

constexpr long long SH_HUGE = 1ll << 31;                // |n| at or above this: no row has a source

__global__ void __launch_bounds__(256) k_shift_invert(const int32_t* __restrict__ dest, int32_t* __restrict__ inv, int64_t n) {
    for (int64_t i = blockIdx.x * 256ll + threadIdx.x; i < n; i += gridDim.x * 256ll) inv[dest[i]] = (int32_t)i;
}

// by == NULL: one key, position = row.  sh is the shift clamped to [-2^31, 2^31], so no sum below overflows.
__global__ void __launch_bounds__(256) k_shift_plan(const int32_t* __restrict__ by, const int32_t* __restrict__ dest,
                                                    const int64_t* __restrict__ seg, const int32_t* __restrict__ inv, int64_t n,
                                                    long long sh, int64_t lo, int64_t hi, int32_t* __restrict__ src,
                                                    uint8_t* __restrict__ edge, const int64_t* __restrict__ time,
                                                    unsigned long long* status) {
    unsigned bad = 0;
    for (int64_t i = blockIdx.x * 256ll + threadIdx.x; i < n; i += gridDim.x * 256ll) {
        long long p = i, s = 0, e = n;
        if (by) {
            p = dest[i];
            const int k = by[i];
            s = seg[k];
            e = seg[k + 1];
        }
        if (i >= lo && i < hi) {
            const long long q = p - sh;
            int32_t r = -1;
            if (q >= s && q < e) {
                const long long row = by ? inv[q] : q;
                r = (int32_t)(row >= lo ? row - lo : row - lo + n);      // numbered from lo: [lo, n) first, then [0, lo)
            }
            src[i - lo] = r;
        }
        if (edge) edge[i] = sh > 0 ? p >= e - sh : (sh < 0 ? p < s - sh : 0);
        if (time && p > s) {
            const long long prev = by ? inv[p - 1] : p - 1;
            bad += time[i] < time[prev];
        }
    }
    if (time) {
        for (int o = 16; o; o >>= 1) bad += __shfl_xor_sync(0xffffffffu, bad, o);
        if (lane_id() == 0 && bad) atomicAdd(status, (unsigned long long)bad);
    }
}

struct GatherArgs {
    const void* a[QK_MAX_COLS];
    const void* b[QK_MAX_COLS];
    void* out[QK_MAX_COLS];
    const uint8_t* av[QK_MAX_COLS];
    const uint8_t* bv[QK_MAX_COLS];
    uint8_t* ov[QK_MAX_COLS];
    unsigned long long fill[QK_MAX_COLS];
    int size[QK_MAX_COLS];
    uint8_t fill_valid[QK_MAX_COLS];
    int ncols;
};

template <typename T>
__device__ __forceinline__ void move_value(const void* a, const void* b, void* out, unsigned long long fill, int64_t i, int32_t s,
                                           int64_t n_a) {
    T v;
    if (s < 0) v = (T)fill;
    else if (s < n_a) v = ((const T*)a)[s];
    else v = ((const T*)b)[s - n_a];
    ((T*)out)[i] = v;
}

__global__ void __launch_bounds__(256) k_shift_gather(const __grid_constant__ GatherArgs G, const int32_t* __restrict__ src,
                                                      int64_t n, int64_t n_a) {
    for (int64_t i = blockIdx.x * 256ll + threadIdx.x; i < n; i += gridDim.x * 256ll) {
        const int32_t s = src[i];
        for (int c = 0; c < G.ncols; ++c) {
            switch (G.size[c]) {
                case 1: move_value<uint8_t>(G.a[c], G.b[c], G.out[c], G.fill[c], i, s, n_a); break;
                case 4: move_value<uint32_t>(G.a[c], G.b[c], G.out[c], G.fill[c], i, s, n_a); break;
                default: move_value<unsigned long long>(G.a[c], G.b[c], G.out[c], G.fill[c], i, s, n_a); break;
            }
            if (G.ov[c]) {
                const uint8_t* v = s < n_a ? G.av[c] : G.bv[c];
                const int64_t j = s < n_a ? s : s - n_a;
                G.ov[c][i] = s < 0 ? G.fill_valid[c] : (v ? (uint8_t)(v[j] != 0) : (uint8_t)1);
            }
        }
    }
}

// the keyed plan's workspace: the inverse permutation, then 256 spare bytes
struct ShiftWs {
    int32_t* inv; size_t bytes;
    ShiftWs(int64_t n, void* base) {
        Carve c(base);
        inv = c.take<int32_t>(n);
        c.take<char>(256);                              // spare
        bytes = c.bytes;
    }
};

}  // namespace
}  // namespace qk

using namespace qk;

extern "C" size_t qk_shift_workspace_bytes(int64_t nrows) {
    return nrows < 0 ? 0 : ShiftWs(nrows, nullptr).bytes;
}

extern "C" int qk_shift_plan(const int32_t* by, int32_t n_by, const int32_t* dest, const int64_t* seg, int64_t nrows, int64_t n,
                             int64_t lo, int64_t hi, int32_t* src, uint8_t* edge, const int64_t* time, uint64_t* status,
                             void* workspace, size_t ws_bytes, void* stream) {
    const char* who = "qk_shift_plan";
    if (nrows > 0x7fffffffLL) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: %lld rows; row numbers are int32", who, (long long)nrows);
    if (nrows < 0) QK_FAIL(QK_ERR_INVALID, "%s: nrows %lld", who, (long long)nrows);
    if ((by == nullptr) != (dest == nullptr) || (by == nullptr) != (seg == nullptr))
        QK_FAIL(QK_ERR_INVALID, "%s: by, dest and seg are given together or not at all", who);
    if (by && n_by < 1) QK_FAIL(QK_ERR_INVALID, "%s: n_by %d", who, (int)n_by);
    if (lo < 0 || hi < lo || hi > nrows) QK_FAIL(QK_ERR_INVALID, "%s: rows [%lld, %lld) outside [0, %lld)", who, (long long)lo, (long long)hi, (long long)nrows);
    if (hi > lo && !src) QK_FAIL(QK_ERR_INVALID, "%s: null src", who);
    if (time && !status) QK_FAIL(QK_ERR_INVALID, "%s: a time column needs a status word", who);
    cudaStream_t st = (cudaStream_t)stream;
    if (status) QK_CUDA(cudaMemsetAsync(status, 0, sizeof(uint64_t), st));
    if (nrows == 0) return QK_OK;
    int32_t* inv = nullptr;
    if (by) {
        const ShiftWs w(nrows, workspace);
        if (!workspace || ws_bytes < w.bytes) QK_FAIL(QK_ERR_CAPACITY, "%s: workspace too small", who);
        inv = w.inv;
        k_shift_invert<<<grid_size(nrows, 16), 256, 0, st>>>(dest, inv, nrows);
        QK_LAUNCH_CHECK("k_shift_invert");
    }
    const long long sh = n >= SH_HUGE ? SH_HUGE : (n <= -SH_HUGE ? -SH_HUGE : (long long)n);
    k_shift_plan<<<grid_size(nrows, 16), 256, 0, st>>>(by, dest, seg, inv, nrows, sh, lo, hi, src, edge, time,
                                                      (unsigned long long*)status);
    QK_LAUNCH_CHECK("k_shift_plan");
    return QK_OK;
}

extern "C" int qk_shift_gather(const qk_column* a_cols, const qk_column* b_cols, int32_t ncols, const uint8_t* const* a_valid,
                               const uint8_t* const* b_valid, const uint64_t* fill, const uint8_t* fill_valid, const int32_t* src,
                               int64_t nrows, int64_t n_b, qk_column* out, uint8_t* const* out_valid, void* stream) {
    const char* who = "qk_shift_gather";
    if (ncols < 0 || ncols > QK_MAX_COLS) QK_FAIL(QK_ERR_INVALID, "%s: ncols %d out of range", who, (int)ncols);
    if (ncols == 0) return QK_OK;
    if (!a_cols || !out || !fill || !fill_valid || (n_b > 0 && !b_cols)) QK_FAIL(QK_ERR_INVALID, "%s: null arguments", who);
    if (nrows < 0 || n_b < 0) QK_FAIL(QK_ERR_INVALID, "%s: negative row counts", who);
    GatherArgs G;
    const int64_t n_a = a_cols[0].length;
    if (n_a + n_b > 0x7fffffffLL || nrows > 0x7fffffffLL) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: row numbers are int32", who);
    for (int c = 0; c < ncols; ++c) {
        if (int rc = check_col(&a_cols[c], who)) return rc;
        if (int rc = check_col(&out[c], who)) return rc;
        if (n_b > 0) {
            if (int rc = check_col(&b_cols[c], who)) return rc;
            if (b_cols[c].dtype != a_cols[c].dtype || b_cols[c].length != n_b)
                QK_FAIL(QK_ERR_INVALID, "%s: column %d of table B is not %lld rows of A's dtype", who, c, (long long)n_b);
        }
        if (a_cols[c].length != n_a) QK_FAIL(QK_ERR_INVALID, "%s: the columns of table A differ in length", who);
        if (out[c].dtype != a_cols[c].dtype) QK_FAIL(QK_ERR_INVALID, "%s: output %d has another dtype", who, c);
        if (out[c].length < nrows) QK_FAIL(QK_ERR_CAPACITY, "%s: output %d too small", who, c);
        G.a[c] = a_cols[c].data;
        G.b[c] = n_b > 0 ? b_cols[c].data : nullptr;
        G.out[c] = (void*)out[c].data;
        G.av[c] = a_valid ? a_valid[c] : nullptr;
        G.bv[c] = b_valid ? b_valid[c] : nullptr;
        G.ov[c] = out_valid ? out_valid[c] : nullptr;
        G.fill[c] = fill[c];
        G.fill_valid[c] = fill_valid[c] ? 1 : 0;
        G.size[c] = dtype_size(a_cols[c].dtype);
    }
    G.ncols = ncols;
    if (nrows == 0) return QK_OK;
    if (!src) QK_FAIL(QK_ERR_INVALID, "%s: null src", who);
    k_shift_gather<<<grid_size(nrows, 16), 256, 0, (cudaStream_t)stream>>>(G, src, nrows, n_a);
    QK_LAUNCH_CHECK("k_shift_gather");
    return QK_OK;
}
