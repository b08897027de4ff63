// common.cuh -- shared host/device helpers for libqk.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include <atomic>
#include <map>
#include <mutex>
#include <utility>
#include <string>
#include "../../include/qk.h"

namespace qk {

// ---------------------------------------------------------------- host side
void set_err(const char* fmt, ...);
extern std::atomic<int64_t> g_launches;
int sm_count();

#define QK_FAIL(code, ...)              \
    do {                                \
        qk::set_err(__VA_ARGS__);       \
        return (code);                  \
    } while (0)

#define QK_LAUNCH_CHECK(name)                                                          \
    do {                                                                               \
        qk::g_launches.fetch_add(1, std::memory_order_relaxed);                        \
        cudaError_t e__ = cudaGetLastError();                                          \
        if (e__ != cudaSuccess) QK_FAIL(QK_ERR_CUDA, "%s: %s", name, cudaGetErrorString(e__)); \
    } while (0)

#define QK_CUDA(call)                                                                  \
    do {                                                                               \
        cudaError_t e__ = (call);                                                      \
        if (e__ != cudaSuccess) QK_FAIL(QK_ERR_CUDA, "%s: %s", #call, cudaGetErrorString(e__)); \
    } while (0)

static inline int dtype_size(int dt) {
    switch (dt) {
        case QK_U8: return 1;
        case QK_I32: case QK_F32: return 4;
        case QK_I64: case QK_F64: return 8;
        case QK_F16: return 2;
        default: return 0;
    }
}
static inline bool dtype_is_int(int dt) { return dt == QK_U8 || dt == QK_I32 || dt == QK_I64; }

// a column of any row width: scalar (lanes 0 / 1) or vector (lanes > 1) -- for the kernels that only move rows
static inline int check_rows_col(const qk_column* c, const char* what) {
    if (!c) QK_FAIL(QK_ERR_INVALID, "%s: null column", what);
    if (dtype_size(c->dtype) == 0) QK_FAIL(QK_ERR_INVALID, "%s: bad dtype %d", what, c->dtype);
    if (c->lanes < 0 || c->lanes > QK_KNN_MAX_DIM) QK_FAIL(QK_ERR_INVALID, "%s: lanes %d out of range", what, (int)c->lanes);
    if (c->validity) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: validity bitmaps are not supported on the hot path", what);
    if (c->length < 0 || c->length > 0x7fffffffLL) QK_FAIL(QK_ERR_INVALID, "%s: length %lld out of range", what, (long long)c->length);
    if (c->length > 0 && !c->data) QK_FAIL(QK_ERR_INVALID, "%s: null data", what);
    return 0;
}
static inline int row_lanes(const qk_column* c) { return c->lanes > 1 ? c->lanes : 1; }
static inline long long row_bytes(const qk_column* c) { return (long long)dtype_size(c->dtype) * row_lanes(c); }

// a scalar column: what every kernel that reads values takes
static inline int check_col(const qk_column* c, const char* what) {
    if (int rc = check_rows_col(c, what)) return rc;
    if (c->lanes > 1) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: vector columns (lanes %d) are not supported here", what, (int)c->lanes);
    if (c->dtype == QK_F16) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: f16 elements are only supported in vector columns", what);
    return 0;
}

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// A caller-provided workspace, laid out once.  A kernel's layout function takes its pieces in order from one Carve:
// over a null base it only adds up the bytes (what its qk_*_workspace_bytes returns), over the caller's buffer it also
// hands out every piece, at the same offsets.  Each piece is rounded up to `align` bytes (256 unless said otherwise).
// A nested layout (another kernel's workspace) is taken as one piece of its total.
struct Carve {
    char* base;
    size_t bytes = 0;
    explicit Carve(void* b) : base((char*)b) {}
    template <typename T>
    T* take(size_t count, size_t align = 256) {
        T* p = base ? (T*)(base + bytes) : nullptr;
        bytes += align_up(count * sizeof(T), align);
        return p;
    }
};

// grid of a grid-stride launch: one CTA per `per_cta` work items, at most `per_sm` CTAs per SM, at least one CTA
static inline unsigned grid_size(int64_t n, int per_sm, int64_t per_cta = 256) {
    const int64_t nb = (n + per_cta - 1) / per_cta, cap = (int64_t)sm_count() * per_sm;
    return (unsigned)(nb < 1 ? 1 : (nb > cap ? cap : nb));
}

// counts -> exclusive offsets, one CTA per row of a row-major rows x n count matrix:
// offsets[b * n + i] = counts[b * n] + ... + counts[b * n + i - 1] and totals[b] = the sum of row b.
// With rows = 1 and totals = offsets + n, offsets[n] holds the total.  Instantiated for uint32_t and int64_t counts.
template <typename T>
int count_offsets(const T* counts, int64_t rows, int64_t n, int64_t* offsets, int64_t* totals, cudaStream_t st);

// An integer-range predicate node (QK_OP_CMP_COL_IMM or QK_OP_RANGE_COL_IMM) as the branch-free test
// ((lo <= x) & (x <= hi)) != neg, its bounds clamped to 32 bits when the column is QK_I32 (a kernel that compares in
// 32 bits must not truncate a bound beyond int32) and to 64 bits otherwise.  An empty range is lo = 1, hi = 0.
struct IntRange { int64_t lo, hi; bool neg; };
static inline IntRange int_range(const qk_expr_node& nd, int dtype) {
    const int64_t tmin = dtype == QK_I32 ? INT32_MIN : INT64_MIN, tmax = dtype == QK_I32 ? INT32_MAX : INT64_MAX;
    IntRange r{tmin, tmax, false};
    bool empty = false;
    if (nd.op == QK_OP_RANGE_COL_IMM) {
        r.neg = nd.a1 != 0;
        const int64_t lo = nd.imm_i, hi = (int64_t)nd.imm;
        empty = lo > tmax || hi < tmin || lo > hi;
        if (lo > tmin) r.lo = lo;
        if (hi < tmax) r.hi = hi;
    } else {
        const int64_t imm = nd.imm_i;
        switch (nd.a1) {
            case QK_CMP_LT: if (imm <= tmin) empty = true; else r.hi = imm > tmax ? tmax : imm - 1; break;
            case QK_CMP_LE: if (imm < tmin) empty = true; else r.hi = imm > tmax ? tmax : imm; break;
            case QK_CMP_GT: if (imm >= tmax) empty = true; else r.lo = imm < tmin ? tmin : imm + 1; break;
            case QK_CMP_GE: if (imm > tmax) empty = true; else r.lo = imm < tmin ? tmin : imm; break;
            case QK_CMP_EQ: if (imm < tmin || imm > tmax) empty = true; else r.lo = r.hi = imm; break;
            default: r.neg = true; if (imm < tmin || imm > tmax) empty = true; else r.lo = r.hi = imm; break;   // !=
        }
    }
    if (empty) { r.lo = 1; r.hi = 0; }
    return r;
}

// ---------------------------------------------------------------- device side
__host__ __device__ __forceinline__ uint64_t mix64(uint64_t x) {
    x ^= x >> 30; x *= 0xBF58476D1CE4E5B9ULL;
    x ^= x >> 27; x *= 0x94D049BB133111EBULL;
    x ^= x >> 31;
    return x;
}

__device__ __forceinline__ double load_f64(const void* p, int dt, int64_t i) {
    switch (dt) {
        case QK_U8: return (double)((const uint8_t*)p)[i];
        case QK_I32: return (double)((const int32_t*)p)[i];
        case QK_I64: return (double)((const int64_t*)p)[i];
        case QK_F32: return (double)((const float*)p)[i];
        default: return ((const double*)p)[i];
    }
}
__device__ __forceinline__ int64_t load_i64(const void* p, int dt, int64_t i) {
    switch (dt) {
        case QK_U8: return (int64_t)((const uint8_t*)p)[i];
        case QK_I32: return (int64_t)((const int32_t*)p)[i];
        default: return ((const int64_t*)p)[i];
    }
}
// The ascending order image of element i (DESIGN.md section 2 "Ordering rules"): unsigned comparison of images is DuckDB's
// ORDER BY.  Integers are exact over their whole range, -0.0 is folded onto +0.0 and every NaN, whatever its sign and
// payload, takes the greatest image (after +inf).  32-bit and 8-bit types sit in the top bytes.  Descending = ~image.
__device__ __forceinline__ unsigned long long order_image(const void* p, int dt, int64_t i) {
    switch (dt) {
        case QK_F64: {
            unsigned long long b = ((const unsigned long long*)p)[i];
            if (b == 0x8000000000000000ULL) b = 0;
            return (b << 1) > 0xffe0000000000000ULL ? ~0ULL : (b >> 63) ? ~b : (b | 0x8000000000000000ULL);
        }
        case QK_F32: {
            unsigned b = ((const unsigned*)p)[i];
            if (b == 0x80000000u) b = 0;
            const unsigned v = (b << 1) > 0xff000000u ? ~0u : (b >> 31) ? ~b : (b | 0x80000000u);
            return (unsigned long long)v << 32;
        }
        case QK_I64: return ((const unsigned long long*)p)[i] ^ 0x8000000000000000ULL;
        case QK_I32: return (unsigned long long)(((const unsigned*)p)[i] ^ 0x80000000u) << 32;
        default: return (unsigned long long)((const uint8_t*)p)[i] << 56;
    }
}
__device__ __forceinline__ bool cmp_i64(int64_t a, int cmp, int64_t b) {
    switch (cmp) {
        case QK_CMP_LT: return a < b;
        case QK_CMP_LE: return a <= b;
        case QK_CMP_GT: return a > b;
        case QK_CMP_GE: return a >= b;
        case QK_CMP_EQ: return a == b;
        default: return a != b;
    }
}
// L2 residency hints (H100: 50 MB L2 shared by streams and small hot structures).  A table that is probed at random
// while column streams many times its size pass through the same L2 -- a Bloom filter, a hash table -- is loaded with
// evict_last; the streams are loaded with evict_first (and bypass L1), so they do not push the table out.
__device__ __forceinline__ unsigned long long l2_policy_evict_first() {
    unsigned long long p; asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p)); return p;
}
__device__ __forceinline__ unsigned long long l2_policy_evict_last() {
    unsigned long long p; asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p)); return p;
}

// key mod nparts (non-negative result) without a 64-bit division: nparts is the number of ranks (1, 2, 4, 8 in practice).
// A 64-bit `%` by a runtime divisor costs ~120 instructions per row and made the mask kernel instruction-bound.
__device__ __forceinline__ unsigned part_mod(long long key, unsigned nparts) {
    if (nparts == 1u) return 0u;
    if ((nparts & (nparts - 1u)) == 0u) return (unsigned)((unsigned long long)key & (nparts - 1u));    // two's complement: also right for key < 0
    const unsigned long long u = (unsigned long long)key;
    const unsigned hi = (unsigned)(u >> 32) % nparts, lo = (unsigned)u % nparts;
    const unsigned two32 = (unsigned)((1ull << 32) % nparts);
    unsigned r = (hi * two32 + lo) % nparts;                       // u mod nparts (hi, two32 < nparts <= 65535: no overflow)
    if (key < 0) {                                                 // u = key + 2^64: take 2^64 mod nparts back out
        const unsigned two64 = (unsigned)(((unsigned long long)two32 * two32) % nparts);
        r = (r + nparts - two64) % nparts;
    }
    return r;
}
__device__ __forceinline__ unsigned lane_id() { return threadIdx.x & 31; }
__device__ __forceinline__ unsigned lanemask_lt() {
    unsigned m; asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m)); return m;
}

// inclusive prefix sum over the lanes of a warp (all 32 lanes active)
template <typename T>
__device__ __forceinline__ T warp_inclusive_scan(T x) {
    for (int o = 1; o < 32; o <<= 1) {
        const T y = __shfl_up_sync(0xffffffffu, x, o);
        if ((int)lane_id() >= o) x += y;
    }
    return x;
}

// CTA-wide sums over NT threads.  Each takes a shared buffer of NT / 32 slots and holds the one __syncthreads between
// writing it and reading it; a caller that uses the buffer again must pass a __syncthreads of its own first.

// exclusive prefix sum of v in thread order; total = the CTA's sum
template <int NT, typename T>
__device__ __forceinline__ T cta_exclusive_scan(T v, T* wsum, T& total) {
    const int warp = threadIdx.x >> 5;
    const T x = warp_inclusive_scan(v);
    if (lane_id() == 31) wsum[warp] = x;
    __syncthreads();
    T before = 0;
    total = 0;
    for (int w = 0; w < NT / 32; ++w) { if (w < warp) before += wsum[w]; total += wsum[w]; }
    return before + x - v;
}
// the same over one flag per thread, given as its warp's ballot `bal`: the thread's rank among the CTA's set flags
// (meaningful where the thread's own bit is set); total = the CTA's number of set flags
template <int NT>
__device__ __forceinline__ int cta_ballot_rank(unsigned bal, int* wsum, int& total) {
    const int warp = threadIdx.x >> 5;
    if (lane_id() == 0) wsum[warp] = __popc(bal);
    __syncthreads();
    int before = 0;
    total = 0;
    for (int w = 0; w < NT / 32; ++w) { if (w < warp) before += wsum[w]; total += wsum[w]; }
    return before + __popc(bal & lanemask_lt());
}
// sum of v over the CTA, returned in thread 0 (0 elsewhere)
template <int NT, typename T>
__device__ __forceinline__ T cta_sum(T v, T* wsum) {
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane_id() == 0) wsum[threadIdx.x >> 5] = v;
    __syncthreads();
    T t = 0;
    if (threadIdx.x == 0)
        for (int w = 0; w < NT / 32; ++w) t += wsum[w];
    return t;
}

// The dynamic shared-memory limit of a kernel is one value per kernel and device, shared by every host thread.  A call that
// set it to its own size could lower it between another thread's setting and that thread's launch, which then fails with
// "invalid argument".  Here the limit only ever rises, to the most any call has needed, under one lock.
inline cudaError_t raise_smem_limit(const void* kernel, size_t bytes) {
    static std::mutex mu;
    static std::map<std::pair<const void*, int>, size_t> limit;
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    std::lock_guard<std::mutex> lock(mu);
    size_t& cur = limit[{kernel, dev}];
    if (bytes <= cur) return cudaSuccess;
    e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e == cudaSuccess) cur = bytes;
    return e;
}

}  // namespace qk
