// common.cuh -- shared host/device helpers for libqk.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include <atomic>
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
        default: return 0;
    }
}
static inline bool dtype_is_int(int dt) { return dt == QK_U8 || dt == QK_I32 || dt == QK_I64; }

static inline int check_col(const qk_column* c, const char* what) {
    if (!c) QK_FAIL(QK_ERR_INVALID, "%s: null column", what);
    if (dtype_size(c->dtype) == 0) QK_FAIL(QK_ERR_INVALID, "%s: bad dtype %d", what, c->dtype);
    if (c->validity) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: validity bitmaps are not supported on the hot path", what);
    if (c->length < 0 || c->length > 0x7fffffffLL) QK_FAIL(QK_ERR_INVALID, "%s: length %lld out of range", what, (long long)c->length);
    if (c->length > 0 && !c->data) QK_FAIL(QK_ERR_INVALID, "%s: null data", what);
    return 0;
}

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

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
__device__ __forceinline__ unsigned ld_u32_hint(const void* p, unsigned long long pol) {
    unsigned v; asm volatile("ld.global.nc.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pol)); return v;
}
__device__ __forceinline__ unsigned ld_u8_stream(const void* p, unsigned long long pol) {
    unsigned v; asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.u8 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pol)); return v;
}
__device__ __forceinline__ int ld_i32_stream(const void* p, unsigned long long pol) {
    int v; asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.s32 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pol)); return v;
}
__device__ __forceinline__ long long ld_i64_stream(const void* p, unsigned long long pol) {
    long long v; asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.s64 %0, [%1], %2;" : "=l"(v) : "l"(p), "l"(pol)); return v;
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

}  // namespace qk
