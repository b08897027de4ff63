// hashagg.cu -- K2 high-cardinality hash aggregate (Q3: ~1.16 M groups at SF-100).
//
// Open addressing over packed integer keys (<= 128 bits in two 64-bit words, compared exactly).
// Slot protocol: tag EMPTY -> BUSY (atomicCAS by the inserting lane) -> READY (after the key words are
// stored and fenced); a lane that meets a BUSY slot re-reads it (Volta+ independent thread scheduling
// guarantees the owner makes progress).  Aggregation itself is one native fp64 red.global.add per value
// (min/max: CAS loop) -- HBM/L2 random-access bound: per input row one tag+key probe (>= 32 B sector)
// plus 8 B x nagg of atomic traffic; algorithmic bytes in DESIGN.md.
// The state persists across update() calls, which is what SQLAggExecutor's "concat partials, aggregate at
// done()" (sql_executors.py:585-599) amounts to.
#include "common.cuh"

namespace qk {
namespace {

enum : unsigned { TAG_EMPTY = 0u, TAG_BUSY = 1u, TAG_READY = 2u };

struct KeyLayout {          // where each key column lives inside the two packed words
    int32_t nkeys, nwords;
    int32_t word[4], shift[4], bytes[4], dtype[4];
};

struct State {              // carved out of the caller's buffer
    unsigned* tag; unsigned long long* k0; unsigned long long* k1; long long* cnt; double* acc;
};

size_t carve(const qk_hashagg_desc* d, void* base, State& s) {
    Carve c(base);
    const size_t cap = (size_t)d->capacity;
    s.tag = c.take<unsigned>(cap);
    s.k0 = c.take<unsigned long long>(cap);
    s.k1 = c.take<unsigned long long>(cap);
    s.cnt = c.take<long long>(cap);
    s.acc = c.take<double>(cap * (d->nagg > 0 ? d->nagg : 1));
    return c.bytes;
}

int make_layout(const qk_hashagg_desc* d, KeyLayout* L, const char* who) {
    if (!d) QK_FAIL(QK_ERR_INVALID, "%s: null descriptor", who);
    if (d->capacity <= 0 || (d->capacity & (d->capacity - 1))) QK_FAIL(QK_ERR_INVALID, "%s: capacity must be a power of two", who);
    if (d->nkeys < 1 || d->nkeys > 4) QK_FAIL(QK_ERR_INVALID, "%s: nkeys must be 1..4", who);
    if (d->nagg < 0 || d->nagg > QK_MAX_AGGS) QK_FAIL(QK_ERR_INVALID, "%s: nagg out of range", who);
    for (int j = 0; j < d->nagg; ++j) if (d->agg_op[j] < QK_AGG_SUM || d->agg_op[j] > QK_AGG_MAX) QK_FAIL(QK_ERR_INVALID, "%s: bad aggregate op", who);
    int used[2] = {0, 0};
    L->nkeys = d->nkeys; L->nwords = 1;
    for (int k = 0; k < d->nkeys; ++k) {
        if (!dtype_is_int(d->key_dtype[k])) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: group keys must be integer / dictionary-code columns", who);
        const int bits = 8 * dtype_size(d->key_dtype[k]);
        int w = -1;
        for (int c = 0; c < 2; ++c) if (used[c] + bits <= 64) { w = c; break; }
        if (w < 0) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: group keys exceed 128 bits", who);
        L->word[k] = w; L->shift[k] = used[w]; L->bytes[k] = bits / 8; L->dtype[k] = d->key_dtype[k];
        used[w] += bits;
        if (w == 1) L->nwords = 2;
    }
    return 0;
}

__global__ void __launch_bounds__(256) k_ha_init(State S, int64_t cap, int nagg, const __grid_constant__ qk_hashagg_desc D) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < cap; i += (int64_t)gridDim.x * blockDim.x) {
        S.tag[i] = TAG_EMPTY; S.cnt[i] = 0;
        for (int j = 0; j < nagg; ++j)
            S.acc[i * nagg + j] = D.agg_op[j] == QK_AGG_MIN ? __longlong_as_double(0x7ff0000000000000LL)
                                : D.agg_op[j] == QK_AGG_MAX ? __longlong_as_double(0xfff0000000000000LL) : 0.0;
    }
}

struct UpdArgs {
    const void* key[4];
    const double* val[QK_MAX_AGGS];
    int32_t agg_op[QK_MAX_AGGS];
    int32_t nagg;
};

__device__ __forceinline__ uint64_t key_bits(const void* p, int dt, int64_t i) {
    switch (dt) {
        case QK_U8: return ((const uint8_t*)p)[i];
        case QK_I32: return ((const uint32_t*)p)[i];
        default: return ((const uint64_t*)p)[i];
    }
}

__device__ __forceinline__ void atomic_minmax(double* addr, double v, bool is_min) {
    unsigned long long* a = (unsigned long long*)addr;
    unsigned long long old = *a;
    while (true) {
        const double cur = __longlong_as_double((long long)old);
        if (is_min ? !(v < cur) : !(v > cur)) return;
        const unsigned long long prev = atomicCAS(a, old, (unsigned long long)__double_as_longlong(v));
        if (prev == old) return;
        old = prev;
    }
}

__global__ void __launch_bounds__(256) k_ha_update(State S, uint64_t mask, const __grid_constant__ KeyLayout L,
                                                   const __grid_constant__ UpdArgs U, int64_t n, int* overflow) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        uint64_t w0 = 0, w1 = 0;
        for (int k = 0; k < L.nkeys; ++k) {
            const uint64_t b = key_bits(U.key[k], L.dtype[k], i) << L.shift[k];
            if (L.word[k] == 0) w0 |= b; else w1 |= b;
        }
        uint64_t s = mix64(w0 ^ mix64(w1 + 0x9E3779B97F4A7C15ULL)) & mask;
        int64_t found = -1;
        for (uint64_t tries = 0; tries <= mask;) {
            unsigned t = *(volatile unsigned*)&S.tag[s];
            if (t == TAG_EMPTY) {
                t = atomicCAS(&S.tag[s], TAG_EMPTY, TAG_BUSY);
                if (t == TAG_EMPTY) {
                    S.k0[s] = w0;
                    if (L.nwords == 2) S.k1[s] = w1;
                    __threadfence();
                    *(volatile unsigned*)&S.tag[s] = TAG_READY;
                    found = (int64_t)s;
                    break;
                }
            }
            if (t == TAG_BUSY) continue;                 // owner is storing the key: look again
            // TAG_READY
            __threadfence();
            const bool same = *(volatile unsigned long long*)&S.k0[s] == w0 &&
                              (L.nwords == 1 || *(volatile unsigned long long*)&S.k1[s] == w1);
            if (same) { found = (int64_t)s; break; }
            s = (s + 1) & mask;
            ++tries;
        }
        if (found < 0) { if (overflow) atomicExch(overflow, 1); continue; }
        atomicAdd((unsigned long long*)&S.cnt[found], 1ull);
        for (int j = 0; j < U.nagg; ++j) {
            const double v = U.val[j][i];
            double* a = &S.acc[found * U.nagg + j];
            if (U.agg_op[j] == QK_AGG_SUM) atomicAdd(a, v);
            else atomic_minmax(a, v, U.agg_op[j] == QK_AGG_MIN);
        }
    }
}

struct FinArgs {
    void* key_out[4];
    double* val_out[QK_MAX_AGGS];
    int32_t nagg;
};

__global__ void __launch_bounds__(256) k_ha_finalize(State S, int64_t cap, const __grid_constant__ KeyLayout L,
                                                     const __grid_constant__ FinArgs F, long long* out_cnt, int64_t out_cap,
                                                     unsigned long long* out_groups) {
    const int64_t nround = (cap + 31) / 32 * 32;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nround; i += (int64_t)gridDim.x * blockDim.x) {
        const bool occ = i < cap && S.tag[i] == TAG_READY;
        const unsigned m = __ballot_sync(0xffffffffu, occ);
        if (m == 0) continue;
        unsigned long long base = 0;
        if (lane_id() == 0) base = atomicAdd(out_groups, (unsigned long long)__popc(m));
        base = __shfl_sync(0xffffffffu, base, 0);
        if (!occ) continue;
        const int64_t pos = (int64_t)base + __popc(m & lanemask_lt());
        if (pos >= out_cap) continue;
        const uint64_t w0 = S.k0[i], w1 = L.nwords == 2 ? S.k1[i] : 0;
        for (int k = 0; k < L.nkeys; ++k) {
            const uint64_t w = (L.word[k] == 0 ? w0 : w1) >> L.shift[k];
            switch (L.dtype[k]) {
                case QK_U8: ((uint8_t*)F.key_out[k])[pos] = (uint8_t)w; break;
                case QK_I32: ((uint32_t*)F.key_out[k])[pos] = (uint32_t)w; break;
                default: ((uint64_t*)F.key_out[k])[pos] = w; break;
            }
        }
        for (int j = 0; j < F.nagg; ++j) F.val_out[j][pos] = S.acc[i * F.nagg + j];
        if (out_cnt) out_cnt[pos] = S.cnt[i];
    }
}

}  // namespace
}  // namespace qk

using namespace qk;

extern "C" size_t qk_hashagg_state_bytes(const qk_hashagg_desc* desc) {
    if (!desc || desc->capacity <= 0) return 0;
    State S;
    return carve(desc, nullptr, S);
}

extern "C" int qk_hashagg_init(const qk_hashagg_desc* desc, void* state, void* stream) {
    KeyLayout L;
    if (int rc = make_layout(desc, &L, "qk_hashagg_init")) return rc;
    if (!state || ((uintptr_t)state & 15)) QK_FAIL(QK_ERR_INVALID, "qk_hashagg_init: state must be a 16-byte aligned device buffer");
    State S; carve(desc, state, S);
    k_ha_init<<<grid_size(desc->capacity, 16), 256, 0, (cudaStream_t)stream>>>(S, desc->capacity, desc->nagg, *desc);
    QK_LAUNCH_CHECK("k_ha_init");
    return QK_OK;
}

extern "C" int qk_hashagg_update(const qk_hashagg_desc* desc, void* state, const qk_column* keys, const qk_column* vals,
                                 int64_t nrows, int32_t* overflow, void* stream) {
    const char* who = "qk_hashagg_update";
    KeyLayout L;
    if (int rc = make_layout(desc, &L, who)) return rc;
    if (!state || !keys || (desc->nagg > 0 && !vals)) QK_FAIL(QK_ERR_INVALID, "%s: null arguments", who);
    if (nrows < 0 || nrows > 0x7fffffffLL) QK_FAIL(QK_ERR_INVALID, "%s: nrows out of range", who);
    UpdArgs U{};
    for (int k = 0; k < desc->nkeys; ++k) {
        if (int rc = check_col(&keys[k], who)) return rc;
        if (keys[k].dtype != desc->key_dtype[k] || keys[k].length != nrows) QK_FAIL(QK_ERR_INVALID, "%s: key column %d does not match the descriptor", who, k);
        U.key[k] = keys[k].data;
    }
    for (int j = 0; j < desc->nagg; ++j) {
        if (int rc = check_col(&vals[j], who)) return rc;
        if (vals[j].dtype != QK_F64 || vals[j].length != nrows) QK_FAIL(QK_ERR_INVALID, "%s: value column %d must be fp64 with %lld rows", who, j, (long long)nrows);
        U.val[j] = (const double*)vals[j].data; U.agg_op[j] = desc->agg_op[j];
    }
    U.nagg = desc->nagg;
    if (nrows == 0) return QK_OK;
    State S; carve(desc, state, S);
    k_ha_update<<<grid_size(nrows, 16), 256, 0, (cudaStream_t)stream>>>(S, (uint64_t)desc->capacity - 1, L, U, nrows, overflow);
    QK_LAUNCH_CHECK("k_ha_update");
    return QK_OK;
}

extern "C" int qk_hashagg_finalize(const qk_hashagg_desc* desc, const void* state, qk_column* out_keys, qk_column* out_vals,
                                   int64_t* out_cnt, int64_t out_capacity, int64_t* out_groups, void* stream) {
    const char* who = "qk_hashagg_finalize";
    KeyLayout L;
    if (int rc = make_layout(desc, &L, who)) return rc;
    if (!state || !out_keys || !out_groups || out_capacity < 0 || (desc->nagg > 0 && !out_vals)) QK_FAIL(QK_ERR_INVALID, "%s: null arguments", who);
    FinArgs F{};
    for (int k = 0; k < desc->nkeys; ++k) {
        if (out_keys[k].dtype != desc->key_dtype[k] || out_keys[k].length < out_capacity || (out_capacity > 0 && !out_keys[k].data))
            QK_FAIL(QK_ERR_INVALID, "%s: key output %d does not match the descriptor / capacity", who, k);
        F.key_out[k] = (void*)out_keys[k].data;
    }
    for (int j = 0; j < desc->nagg; ++j) {
        if (out_vals[j].dtype != QK_F64 || out_vals[j].length < out_capacity || (out_capacity > 0 && !out_vals[j].data))
            QK_FAIL(QK_ERR_INVALID, "%s: value output %d must be fp64 with room for out_capacity rows", who, j);
        F.val_out[j] = (double*)out_vals[j].data;
    }
    F.nagg = desc->nagg;
    cudaStream_t st = (cudaStream_t)stream;
    QK_CUDA(cudaMemsetAsync(out_groups, 0, sizeof(int64_t), st));
    State S; carve(desc, (void*)state, S);
    k_ha_finalize<<<grid_size(desc->capacity, 16), 256, 0, st>>>(S, desc->capacity, L, F, (long long*)out_cnt, out_capacity, (unsigned long long*)out_groups);
    QK_LAUNCH_CHECK("k_ha_finalize");
    return QK_OK;
}
