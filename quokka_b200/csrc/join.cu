// join.cu -- K4 hash build / K5 hash probe (BuildProbeJoinExecutor, sql_executors.py:325-377).
//
// Open addressing, linear probing, 16-byte slots {int64 key, int32 build_row, pad}: one 16-byte load
// fetches key and payload index, and a probe touches one 32-byte DRAM sector in the common case.
// Bound: HBM random access -- 16 B/build row written, >= 32 B sector per probe row read (DESIGN.md).
// Duplicate build keys each own a slot (Polars multiplies rows); the probe counts matches first, a warp
// shuffle scan turns counts into offsets and ONE atomic per warp reserves output space (ballot/shfl
// conflict resolution instead of one atomic per row), then the chain is re-walked (L1/L2 hits) to write.
#include "common.cuh"

namespace qk {
namespace {

constexpr long long EMPTY_KEY = (long long)0x8000000000000000ULL;
struct __align__(16) Slot { long long key; int idx; int pad; };

__global__ void __launch_bounds__(256) k_join_init(Slot* slots, int64_t capacity) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < capacity; i += (int64_t)gridDim.x * blockDim.x)
        slots[i] = Slot{EMPTY_KEY, -1, 0};
}

__global__ void __launch_bounds__(256) k_join_build(Slot* slots, uint64_t mask, const void* key, int dt, int64_t n,
                                                    int row_base, int* flags) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const long long k = load_i64(key, dt, i);
        if (k == EMPTY_KEY) { if (flags) atomicOr(flags, 2); continue; }
        uint64_t s = mix64((uint64_t)k) & mask;
        bool placed = false;
        for (uint64_t tries = 0; tries <= mask; ++tries) {
            const long long old = (long long)atomicCAS((unsigned long long*)&slots[s].key, (unsigned long long)EMPTY_KEY, (unsigned long long)k);
            if (old == EMPTY_KEY) { slots[s].idx = row_base + (int)i; placed = true; break; }
            if (old == k && flags) atomicOr(flags, 4);
            s = (s + 1) & mask;
        }
        if (!placed && flags) atomicOr(flags, 1);
    }
}

__device__ __forceinline__ Slot load_slot(const Slot* p) {
    const int4 v = *reinterpret_cast<const int4*>(p);
    Slot s;
    s.key = ((long long)(unsigned)v.y << 32) | (unsigned)v.x;
    s.idx = v.z; s.pad = 0;
    return s;
}

__global__ void __launch_bounds__(256) k_join_probe(const Slot* slots, uint64_t mask, const void* key, int dt, int64_t n, int how,
                                                    int* out_probe, int* out_build, int64_t cap, unsigned long long* out_count) {
    const int64_t nround = (n + 31) / 32 * 32;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nround; i += (int64_t)gridDim.x * blockDim.x) {
        const bool valid = i < n;
        long long k = 0;
        uint64_t s0 = 0;
        int matches = 0;
        if (valid) {
            k = load_i64(key, dt, i);
            s0 = mix64((uint64_t)k) & mask;
            if (k != EMPTY_KEY) {
                uint64_t s = s0;
                for (uint64_t tries = 0; tries <= mask; ++tries) {
                    const Slot sl = load_slot(&slots[s]);
                    if (sl.key == EMPTY_KEY) break;
                    if (sl.key == k) { matches++; if (how >= QK_JOIN_SEMI) break; }
                    s = (s + 1) & mask;
                }
            }
        }
        int emit;
        switch (how) {
            case QK_JOIN_INNER: emit = matches; break;
            case QK_JOIN_LEFT: emit = valid ? (matches > 0 ? matches : 1) : 0; break;
            case QK_JOIN_SEMI: emit = matches > 0 ? 1 : 0; break;
            default: emit = (valid && matches == 0) ? 1 : 0; break;
        }
        const int x = warp_inclusive_scan(emit);
        const int total = __shfl_sync(0xffffffffu, x, 31);
        if (total == 0) continue;
        unsigned long long base = 0;
        if (lane_id() == 31) base = atomicAdd(out_count, (unsigned long long)total);
        base = __shfl_sync(0xffffffffu, base, 31);
        int64_t pos = (int64_t)base + x - emit;
        if (emit == 0) continue;
        if (how == QK_JOIN_SEMI || how == QK_JOIN_ANTI || matches == 0) {
            if (pos < cap) { out_probe[pos] = (int)i; if (out_build) out_build[pos] = -1; }
            continue;
        }
        uint64_t s = s0;
        for (uint64_t tries = 0; tries <= mask; ++tries) {
            const Slot sl = load_slot(&slots[s]);
            if (sl.key == EMPTY_KEY) break;
            if (sl.key == k) {
                if (pos < cap) { out_probe[pos] = (int)i; out_build[pos] = sl.idx; }
                pos++;
            }
            s = (s + 1) & mask;
        }
    }
}

bool pow2(int64_t x) { return x > 0 && (x & (x - 1)) == 0; }

}  // namespace
}  // namespace qk

using namespace qk;

extern "C" size_t qk_join_table_bytes(int64_t capacity) { return capacity > 0 ? (size_t)capacity * sizeof(Slot) : 0; }

extern "C" int qk_join_init(void* table, int64_t capacity, void* stream) {
    if (!table || !pow2(capacity)) QK_FAIL(QK_ERR_INVALID, "qk_join_init: table null or capacity %lld not a power of two", (long long)capacity);
    if (((uintptr_t)table & 15) != 0) QK_FAIL(QK_ERR_INVALID, "qk_join_init: table must be 16-byte aligned");
    k_join_init<<<grid_size(capacity, 16), 256, 0, (cudaStream_t)stream>>>((Slot*)table, capacity);
    QK_LAUNCH_CHECK("k_join_init");
    return QK_OK;
}

extern "C" int qk_join_build(void* table, int64_t capacity, const qk_column* key, int32_t row_base, int32_t* flags, void* stream) {
    const char* who = "qk_join_build";
    if (!table || !pow2(capacity)) QK_FAIL(QK_ERR_INVALID, "%s: bad table / capacity", who);
    if (int rc = check_col(key, who)) return rc;
    if (!dtype_is_int(key->dtype)) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: join keys must be integer columns", who);
    if (row_base < 0 || (int64_t)row_base + key->length > 0x7fffffffLL) QK_FAIL(QK_ERR_INVALID, "%s: build row numbers exceed int32", who);
    if (key->length == 0) return QK_OK;
    k_join_build<<<grid_size(key->length, 16), 256, 0, (cudaStream_t)stream>>>((Slot*)table, (uint64_t)capacity - 1, key->data, key->dtype, key->length, row_base, flags);
    QK_LAUNCH_CHECK("k_join_build");
    return QK_OK;
}

extern "C" int qk_join_probe(const void* table, int64_t capacity, const qk_column* key, int32_t how, int32_t* out_probe_idx,
                             int32_t* out_build_idx, int64_t out_capacity, int64_t* out_count, void* stream) {
    const char* who = "qk_join_probe";
    if (!table || !pow2(capacity)) QK_FAIL(QK_ERR_INVALID, "%s: bad table / capacity", who);
    if (int rc = check_col(key, who)) return rc;
    if (!dtype_is_int(key->dtype)) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: join keys must be integer columns", who);
    if (how < QK_JOIN_INNER || how > QK_JOIN_ANTI) QK_FAIL(QK_ERR_INVALID, "%s: bad join type %d", who, how);
    if (!out_count || out_capacity < 0 || (out_capacity > 0 && !out_probe_idx)) QK_FAIL(QK_ERR_INVALID, "%s: bad output arguments", who);
    if ((how == QK_JOIN_INNER || how == QK_JOIN_LEFT) && out_capacity > 0 && !out_build_idx) QK_FAIL(QK_ERR_INVALID, "%s: inner/left joins need out_build_idx", who);
    cudaStream_t st = (cudaStream_t)stream;
    QK_CUDA(cudaMemsetAsync(out_count, 0, sizeof(int64_t), st));
    if (key->length == 0) return QK_OK;
    k_join_probe<<<grid_size(key->length, 16), 256, 0, st>>>((const Slot*)table, (uint64_t)capacity - 1, key->data, key->dtype, key->length, how,
                                               out_probe_idx, out_build_idx, out_capacity, (unsigned long long*)out_count);
    QK_LAUNCH_CHECK("k_join_probe");
    return QK_OK;
}
