// topk.cu -- K8 top-k candidates by radix select (DataStream.top_k, datastream.py:1746-1767).
//
// The primary sort column is mapped to an order-preserving 64-bit image (flipped for ascending order so
// "best" is always "largest"), eight 8-bit histogram passes find the k-th largest image exactly, and one
// compaction pass emits every row at or above it (ties included).  The handful of survivors is ordered on
// all sort columns by the host.  Negligible next to the scan (a8 in SURVEY.md section 8): ~9 reads of
// 8 B/row over the group table (~1.16 M rows for Q3 at SF-100).
#include "common.cuh"

namespace qk {
namespace {

struct SelState { unsigned long long prefix; long long k_rem; unsigned hist[256]; };

// The order is DuckDB's ORDER BY (DESIGN.md section 2): -0.0 = +0.0, and every NaN, whatever its sign and payload, is
// greater than +inf -- so -0.0 is folded onto +0.0 and a NaN takes the greatest image before the ascending flip.
__device__ __forceinline__ unsigned long long image_of(const void* p, int dt, int64_t i, int descending) {
    unsigned long long u;
    switch (dt) {
        case QK_F64: {
            unsigned long long b = ((const unsigned long long*)p)[i];
            if (b == 0x8000000000000000ULL) b = 0;
            u = (b << 1) > 0xffe0000000000000ULL ? ~0ULL : (b >> 63) ? ~b : (b | 0x8000000000000000ULL);
        } break;
        case QK_F32: {
            unsigned b = ((const unsigned*)p)[i];
            if (b == 0x80000000u) b = 0;
            const unsigned v = (b << 1) > 0xff000000u ? ~0u : (b >> 31) ? ~b : (b | 0x80000000u);
            u = (unsigned long long)v << 32;
        } break;
        case QK_I64: u = ((const unsigned long long*)p)[i] ^ 0x8000000000000000ULL; break;
        case QK_I32: u = (unsigned long long)(((const unsigned*)p)[i] ^ 0x80000000u) << 32; break;
        default: u = (unsigned long long)((const uint8_t*)p)[i] << 56; break;
    }
    return descending ? u : ~u;
}

__global__ void __launch_bounds__(256) k_topk_image(const void* p, int dt, int64_t n, int descending, unsigned long long* img) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        img[i] = image_of(p, dt, i, descending);
}
__global__ void k_topk_reset(SelState* S, long long k) {
    if (threadIdx.x == 0) { S->prefix = 0; S->k_rem = k; }
    S->hist[threadIdx.x] = 0;
}
// histogram of byte `pass` (0 = most significant) among rows whose higher bytes equal the prefix
__global__ void __launch_bounds__(256) k_topk_hist(const unsigned long long* img, int64_t n, int pass, SelState* S) {
    __shared__ unsigned sh[256];
    sh[threadIdx.x] = 0;
    __syncthreads();
    const unsigned long long prefix = S->prefix;
    const int shift = 56 - 8 * pass;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const unsigned long long v = img[i];
        const bool in = pass == 0 || (v >> (shift + 8)) == prefix;
        if (in) atomicAdd(&sh[(v >> shift) & 0xff], 1u);
    }
    __syncthreads();
    if (sh[threadIdx.x]) atomicAdd(&S->hist[threadIdx.x], sh[threadIdx.x]);
}
__global__ void k_topk_pick(SelState* S) {
    if (threadIdx.x == 0) {
        long long k = S->k_rem;
        int b = 255;
        for (; b > 0; --b) {
            if ((long long)S->hist[b] >= k) break;
            k -= S->hist[b];
        }
        S->prefix = (S->prefix << 8) | (unsigned)b;
        S->k_rem = k;
    }
    __syncthreads();
    S->hist[threadIdx.x] = 0;
}
__global__ void __launch_bounds__(256) k_topk_emit(const unsigned long long* img, int64_t n, const SelState* S, int take_all,
                                                   int32_t* out_idx, unsigned long long* out_n) {
    const unsigned long long thr = take_all ? 0ull : S->prefix;
    const int64_t nround = (n + 31) / 32 * 32;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nround; i += (int64_t)gridDim.x * blockDim.x) {
        const bool keep = i < n && img[i] >= thr;
        const unsigned m = __ballot_sync(0xffffffffu, keep);
        if (m == 0) continue;
        unsigned long long base = 0;
        if (lane_id() == 0) base = atomicAdd(out_n, (unsigned long long)__popc(m));
        base = __shfl_sync(0xffffffffu, base, 0);
        if (keep) out_idx[base + __popc(m & lanemask_lt())] = (int32_t)i;
    }
}

}  // namespace
}  // namespace qk

using namespace qk;

extern "C" size_t qk_topk_workspace_bytes(int64_t nrows) {
    if (nrows < 0) return 0;
    return align_up((size_t)nrows * 8, 256) + align_up(sizeof(SelState), 256);
}

extern "C" int qk_topk_candidates(const qk_column* key, int32_t k, int32_t descending, int32_t* out_idx,
                                  int64_t* out_n, void* workspace, size_t ws_bytes, void* stream) {
    const char* who = "qk_topk_candidates";
    if (int rc = check_col(key, who)) return rc;
    if (k <= 0) QK_FAIL(QK_ERR_INVALID, "%s: k must be positive", who);
    if (!out_n) QK_FAIL(QK_ERR_INVALID, "%s: null out_n", who);
    cudaStream_t st = (cudaStream_t)stream;
    QK_CUDA(cudaMemsetAsync(out_n, 0, sizeof(int64_t), st));
    const int64_t n = key->length;
    if (n == 0) return QK_OK;
    if (!out_idx) QK_FAIL(QK_ERR_INVALID, "%s: null out_idx", who);
    if (!workspace || ws_bytes < qk_topk_workspace_bytes(n)) QK_FAIL(QK_ERR_CAPACITY, "%s: workspace too small", who);
    unsigned long long* img = (unsigned long long*)workspace;
    SelState* S = (SelState*)((char*)workspace + align_up((size_t)n * 8, 256));
    int64_t nb = (n + 255) / 256;
    if (nb > (int64_t)sm_count() * 8) nb = (int64_t)sm_count() * 8;
    k_topk_image<<<(unsigned)nb, 256, 0, st>>>(key->data, key->dtype, n, descending, img);
    QK_LAUNCH_CHECK("k_topk_image");
    const int take_all = n <= k;
    if (!take_all) {
        k_topk_reset<<<1, 256, 0, st>>>(S, k);
        QK_LAUNCH_CHECK("k_topk_reset");
        for (int pass = 0; pass < 8; ++pass) {
            k_topk_hist<<<(unsigned)nb, 256, 0, st>>>(img, n, pass, S);
            QK_LAUNCH_CHECK("k_topk_hist");
            k_topk_pick<<<1, 256, 0, st>>>(S);
            QK_LAUNCH_CHECK("k_topk_pick");
        }
    }
    k_topk_emit<<<(unsigned)nb, 256, 0, st>>>(img, n, S, take_all, out_idx, (unsigned long long*)out_n);
    QK_LAUNCH_CHECK("k_topk_emit");
    return QK_OK;
}
