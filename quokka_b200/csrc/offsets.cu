// offsets.cu -- counts -> exclusive offsets, the middle pass of every stable two-pass operator (count per chunk, scan the
// counts, rank each row inside its chunk): the interpreter's filter (scan.cu), the TMA compaction (compact.cu), the
// partition plan (partition.cu) and the session ids (window.cu).
#include "common.cuh"

namespace qk {
namespace {

// CTA b scans row b in tiles of blockDim.x counts (a multiple of 32, at most 1024): a warp scan, then warp 0 scans the
// warp totals; wtot[32] carries the tile total to every thread.  Two barriers per tile are enough: before the next
// tile's first barrier a warp writes only its own slot, and no other warp is still reading that slot.
template <typename T>
__global__ void __launch_bounds__(1024) k_count_offsets(const T* counts, int64_t n, int64_t* offsets, int64_t* totals) {
    __shared__ int64_t wtot[33];
    const T* in = counts + (int64_t)blockIdx.x * n;
    int64_t* out = offsets + (int64_t)blockIdx.x * n;
    const int warp = threadIdx.x >> 5, lane = lane_id(), nw = blockDim.x >> 5;
    int64_t carry = 0;
    for (int64_t base = 0; base < n; base += blockDim.x) {
        const int64_t i = base + threadIdx.x;
        const int64_t v = i < n ? (int64_t)in[i] : 0, x = warp_inclusive_scan(v);
        if (lane == 31) wtot[warp] = x;
        __syncthreads();
        if (warp == 0) {
            const int64_t w = lane < nw ? wtot[lane] : 0, t = warp_inclusive_scan(w);
            wtot[lane] = t - w;
            if (lane == 31) wtot[32] = t;
        }
        __syncthreads();
        if (i < n) out[i] = carry + wtot[warp] + x - v;
        carry += wtot[32];
    }
    if (threadIdx.x == 0) totals[blockIdx.x] = carry;
}

}  // namespace

template <typename T>
int count_offsets(const T* counts, int64_t rows, int64_t n, int64_t* offsets, int64_t* totals, cudaStream_t st) {
    const int64_t width = n < 32 ? 32 : (n > 1024 ? 1024 : n);           // as wide as the row, 32 to 1024 threads
    k_count_offsets<T><<<(unsigned)rows, (unsigned)(width + 31) / 32 * 32, 0, st>>>(counts, n, offsets, totals);
    QK_LAUNCH_CHECK("k_count_offsets");
    return QK_OK;
}
template int count_offsets<uint32_t>(const uint32_t*, int64_t, int64_t, int64_t*, int64_t*, cudaStream_t);
template int count_offsets<int64_t>(const int64_t*, int64_t, int64_t, int64_t*, int64_t*, cudaStream_t);

}  // namespace qk
