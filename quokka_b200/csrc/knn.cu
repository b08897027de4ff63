// knn.cu -- K11: nearest neighbours of a set of probes in a vector column, by cosine similarity (DataStream.vector_nn_join).
//
// Replaces the per-batch `np.dot(normalized_vectors, query_vecs.T)` + `argsort` of DFProbeDataStreamNNExecutor1
// (pyquokka/executors/vector_executors.py:8-52).  Scores and selection are fused: the n x q score matrix (40 GB of fp32 for
// 10 M rows x 1 000 probes) is never written.
//
//   k_knn_scan   grid (probe tile, row slice).  A CTA walks its 128-row tiles; every tile is staged into shared memory in
//                chunks of KC elements by cp.async (16-byte copies when the column allows it), double-buffered so the next
//                chunk lands while the current one is multiplied.  Dot products run on the tensor cores: mma.sync m16n8k8
//                TF32 with 3xTF32 splitting (x_lo p_hi + x_hi p_lo + x_hi p_hi, f32 accumulation); an f16 row is exact in
//                TF32, so f16 input runs the two probe terms only.  The squared row norm accumulates in fp64 from the staged
//                chunk.  Scores s = dot / sqrt(norm2) that beat a probe's current k-th best are appended to a per-probe
//                candidate buffer in shared memory; after the tile one warp per probe inserts them into the probe's sorted
//                top-k list.  The CTA's lists go to the workspace.
//   k_knn_fold   one warp per probe folds the per-CTA lists in CTA order.
//
// Determinism: the dot of (row, probe) is the same chain of MMAs (k-steps of 8 elements in order, three terms in a fixed order)
// whatever the row's slot in the tile, and the squared norm is the sum over KC-element chunks of (h0 + h1), h_i the fp64 FMA
// chain over 16 elements: neither depends on where the row lies, on the tile shape or on the grid.  Selection is by the total order (score desc, row asc), so the
// output does not depend on the order in which candidates arrive.
#include "common.cuh"

#include <math.h>

namespace qk {
namespace {

constexpr int KNN_NT = 256;
constexpr int KC = 32;                  // elements per staged chunk
constexpr unsigned FULL = 0xffffffffu;

__device__ __forceinline__ bool better(float sa, long long ka, float sb, long long kb) {
    return sa > sb || (sa == sb && ka < kb);
}

// Inserts (s, r) into the sorted list ls / lr of m entries (capacity k) with the whole warp; returns the new length.
__device__ __forceinline__ int warp_insert(float* ls, int* lr, int m, int k, float s, int r, unsigned lane) {
    if (m == k && !better(s, r, ls[k - 1], lr[k - 1])) return m;
    int pos = 0;
    for (int b = 0; b < m; b += 32) {
        const int i = b + (int)lane;
        const bool bt = i < m && better(ls[i], lr[i], s, r);
        pos += __popc(__ballot_sync(FULL, bt));
    }
    const int newm = m + 1 < k ? m + 1 : k;
    for (int b = ((newm - 1) / 32) * 32; b >= (pos / 32) * 32; b -= 32) {      // shift [pos, newm - 1) up by one, top chunk first
        const int i = b + (int)lane;
        const bool mv = i >= pos && i < newm - 1;
        float sv = 0.f; int rv = 0;
        if (mv) { sv = ls[i]; rv = lr[i]; }
        __syncwarp();
        if (mv) { ls[i + 1] = sv; lr[i + 1] = rv; }
        __syncwarp();
    }
    if (lane == 0) { ls[pos] = s; lr[pos] = r; }
    __syncwarp();
    return newm;
}

constexpr int RT = 128;                 // rows per tile
constexpr int XS = KC + 4;              // f32 stride of a staged row chunk (words): conflict-free fragment loads, 16-byte rows
constexpr int HS = KC + 8;              // f16 stride (halves)

// WROWS warps along the rows, 8 / WROWS along the probes; a warp owns WM m16 tiles x WN n8 tiles
template <int WROWS_, int WM_, int WN_>
struct Cfg {
    static constexpr int WROWS = WROWS_, WM = WM_, WN = WN_;
    static constexpr int PT = 8 * WN * (8 / WROWS);          // probes per CTA
    static_assert(16 * WM * WROWS == RT, "a CTA covers one row tile");
    __host__ __device__ static constexpr size_t xbuf(int esize) { return esize == 4 ? (size_t)RT * XS * 4 : (size_t)RT * HS * 2; }
    static size_t smem(int k, int esize) {
        return 2 * xbuf(esize) + 2 * (size_t)PT * XS * 4 + (size_t)RT * 8      // X and probe chunks (double-buffered), norm2 (fp64)
               + (size_t)PT * k * 8 + (size_t)PT * RT * 8 + (size_t)PT * 16;  // lists, candidates, counts + thresholds
    }
};
using Small = Cfg<8, 1, 1>;             // 128 rows x 8 probes: q <= 8
using Large = Cfg<4, 2, 2>;             // 128 rows x 32 probes

struct KnnArgs {
    const void* x;
    const float* probes;
    float* ws_score;
    int32_t* ws_row;
    long long n;
    int d, q, k;
    int row_ctas;
};

__device__ __forceinline__ unsigned smem_addr(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void cp_async16(void* dst, const void* src, int src_bytes) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_addr(dst)), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async4(void* dst, const void* src, int src_bytes) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(smem_addr(dst)), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ unsigned tf32_hi(float x) { unsigned r; asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x)); return r; }
__device__ __forceinline__ void split(float x, unsigned& hi, unsigned& lo) {
    hi = tf32_hi(x);
    lo = tf32_hi(__fsub_rn(x, __uint_as_float(hi)));       // x - hi is exact
}
__device__ __forceinline__ void mma_tf32(float* c, const unsigned* a, unsigned b0, unsigned b1) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ float half_to_f32(unsigned short h) { float f; asm("cvt.f32.f16 %0, %1;" : "=f"(f) : "h"(h)); return f; }

// Rows [r0, r0 + RT) x elements [k0, k0 + KC) of X into a shared chunk (zeros past n / d), and the probe chunk.  VEC: 16-byte
// cp.async (X 16-byte aligned, rows a multiple of 16 bytes); otherwise 4-byte cp.async (f32) or plain loads (f16).
template <class T, bool VEC, class C>
__device__ __forceinline__ void stage(const KnnArgs& A, long long r0, int k0, int p0, void* xbuf, float* pbuf) {
    const int tid = threadIdx.x, d = A.d;
    if constexpr (sizeof(T) == 4) {
        const float* X = (const float*)A.x;
        float* xs = (float*)xbuf;
        if constexpr (VEC) {
#pragma unroll
            for (int m = 0; m < RT * KC / 4 / KNN_NT; ++m) {
                const int seg = tid + m * KNN_NT, row = seg / (KC / 4), e0 = k0 + (seg % (KC / 4)) * 4;
                const long long gr = r0 + row;
                const int bytes = gr < A.n ? max(0, min(16, (d - e0) * 4)) : 0;
                cp_async16(xs + row * XS + (e0 - k0), bytes ? (const void*)(X + gr * d + e0) : (const void*)X, bytes);
            }
        } else {
#pragma unroll 4
            for (int m = 0; m < RT * KC / KNN_NT; ++m) {
                const int e = tid + m * KNN_NT, row = e / KC, kk = e % KC;
                const long long gr = r0 + row;
                const int bytes = (gr < A.n && k0 + kk < d) ? 4 : 0;
                cp_async4(xs + row * XS + kk, bytes ? (const void*)(X + gr * d + k0 + kk) : (const void*)X, bytes);
            }
        }
    } else {
        const unsigned short* X = (const unsigned short*)A.x;
        unsigned short* xs = (unsigned short*)xbuf;
        if constexpr (VEC) {
#pragma unroll
            for (int m = 0; m < RT * KC / 8 / KNN_NT; ++m) {
                const int seg = tid + m * KNN_NT, row = seg / (KC / 8), e0 = k0 + (seg % (KC / 8)) * 8;
                const long long gr = r0 + row;
                const int bytes = gr < A.n ? max(0, min(16, (d - e0) * 2)) : 0;
                cp_async16(xs + row * HS + (e0 - k0), bytes ? (const void*)(X + gr * d + e0) : (const void*)X, bytes);
            }
        } else {
#pragma unroll 4
            for (int m = 0; m < RT * KC / KNN_NT; ++m) {
                const int e = tid + m * KNN_NT, row = e / KC, kk = e % KC;
                const long long gr = r0 + row;
                xs[row * HS + kk] = (gr < A.n && k0 + kk < d) ? X[gr * d + k0 + kk] : (unsigned short)0;
            }
        }
    }
    for (int e = tid; e < C::PT * KC; e += KNN_NT) {
        const int p = e / KC, kk = e % KC;
        const int bytes = (p0 + p < A.q && k0 + kk < d) ? 4 : 0;
        cp_async4(pbuf + p * XS + kk, bytes ? (const void*)(A.probes + (long long)(p0 + p) * d + k0 + kk) : (const void*)A.probes, bytes);
    }
}

template <class T>
__device__ __forceinline__ float staged(const void* xbuf, int row, int kk) {
    if constexpr (sizeof(T) == 4) return ((const float*)xbuf)[row * XS + kk];
    else return half_to_f32(((const unsigned short*)xbuf)[row * HS + kk]);
}

template <class T, bool VEC, class C>
__global__ void __launch_bounds__(KNN_NT, 1) k_knn_scan(const __grid_constant__ KnnArgs A) {
    constexpr int PT = C::PT, WM = C::WM, WN = C::WN;
    constexpr bool F32 = sizeof(T) == 4;
    extern __shared__ __align__(16) unsigned char smem[];
    const size_t xb = C::xbuf(sizeof(T));
    float* pbuf0 = (float*)(smem + 2 * xb);                   // [2][PT][XS]; X chunks [2] before it
    double* nrm = (double*)(pbuf0 + 2 * PT * XS);             // [RT]
    float* ls = (float*)(nrm + RT);                           // [PT][k]
    int* lr = (int*)(ls + PT * A.k);                          // [PT][k]
    float* cs = (float*)(lr + PT * A.k);                      // [PT][RT]
    int* cr = (int*)(cs + PT * RT);                           // [PT][RT]
    int* ccnt = cr + PT * RT;                                 // [PT]
    int* lcnt = ccnt + PT;                                    // [PT]
    float* ths = (float*)(lcnt + PT);                         // [PT] k-th best score (-inf while the list is short)
    int* thr = (int*)(ths + PT);                              // [PT] its row

    const int tid = threadIdx.x;
    const unsigned lane = tid & 31, warp = tid >> 5;
    const int gid = lane >> 2, tig = lane & 3;
    const int wrow = (warp % C::WROWS) * 16 * WM, wprobe = (warp / C::WROWS) * 8 * WN;
    const int p0 = blockIdx.x * PT;
    const int k = A.k;
    for (int p = tid; p < PT; p += KNN_NT) { ccnt[p] = 0; lcnt[p] = 0; ths[p] = -INFINITY; thr[p] = 0x7fffffff; }
    const long long ntiles = (A.n + RT - 1) / RT;
    const int nchunks = (A.d + KC - 1) / KC;

    for (long long tile = blockIdx.y; tile < ntiles; tile += A.row_ctas) {
        const long long r0 = tile * RT;
        float acc[WM][WN][4];
#pragma unroll
        for (int i = 0; i < WM; ++i)
#pragma unroll
            for (int j = 0; j < WN; ++j)
#pragma unroll
                for (int e = 0; e < 4; ++e) acc[i][j][e] = 0.f;
        if (tid < RT) nrm[tid] = 0.0;
        stage<T, VEC, C>(A, r0, 0, p0, smem, pbuf0);
        cp_async_commit();
        for (int c = 0; c < nchunks; ++c) {
            if (c + 1 < nchunks) {                           // the next chunk lands while this one is multiplied
                stage<T, VEC, C>(A, r0, (c + 1) * KC, p0, smem + ((c + 1) & 1) * xb, pbuf0 + ((c + 1) & 1) * PT * XS);
                cp_async_commit();
                cp_async_wait<1>();
            } else {
                cp_async_wait<0>();
            }
            __syncthreads();
            const void* xs = smem + (c & 1) * xb;
            const float* ps = pbuf0 + (c & 1) * PT * XS;
            {   // squared norm in fp64: row = tid / 2, half h sums elements [16 h, 16 h + 16) of the chunk in order
                const int row = tid >> 1, h = tid & 1;
                double s = 0.0;
#pragma unroll
                for (int e = 0; e < 16; ++e) { const double v = staged<T>(xs, row, 16 * h + e); s = __fma_rn(v, v, s); }
                const double t2 = __dadd_rn(s, __shfl_xor_sync(FULL, s, 1));
                if (h == 0) nrm[row] = __dadd_rn(nrm[row], t2);
            }
#pragma unroll
            for (int kk = 0; kk < KC; kk += 8) {
                unsigned ahi[WM][4], alo[WM][4];
#pragma unroll
                for (int i = 0; i < WM; ++i) {
                    const int r = wrow + 16 * i + gid;
                    const float v[4] = {staged<T>(xs, r, kk + tig), staged<T>(xs, r + 8, kk + tig), staged<T>(xs, r, kk + tig + 4),
                                        staged<T>(xs, r + 8, kk + tig + 4)};
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        if constexpr (F32) split(v[e], ahi[i][e], alo[i][e]);
                        else ahi[i][e] = __float_as_uint(v[e]);       // an f16 value is exact in TF32: no low part
                    }
                }
#pragma unroll
                for (int j = 0; j < WN; ++j) {
                    const int pr = wprobe + 8 * j + gid;
                    unsigned bh0, bl0, bh1, bl1;
                    split(ps[pr * XS + kk + tig], bh0, bl0);
                    split(ps[pr * XS + kk + tig + 4], bh1, bl1);
#pragma unroll
                    for (int i = 0; i < WM; ++i) {               // small terms first, in a fixed order
                        if constexpr (F32) mma_tf32(acc[i][j], alo[i], bh0, bh1);
                        mma_tf32(acc[i][j], ahi[i], bl0, bl1);
                        mma_tf32(acc[i][j], ahi[i], bh0, bh1);
                    }
                }
            }
            __syncthreads();                                 // this buffer is staged again two chunks later
        }
#pragma unroll
        for (int i = 0; i < WM; ++i)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int row = wrow + 16 * i + gid + (e >= 2 ? 8 : 0);
                const long long gr = r0 + row;
                const double n2 = nrm[row];
                if (gr >= A.n || !(n2 > 0.0) || !isfinite(n2)) continue;
                const double norm = __dsqrt_rn(n2);
#pragma unroll
                for (int j = 0; j < WN; ++j) {
                    const int p = wprobe + 8 * j + 2 * tig + (e & 1);
                    if (p0 + p >= A.q) continue;
                    const float s = (float)__ddiv_rn((double)acc[i][j][e], norm);
                    if (!isfinite(s)) continue;
                    if (better(s, gr, ths[p], thr[p])) {
                        const int slot = atomicAdd(&ccnt[p], 1);
                        cs[p * RT + slot] = s;
                        cr[p * RT + slot] = (int)gr;
                    }
                }
            }
        __syncthreads();
        for (int p = warp; p < PT; p += KNN_NT / 32) {
            const int nc = ccnt[p];
            if (nc == 0) continue;
            int m = lcnt[p];
            for (int c = 0; c < nc; ++c) m = warp_insert(ls + p * k, lr + p * k, m, k, cs[p * RT + c], cr[p * RT + c], lane);
            if (lane == 0) {
                lcnt[p] = m; ccnt[p] = 0;
                if (m == k) { ths[p] = ls[p * k + k - 1]; thr[p] = lr[p * k + k - 1]; }
            }
            __syncwarp();
        }
        __syncthreads();
    }
    __syncthreads();
    for (int p = 0; p < PT && p0 + p < A.q; ++p) {
        const long long base = ((long long)blockIdx.y * A.q + p0 + p) * k;
        for (int i = tid; i < k; i += KNN_NT) {
            const bool ok = i < lcnt[p];
            A.ws_score[base + i] = ok ? ls[p * k + i] : -INFINITY;
            A.ws_row[base + i] = ok ? lr[p * k + i] : -1;
        }
    }
}

// one warp per probe: the per-CTA lists, CTA by CTA, into the final k
__global__ void __launch_bounds__(KNN_NT) k_knn_fold(const float* ws_score, const int32_t* ws_row, int row_ctas, int q, int k,
                                                     float* out_score, int64_t* out_row) {
    extern __shared__ __align__(16) unsigned char smem[];
    const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float* ls = (float*)smem + warp * k;
    int* lr = (int*)((float*)smem + (KNN_NT / 32) * k) + warp * k;
    const int p = blockIdx.x * (KNN_NT / 32) + warp;
    if (p >= q) return;
    int m = 0;
    for (int b = 0; b < row_ctas; ++b) {
        const long long base = ((long long)b * q + p) * k;
        for (int i = 0; i < k; ++i) {
            const int r = ws_row[base + i];
            const float s = ws_score[base + i];
            if (r < 0 || (m == k && !better(s, r, ls[k - 1], lr[k - 1]))) break;    // each list is sorted
            m = warp_insert(ls, lr, m, k, s, r, lane);
        }
    }
    for (int i = lane; i < k; i += 32) {
        out_score[(long long)p * k + i] = i < m ? ls[i] : -INFINITY;
        out_row[(long long)p * k + i] = i < m ? (int64_t)lr[i] : -1;
    }
}

// one thread per probe: two sorted candidate lists into the best k
__global__ void __launch_bounds__(128) k_knn_merge(int q, const float* as, const int64_t* ak, int ka, const float* bs, const int64_t* bk,
                                                  int kb, int k, float* os, int64_t* ok, int32_t* osrc) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= q) return;
    int i = 0, j = 0;
    for (int o = 0; o < k; ++o) {
        const bool ha = i < ka && ak[(long long)p * ka + i] >= 0, hb = j < kb && bk[(long long)p * kb + j] >= 0;
        const long long out = (long long)p * k + o;
        if (!ha && !hb) { os[out] = -INFINITY; ok[out] = -1; osrc[out] = -1; continue; }
        bool take_a = ha;
        if (ha && hb) {
            const float sa = as[(long long)p * ka + i], sb = bs[(long long)p * kb + j];
            take_a = !better(sb, bk[(long long)p * kb + j], sa, ak[(long long)p * ka + i]);
        }
        if (take_a) { os[out] = as[(long long)p * ka + i]; ok[out] = ak[(long long)p * ka + i]; osrc[out] = p * ka + i; ++i; }
        else { os[out] = bs[(long long)p * kb + j]; ok[out] = bk[(long long)p * kb + j]; osrc[out] = q * ka + p * kb + j; ++j; }
    }
}

// q <= 8: 128 rows x 8 probes (the n8 minimum of the MMA); above: 128 x 32 (more reuse per staged element)
inline bool small_cfg(int q) { return q <= Small::PT; }

template <class C>
int blocks_per_sm(int k) {
    int nb = 0;
    const size_t sm = C::smem(k, 4);
    qk::raise_smem_limit((const void*)k_knn_scan<float, true, C>, (size_t)sm);
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k_knn_scan<float, true, C>, KNN_NT, sm) != cudaSuccess || nb < 1) nb = 1;
    return nb;
}

// row slices of the grid: enough CTAs for every SM, never more than there are row tiles
int row_ctas_for(int64_t n, int q, int k) {
    const bool small = small_cfg(q);
    const int PT = small ? Small::PT : Large::PT;
    const int per_sm = small ? blocks_per_sm<Small>(k) : blocks_per_sm<Large>(k);
    const long long ptiles = (q + PT - 1) / PT, rtiles = (n + RT - 1) / RT;
    long long want = ((long long)sm_count() * per_sm + ptiles - 1) / ptiles;
    if (want > rtiles) want = rtiles;
    return (int)(want < 1 ? 1 : want);
}

template <class T, bool VEC, class C>
int launch_cfg(const KnnArgs& A, cudaStream_t st) {
    const size_t sm = C::smem(A.k, sizeof(T));
    QK_CUDA(qk::raise_smem_limit((const void*)k_knn_scan<T, VEC, C>, (size_t)sm));
    k_knn_scan<T, VEC, C><<<dim3((A.q + C::PT - 1) / C::PT, A.row_ctas), KNN_NT, sm, st>>>(A);
    QK_LAUNCH_CHECK("k_knn_scan");
    return QK_OK;
}

template <class T>
int launch_scan(const KnnArgs& A, cudaStream_t st) {
    // 16-byte staging needs a 16-byte aligned column whose rows are whole 16-byte units
    const bool vec = ((uintptr_t)A.x & 15) == 0 && (A.d * (int)sizeof(T)) % 16 == 0;
    if (small_cfg(A.q)) return vec ? launch_cfg<T, true, Small>(A, st) : launch_cfg<T, false, Small>(A, st);
    return vec ? launch_cfg<T, true, Large>(A, st) : launch_cfg<T, false, Large>(A, st);
}

// the workspace: every row slice's k best scores per probe, then their rows, then 256 spare bytes
struct KnnWs {
    int row_ctas; float* score; int32_t* row; size_t bytes;
    KnnWs(int64_t n, int q, int k, void* base) : row_ctas(n > 0 ? row_ctas_for(n, q, k) : 0) {
        Carve c(base);
        score = c.take<float>((size_t)row_ctas * q * k);
        row = c.take<int32_t>((size_t)row_ctas * q * k);
        c.take<char>(256);                              // spare
        bytes = c.bytes;
    }
};

}  // namespace
}  // namespace qk

using namespace qk;

extern "C" size_t qk_knn_workspace_bytes(int64_t n, int32_t d, int32_t q, int32_t k) {
    if (n < 0 || d < 1 || q < 1 || k < 1 || k > QK_KNN_MAX_K) return 0;
    return KnnWs(n, q, k, nullptr).bytes;
}

extern "C" int qk_knn_topk(const qk_column* x, const float* probes, int32_t q, int32_t k, float* out_score, int64_t* out_row,
                           void* workspace, size_t ws_bytes, void* stream) {
    const char* who = "qk_knn_topk";
    if (int rc = check_rows_col(x, who)) return rc;
    if (x->dtype != QK_F32 && x->dtype != QK_F16) QK_FAIL(QK_ERR_INVALID, "%s: vectors must be f32 or f16 (dtype %d)", who, x->dtype);
    const int d = row_lanes(x);
    if (d < 1 || d > QK_KNN_MAX_DIM) QK_FAIL(QK_ERR_INVALID, "%s: dimension %d outside [1, %d]", who, d, QK_KNN_MAX_DIM);
    if (q < 1) QK_FAIL(QK_ERR_INVALID, "%s: q must be >= 1", who);
    if (k < 1 || k > QK_KNN_MAX_K) QK_FAIL(QK_ERR_INVALID, "%s: k must be in [1, %d]", who, QK_KNN_MAX_K);
    if (!probes || !out_score || !out_row) QK_FAIL(QK_ERR_INVALID, "%s: null probes / outputs", who);
    const KnnWs w(x->length, q, k, workspace);
    if (!workspace || ws_bytes < w.bytes) QK_FAIL(QK_ERR_CAPACITY, "%s: workspace of %zu bytes, %zu needed", who, ws_bytes, w.bytes);
    cudaStream_t st = (cudaStream_t)stream;
    KnnArgs A;
    A.x = x->data; A.probes = probes; A.n = x->length; A.d = d; A.q = q; A.k = k;
    A.ws_score = w.score;
    A.ws_row = w.row;
    A.row_ctas = w.row_ctas;
    if (A.row_ctas > 0) {
        if (int rc = x->dtype == QK_F32 ? launch_scan<float>(A, st) : launch_scan<unsigned short>(A, st)) return rc;
    }
    const size_t fold_smem = (size_t)(KNN_NT / 32) * k * 8;
    k_knn_fold<<<(q + KNN_NT / 32 - 1) / (KNN_NT / 32), KNN_NT, fold_smem, st>>>(A.ws_score, A.ws_row, A.row_ctas, q, k, out_score, out_row);
    QK_LAUNCH_CHECK("k_knn_fold");
    return QK_OK;
}

extern "C" int qk_knn_merge(int32_t q, const float* a_score, const int64_t* a_key, int32_t ka, const float* b_score,
                            const int64_t* b_key, int32_t kb, int32_t k, float* out_score, int64_t* out_key, int32_t* out_src,
                            void* stream) {
    const char* who = "qk_knn_merge";
    if (q < 0 || ka < 0 || kb < 0 || k < 1) QK_FAIL(QK_ERR_INVALID, "%s: bad sizes", who);
    if ((long long)q * (ka + kb) > 0x7fffffffLL) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: more than 2^31 - 1 candidates", who);
    if (q == 0) return QK_OK;
    if ((ka > 0 && (!a_score || !a_key)) || (kb > 0 && (!b_score || !b_key)) || !out_score || !out_key || !out_src)
        QK_FAIL(QK_ERR_INVALID, "%s: null arguments", who);
    k_knn_merge<<<(q + 127) / 128, 128, 0, (cudaStream_t)stream>>>(q, a_score, a_key, ka, b_score, b_key, kb, k, out_score, out_key, out_src);
    QK_LAUNCH_CHECK("k_knn_merge");
    return QK_OK;
}
