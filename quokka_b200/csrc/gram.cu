// gram.cu -- Gram matrix G += (X - c)^T (X - c) and column sums s += sum_rows (X - c) on the FP64 tensor cores
// (DataStream.gramian / covariance, pyquokka/datastream.py:1033-1147, where numpy's np.dot does it on the host).
//
// X is nrows x k, one Arrow buffer per column, contiguous along the rows.  The contraction runs over the rows, so both
// MMA operands come straight from the column buffers: A = X^T (row-major, rows of A = columns of X) and B = X (col-major),
// each a slab of rows of a block of T columns.  Only output tiles I <= J are computed; the fold mirrors them.
//
//   k_gram_tiles  grid (upper-triangle tile) x (row range).  A CTA streams its row range in slabs of R rows: cp.async
//                 copies the raw elements (4 or 8 bytes, any element-aligned start, so column views that start at an odd
//                 offset need no special path) into a two-stage ring; the threads widen them to fp64 and subtract the shift
//                 into a padded column-major slab; warps run mma.sync f64 (DMMA) over it.  Each CTA writes its T x T
//                 partial tile to the workspace.  A diagonal tile stages one block and uses it for both operands.
//   k_gram_fold   sums the partials of every tile over the row ranges in a fixed order and adds them into G (and its
//                 mirror) -- bit-identical results for the same inputs on the same device, as qk_scan_filter_agg_dense.
//
// Column sums ride along as a virtual column of ones at index k: G_ext[i][k] = sum_rows (X - c)_i.  They cost one extra
// column of the contraction instead of a second pass over X.
#include "common.cuh"
#include "tma.cuh"
#include <vector>

namespace qk {
namespace {

struct GramCol { const void* data; int32_t dtype; int32_t pad; };

constexpr int GROUP = 8;       // tiles are rasterised in GROUP x GROUP blocks of column blocks: CTAs resident together
                               // share column blocks in L2

__device__ __forceinline__ void cp_async(unsigned dst, const void* src, int bytes, int src_bytes) {
    if (bytes == 8) asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
    else asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait1() { asm volatile("cp.async.wait_group 1;" ::: "memory"); }

__device__ __forceinline__ void dmma_m8n8k4(double (&c)[2], double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                 : "+d"(c[0]), "+d"(c[1]) : "d"(a), "d"(b));
}
__device__ __forceinline__ void dmma_m16n8k16(double (&c)[4], const double (&a)[8], const double (&b)[4]) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, "
                 "{%12,%13,%14,%15}, {%0,%1,%2,%3};"
                 : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
                 : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]),
                   "d"(b[0]), "d"(b[1]), "d"(b[2]), "d"(b[3]));
}

// WM x WN warps over the T x T output tile, WK warps along the rows (each its own SLAB rows of the CTA's slab), a warp
// tile of (8 FM) x (8 FN).  MMA = 1: m8n8k4, MMA = 2: m16n8k16 (FM even).
template <int WM_, int WN_, int WK_, int FM_, int FN_, int SLAB_ = 32>
struct Cfg {
    static constexpr int WM = WM_, WN = WN_, WK = WK_, FM = FM_, FN = FN_, SLAB = SLAB_;
    static constexpr int NT = 32 * WM * WN * WK;
    static constexpr int T = 8 * WM * FM;
    static_assert(T == 8 * WN * FN, "square tiles");
    static constexpr int R = WK * SLAB;                           // rows per CTA slab
    static constexpr int RS = R + 4;                              // padded column stride in doubles: RS % 16 == 4, so the
                                                                  // 8 columns x 4 rows of a fragment hit distinct banks
    static constexpr size_t RAW = (size_t)T * R * 8;              // one operand's raw slab (8-byte slots)
    static constexpr size_t F64 = (size_t)T * RS * 8;             // one operand's fp64 slab
    // raw ring (2 stages x nops operands) + fp64 operands; nops = 1 when every tile is diagonal (k + 1 <= T)
    static constexpr size_t smem(int nops) { return 2 * nops * RAW + nops * F64; }
    static_assert(WK == 1 || (size_t)WK * T * T * 8 <= 2 * RAW, "the cross-warp reduction reuses the raw ring");
};
using CfgT8 = Cfg<1, 1, 8, 1, 1>;       // k <= 8: eight warps along the rows, 3 CTAs per SM (narrow tables are HBM-bound;
                                        // one CTA with 128-row slabs per warp measured slower)
using CfgT32 = Cfg<1, 1, 4, 4, 4>;      // k <= 32
using CfgT64 = Cfg<2, 2, 2, 4, 4>;      // k <= 64
using CfgT128 = Cfg<2, 4, 1, 8, 4>;     // wide: 128 x 128 tiles, 8 warps of 64 x 32

struct TileArgs {
    const GramCol* cols;     // workspace copy of the column table [k]
    const double* shift;     // device [k] or NULL
    const int2* tiles;       // (I, J) column blocks of each tile, I <= J
    double* part;            // [nsplit][ntiles][T][T]
    int32_t k, kext, ntiles, nops;        // nops: operands the smem ring holds (1: every tile is diagonal)
    int64_t nrows, rows_per_split;
};

template <class C>
__device__ __forceinline__ void stage_raw(const GramCol* desc, int colbase, int k, int64_t row0, int64_t row_hi, unsigned raw) {
#pragma unroll 4
    for (int e = threadIdx.x; e < C::T * C::R; e += C::NT) {
        const int c = e / C::R, r = e % C::R;
        const int gc = colbase + c;
        if (gc >= k) continue;
        const GramCol d = desc[c];
        const int sz = (d.dtype == QK_F64 || d.dtype == QK_I64) ? 8 : 4;
        const int64_t row = row0 + r;
        const bool ok = row < row_hi;
        cp_async(raw + (unsigned)(e * 8), ok ? (const char*)d.data + row * sz : d.data, sz, ok ? sz : 0);
    }
}

template <class C>
__device__ __forceinline__ void widen(const GramCol* desc, const double* sh, int colbase, int k, int kext, int64_t row0,
                                      int64_t row_hi, const unsigned char* raw, double* f) {
#pragma unroll 4
    for (int e = threadIdx.x; e < C::T * C::R; e += C::NT) {
        const int c = e / C::R, r = e % C::R;
        const int gc = colbase + c;
        const bool ok = row0 + r < row_hi;
        double v = 0.0;
        if (gc < k) {
            const unsigned char* p = raw + (size_t)e * 8;
            switch (desc[c].dtype) {
                case QK_F64: v = *(const double*)p; break;
                case QK_F32: v = (double)*(const float*)p; break;
                case QK_I64: v = (double)*(const long long*)p; break;
                default: v = (double)*(const int*)p; break;
            }
            v = ok ? v - sh[c] : 0.0;
        } else if (gc < kext) {
            v = ok ? 1.0 : 0.0;                      // the virtual column of ones (column sums)
        }
        f[c * C::RS + r] = v;
    }
}

template <class C, int MMA>
__global__ void __launch_bounds__(C::NT, 1) k_gram_tiles(const __grid_constant__ TileArgs A) {
    extern __shared__ __align__(16) unsigned char smem[];
    __shared__ GramCol desc[2][C::T];
    __shared__ double sh[2][C::T];
    const int tile = blockIdx.x, split = blockIdx.y;
    const int2 IJ = A.tiles[tile];
    const bool diag = IJ.x == IJ.y;
    for (int i = threadIdx.x; i < 2 * C::T; i += C::NT) {
        const int o = i / C::T, c = i % C::T, gc = (o ? IJ.y : IJ.x) * C::T + c;
        desc[o][c] = gc < A.k ? A.cols[gc] : GramCol{nullptr, QK_F64, 0};
        sh[o][c] = (gc < A.k && A.shift) ? A.shift[gc] : 0.0;
    }
    __syncthreads();

    unsigned char* raw = smem;                                            // [stage][operand][T * R] 8-byte slots
    double* fA = (double*)(smem + 2 * A.nops * C::RAW);
    double* fB = diag ? fA : fA + C::T * C::RS;
    const unsigned raw_s = smem_u32(raw);

    const int64_t row_lo = (int64_t)split * A.rows_per_split;
    const int64_t row_hi = min(A.nrows, row_lo + A.rows_per_split);
    const int nslabs = row_hi > row_lo ? (int)((row_hi - row_lo + C::R - 1) / C::R) : 0;
    const int nops = diag ? 1 : 2;

    const int warp = threadIdx.x / 32, lane = threadIdx.x % 32, g = lane >> 2, t = lane & 3;
    const int wk = warp % C::WK, wn = (warp / C::WK) % C::WN, wm = warp / (C::WK * C::WN);
    constexpr int FM2 = MMA == 1 ? C::FM : C::FM / 2;
    constexpr int NACC = MMA == 1 ? 2 : 4;
    double acc[FM2][C::FN][NACC];
#pragma unroll
    for (int i = 0; i < FM2; ++i)
#pragma unroll
        for (int j = 0; j < C::FN; ++j)
#pragma unroll
            for (int q = 0; q < NACC; ++q) acc[i][j][q] = 0.0;

    if (nslabs > 0) {
        for (int o = 0; o < nops; ++o)
            stage_raw<C>(desc[o], (o ? IJ.y : IJ.x) * C::T, A.k, row_lo, row_hi, raw_s + (unsigned)(o * C::RAW));
        cp_async_commit();
    }
    for (int s = 0; s < nslabs; ++s) {
        const int64_t row0 = row_lo + (int64_t)s * C::R;
        if (s + 1 < nslabs)
            for (int o = 0; o < nops; ++o)
                stage_raw<C>(desc[o], (o ? IJ.y : IJ.x) * C::T, A.k, row0 + C::R, row_hi, raw_s + (unsigned)((((s + 1) & 1) * A.nops + o) * C::RAW));
        cp_async_commit();
        cp_async_wait1();
        __syncthreads();                                                  // slab s landed; every warp is done with slab s-1
        for (int o = 0; o < nops; ++o)
            widen<C>(desc[o], sh[o], (o ? IJ.y : IJ.x) * C::T, A.k, A.kext, row0, row_hi, raw + ((s & 1) * A.nops + o) * C::RAW, o ? fB : fA);
        __syncthreads();
        const double* a0 = fA + (wm * C::FM * 8 + g) * C::RS + wk * C::SLAB + t;
        const double* b0 = fB + (wn * C::FN * 8 + g) * C::RS + wk * C::SLAB + t;
        if constexpr (MMA == 1) {
#pragma unroll
            for (int kk = 0; kk < C::SLAB; kk += 4) {
                double a[C::FM], b[C::FN];
#pragma unroll
                for (int i = 0; i < C::FM; ++i) a[i] = a0[i * 8 * C::RS + kk];
#pragma unroll
                for (int j = 0; j < C::FN; ++j) b[j] = b0[j * 8 * C::RS + kk];
#pragma unroll
                for (int i = 0; i < C::FM; ++i)
#pragma unroll
                    for (int j = 0; j < C::FN; ++j) dmma_m8n8k4(acc[i][j], a[i], b[j]);
            }
        } else {
#pragma unroll
            for (int kk = 0; kk < C::SLAB; kk += 16) {
                double b[C::FN][4];
#pragma unroll
                for (int j = 0; j < C::FN; ++j)
#pragma unroll
                    for (int q = 0; q < 4; ++q) b[j][q] = b0[j * 8 * C::RS + kk + 4 * q];
#pragma unroll
                for (int i = 0; i < FM2; ++i) {
                    double a[8];
#pragma unroll
                    for (int q = 0; q < 8; ++q) a[q] = a0[(i * 16 + 8 * (q & 1)) * C::RS + kk + 4 * (q >> 1)];
#pragma unroll
                    for (int j = 0; j < C::FN; ++j) dmma_m16n8k16(acc[i][j], a, b[j]);
                }
            }
        }
    }

    // partial tile out: C fragment element q of sub-tile (i, j) sits at row g (+8 for q >= 2 in m16n8k16), column 2t + (q & 1)
    double* out = A.part + ((size_t)split * A.ntiles + tile) * C::T * C::T;
    double* red = (double*)smem;
    if (C::WK > 1) __syncthreads();                                       // the raw ring becomes the reduction buffer
#pragma unroll
    for (int i = 0; i < FM2; ++i)
#pragma unroll
        for (int j = 0; j < C::FN; ++j)
#pragma unroll
            for (int q = 0; q < NACC; ++q) {
                const int row = wm * C::FM * 8 + (MMA == 1 ? i * 8 : i * 16 + 8 * (q >> 1)) + g;
                const int col = wn * C::FN * 8 + j * 8 + 2 * t + (q & 1);
                if (C::WK == 1) out[row * C::T + col] = acc[i][j][q];
                else red[(wk * C::T + row) * C::T + col] = acc[i][j][q];
            }
    if (C::WK > 1) {
        __syncthreads();
        for (int e = threadIdx.x; e < C::T * C::T; e += C::NT) {
            double v = red[e];
#pragma unroll
            for (int w = 1; w < C::WK; ++w) v += red[w * C::T * C::T + e];          // fixed order over the row warps
            out[e] = v;
        }
    }
}

// one thread per element of every upper-triangle tile: G[gi][gj] (and G[gj][gi]) += sum over the row ranges, in order
__global__ void __launch_bounds__(256) k_gram_fold(const double* part, const int2* tiles, int ntiles, int T, int nsplit, int k,
                                                   double* G, double* sums) {
    const int64_t tt = (int64_t)T * T;
    const int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (idx >= (int64_t)ntiles * tt) return;
    const int tile = (int)(idx / tt), e = (int)(idx % tt);
    const int2 IJ = tiles[tile];
    const int gi = IJ.x * T + e / T, gj = IJ.y * T + e % T;
    if (gi > gj || gi >= k || gj > k) return;                            // lower half of a diagonal tile, padding, n
    if (gj == k && !sums) return;
    double v = 0.0;
    for (int s = 0; s < nsplit; ++s) v += part[((int64_t)s * ntiles + tile) * tt + e];
    if (gj == k) {
        sums[gi] += v;
        return;
    }
    G[(int64_t)gi * k + gj] += v;
    if (gi != gj) G[(int64_t)gj * k + gi] += v;
}

struct Plan {
    int cfg;               // 0: T8, 1: T32, 2: T64, 3: T128
    int T, R, nb, ntiles, nsplit;
    int64_t rows_per_split;
};

Plan make_plan(int64_t nrows, int32_t kext) {
    Plan p{};
    if (kext <= 8) { p.cfg = 0; p.T = CfgT8::T; p.R = CfgT8::R; }
    else if (kext <= 32) { p.cfg = 1; p.T = CfgT32::T; p.R = CfgT32::R; }
    else if (kext <= 64) { p.cfg = 2; p.T = CfgT64::T; p.R = CfgT64::R; }
    else { p.cfg = 3; p.T = CfgT128::T; p.R = CfgT128::R; }
    p.nb = (kext + p.T - 1) / p.T;
    p.ntiles = p.nb * (p.nb + 1) / 2;
    const int per_sm = p.cfg == 0 ? 3 : 1;                                 // resident CTAs per SM (T8: 49 KB smem, 79 registers)
    const int64_t want = 4LL * per_sm * sm_count();                       // >= 4 waves: the last one is a small tail
    const int64_t slabs = (nrows + p.R - 1) / p.R;
    int64_t ns = p.ntiles >= want ? 1 : (want + p.ntiles - 1) / p.ntiles;
    if (ns > slabs) ns = slabs > 0 ? slabs : 1;
    const int64_t per = (slabs + ns - 1) / ns;
    p.rows_per_split = per * p.R;
    p.nsplit = (int)ns;
    return p;
}

size_t plan_bytes(const Plan& p, int32_t k) {
    return align_up((size_t)k * sizeof(GramCol), 256) + align_up((size_t)p.ntiles * sizeof(int2), 256) +
           (size_t)p.nsplit * p.ntiles * p.T * p.T * sizeof(double);
}

template <class C, int MMA>
int launch_tiles(const TileArgs& a, int ntiles, int nsplit, cudaStream_t st) {
    auto kern = k_gram_tiles<C, MMA>;
    const size_t smem = C::smem(a.nops);
    QK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<dim3((unsigned)ntiles, (unsigned)nsplit), C::NT, smem, st>>>(a);
    QK_LAUNCH_CHECK("k_gram_tiles");
    return QK_OK;
}

thread_local char g_gram_variant[32] = "";

}  // namespace
}  // namespace qk

using namespace qk;

extern "C" size_t qk_gram_workspace_bytes(int64_t nrows, int32_t k) {
    if (nrows < 0 || k < 1) return 0;
    const size_t a = plan_bytes(make_plan(nrows, k), k), b = plan_bytes(make_plan(nrows, k + 1), k);
    return a > b ? a : b;                                                  // with or without the column of ones
}

extern "C" int qk_gram(const qk_column* cols, int32_t k, int64_t nrows, const double* shift, double* gram, double* sums,
                       int32_t variant, void* workspace, size_t ws_bytes, void* stream) {
    const char* who = "qk_gram";
    if (k < 1) QK_FAIL(QK_ERR_INVALID, "%s: k must be >= 1", who);
    if (!cols) QK_FAIL(QK_ERR_INVALID, "%s: null column table", who);
    if (nrows < 0) QK_FAIL(QK_ERR_INVALID, "%s: negative nrows", who);
    for (int32_t i = 0; i < k; ++i) {
        if (int rc = check_col(&cols[i], who)) return rc;
        const int dt = cols[i].dtype;
        if (dt != QK_F64 && dt != QK_F32 && dt != QK_I32 && dt != QK_I64)
            QK_FAIL(QK_ERR_INVALID, "%s: column %d has unsupported dtype %d (f64, f32, i32 or i64)", who, i, dt);
        if (cols[i].length != nrows) QK_FAIL(QK_ERR_INVALID, "%s: column %d has %lld rows, expected %lld", who, i,
                                             (long long)cols[i].length, (long long)nrows);
    }
    if (variant < 0 || variant > 2) QK_FAIL(QK_ERR_INVALID, "%s: variant must be 0, 1 or 2", who);
    if (!gram) QK_FAIL(QK_ERR_INVALID, "%s: null gram", who);
    if (nrows == 0) return QK_OK;
    const int32_t kext = k + (sums ? 1 : 0);
    const Plan p = make_plan(nrows, kext);
    if (!workspace || ws_bytes < plan_bytes(p, k)) QK_FAIL(QK_ERR_CAPACITY, "%s: workspace too small (%zu < %zu)", who, ws_bytes,
                                                           plan_bytes(p, k));
    // column table and tile order travel in the workspace, so any k fits
    const size_t off_tiles = align_up((size_t)k * sizeof(GramCol), 256);
    const size_t off_part = off_tiles + align_up((size_t)p.ntiles * sizeof(int2), 256);
    std::vector<unsigned char> host(off_part, 0);
    GramCol* hc = (GramCol*)host.data();
    for (int32_t i = 0; i < k; ++i) hc[i] = GramCol{cols[i].data, cols[i].dtype, 0};
    int2* ht = (int2*)(host.data() + off_tiles);
    int n = 0;
    for (int bi = 0; bi < p.nb; bi += GROUP)
        for (int bj = bi; bj < p.nb; bj += GROUP)
            for (int I = bi; I < bi + GROUP && I < p.nb; ++I)
                for (int J = (I > bj ? I : bj); J < bj + GROUP && J < p.nb; ++J) ht[n++] = make_int2(I, J);
    cudaStream_t st = (cudaStream_t)stream;
    QK_CUDA(cudaMemcpyAsync(workspace, host.data(), off_part, cudaMemcpyHostToDevice, st));
    TileArgs a;
    a.cols = (const GramCol*)workspace;
    a.shift = shift;
    a.tiles = (const int2*)((char*)workspace + off_tiles);
    a.part = (double*)((char*)workspace + off_part);
    a.k = k; a.kext = kext; a.ntiles = p.ntiles; a.nops = p.nb > 1 ? 2 : 1;
    a.nrows = nrows; a.rows_per_split = p.rows_per_split;
    const int mma = variant == 0 ? 2 : variant;                            // m16n8k16 measured faster (DESIGN.md section 4)
    int rc;
    switch (p.cfg) {
        case 0: rc = launch_tiles<CfgT8, 1>(a, p.ntiles, p.nsplit, st); break;        // m16 needs FM even: T8 stays m8n8k4
        case 1: rc = mma == 2 ? launch_tiles<CfgT32, 2>(a, p.ntiles, p.nsplit, st) : launch_tiles<CfgT32, 1>(a, p.ntiles, p.nsplit, st); break;
        case 2: rc = mma == 2 ? launch_tiles<CfgT64, 2>(a, p.ntiles, p.nsplit, st) : launch_tiles<CfgT64, 1>(a, p.ntiles, p.nsplit, st); break;
        default: rc = mma == 2 ? launch_tiles<CfgT128, 2>(a, p.ntiles, p.nsplit, st) : launch_tiles<CfgT128, 1>(a, p.ntiles, p.nsplit, st); break;
    }
    if (rc) return rc;
    snprintf(g_gram_variant, sizeof g_gram_variant, "T%d%s s%d", p.T, (mma == 2 && p.cfg) ? "m16n8k16" : "m8n8k4", p.nsplit);
    const int64_t total = (int64_t)p.ntiles * p.T * p.T;
    k_gram_fold<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(a.part, a.tiles, p.ntiles, p.T, p.nsplit, k, gram, sums);
    QK_LAUNCH_CHECK("k_gram_fold");
    return QK_OK;
}

extern "C" const char* qk_gram_last_plan(void) { return g_gram_variant; }
