// scan.cu -- K1 scan->filter->project and K1+K2 scan->filter->project->dense aggregate.
//
// Three code paths, all HBM-bound by design (no tensor cores: there is no dense contraction):
//   variant 1  generic: a postfix interpreter per row (any predicate / expression the host compiler
//              emits); stack in local memory, columns read straight from global memory.
//   variant 2  fused template: the plan shape (typed column slots, affine-product aggregates) is a
//              C++ type, so every operand lives in a statically named register; 4 rows per thread,
//              128-bit global loads (32-bit for the 1-byte code columns).
//   variant 3  the same fused plan with the column tiles staged into shared memory by the TMA engine
//              (cp.async.bulk + mbarrier complete_tx), 3-stage ring, one elected producer thread.
// The dense aggregate keeps LANE-PRIVATE partial states in shared memory (acc[slot][thread]), so the
// inner loop has no atomics and no bank conflicts; each CTA then reduces its copies with warp shuffles
// and writes one partial per slot; a last tiny kernel folds the per-CTA partials in a FIXED order, which
// makes the fp64 result deterministic run to run.
//
// Algorithmic bytes (DESIGN.md): Q1 = 38 B per lineitem row read (date32 4 + 2 x 1-B codes + 4 x fp64).
#include <string>
#include <vector>
#include "common.cuh"
#include "tma.cuh"

namespace qk {
namespace {

// ---------------------------------------------------------------- compact programs (kernel params)
struct PNode {
    int16_t op;
    int16_t a0;
    int32_t a1;
    union { double imm; int64_t imm_i; };
    int64_t imm2;                      // RANGE_COL_IMM: the upper bound
};
struct ColRef { const void* p; int32_t dt; int32_t pad; };

constexpr int MAX_PROGS = 1 + QK_MAX_PROJ;          // pred + projections / aggregates
constexpr int MAX_NODES = 112;

struct Programs {
    ColRef cols[QK_MAX_COLS];
    PNode nodes[MAX_NODES];
    int16_t off[MAX_PROGS + 1];                       // program k = nodes[off[k], off[k+1])
    int32_t nprog;                                    // program 0 is the predicate (may be empty)
};

int pack_programs(Programs& P, const qk_column* cols, int ncols, int64_t nrows, const qk_expr* pred,
                  const qk_expr* exprs, int nexpr, const char* who) {
    if (ncols < 0 || ncols > QK_MAX_COLS) QK_FAIL(QK_ERR_INVALID, "%s: ncols %d out of range", who, ncols);
    if (nexpr < 0 || nexpr > QK_MAX_PROJ) QK_FAIL(QK_ERR_INVALID, "%s: too many expressions (%d)", who, nexpr);
    if (nrows < 0 || nrows > 0x7fffffffLL) QK_FAIL(QK_ERR_INVALID, "%s: nrows %lld out of range", who, (long long)nrows);
    for (int c = 0; c < ncols; ++c) {
        if (int rc = check_col(&cols[c], who)) return rc;
        if (cols[c].length != nrows) QK_FAIL(QK_ERR_INVALID, "%s: column %d has %lld rows, expected %lld", who, c, (long long)cols[c].length, (long long)nrows);
        P.cols[c] = ColRef{cols[c].data, cols[c].dtype, 0};
    }
    for (int c = ncols; c < QK_MAX_COLS; ++c) P.cols[c] = ColRef{nullptr, 0, 0};
    int n = 0;
    P.nprog = 1 + nexpr;
    for (int k = 0; k < 1 + nexpr; ++k) {
        const qk_expr* e = k == 0 ? pred : &exprs[k - 1];
        P.off[k] = (int16_t)n;
        int cnt = e ? e->n_nodes : 0;
        if (cnt < 0 || cnt > QK_MAX_EXPR_NODES) QK_FAIL(QK_ERR_INVALID, "%s: expression %d has %d nodes", who, k, cnt);
        if (k > 0 && cnt == 0) QK_FAIL(QK_ERR_INVALID, "%s: empty expression %d", who, k - 1);
        if (n + cnt > MAX_NODES) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: programs exceed %d nodes in total", who, MAX_NODES);
        int depth = 0;
        for (int i = 0; i < cnt; ++i) {
            const qk_expr_node& s = e->nodes[i];
            PNode d;
            d.op = (int16_t)s.op; d.a0 = (int16_t)s.a0; d.a1 = s.a1; d.imm = s.imm; d.imm2 = 0;
            switch (s.op) {
                case QK_OP_COL:
                    if (s.a0 < 0 || s.a0 >= ncols) QK_FAIL(QK_ERR_INVALID, "%s: column slot %d out of range", who, s.a0);
                    depth++; break;
                case QK_OP_CONST: depth++; break;
                case QK_OP_ADD: case QK_OP_SUB: case QK_OP_MUL: case QK_OP_DIV: case QK_OP_LT: case QK_OP_LE:
                case QK_OP_GT: case QK_OP_GE: case QK_OP_EQ: case QK_OP_NE: case QK_OP_AND: case QK_OP_OR:
                    if (depth < 2) QK_FAIL(QK_ERR_INVALID, "%s: stack underflow in expression %d", who, k);
                    depth--; break;
                case QK_OP_NEG: case QK_OP_NOT: case QK_OP_RINT:
                    if (depth < 1) QK_FAIL(QK_ERR_INVALID, "%s: stack underflow in expression %d", who, k);
                    break;
                case QK_OP_EXTRACT:
                    if (depth < 1) QK_FAIL(QK_ERR_INVALID, "%s: stack underflow in expression %d", who, k);
                    if (s.a1 < 0 || s.a1 > 2) QK_FAIL(QK_ERR_INVALID, "%s: EXTRACT part must be 0 (year), 1 (month) or 2 (day)", who);
                    break;
                case QK_OP_SELECT:
                    if (depth < 3) QK_FAIL(QK_ERR_INVALID, "%s: stack underflow in expression %d", who, k);
                    depth -= 2; break;
                case QK_OP_IN_SET:
                    if (s.a0 < 0 || s.a0 >= ncols || !dtype_is_int(cols[s.a0].dtype)) QK_FAIL(QK_ERR_INVALID, "%s: IN_SET needs an integer column", who);
                    if (s.a1 < 0) QK_FAIL(QK_ERR_INVALID, "%s: IN_SET with a negative bit count", who);
                    if (s.a1 > 64 && s.imm_i == 0) QK_FAIL(QK_ERR_INVALID, "%s: IN_SET over %d bits needs a device bitmap", who, s.a1);
                    d.imm_i = s.imm_i; depth++; break;
                case QK_OP_CMP_COL_IMM:
                    if (s.a0 < 0 || s.a0 >= ncols || !dtype_is_int(cols[s.a0].dtype)) QK_FAIL(QK_ERR_INVALID, "%s: CMP_COL_IMM needs an integer column", who);
                    if (s.a1 < 0 || s.a1 > QK_CMP_NE) QK_FAIL(QK_ERR_INVALID, "%s: bad compare code", who);
                    d.imm_i = s.imm_i; depth++; break;
                case QK_OP_RANGE_COL_IMM:
                    if (s.a0 < 0 || s.a0 >= ncols || !dtype_is_int(cols[s.a0].dtype)) QK_FAIL(QK_ERR_INVALID, "%s: RANGE_COL_IMM needs an integer column", who);
                    if (!(s.imm >= -9007199254740992.0 && s.imm <= 9007199254740992.0)) QK_FAIL(QK_ERR_INVALID, "%s: RANGE_COL_IMM upper bound out of range", who);
                    d.imm_i = s.imm_i; d.imm2 = (int64_t)s.imm; d.a1 = s.a1 != 0; depth++; break;
                case QK_OP_CMP_COL_COL: {
                    int b = s.a1 >> 8, cmp = s.a1 & 0xff;
                    if (s.a0 < 0 || s.a0 >= ncols || b < 0 || b >= ncols || !dtype_is_int(cols[s.a0].dtype) || !dtype_is_int(cols[b].dtype))
                        QK_FAIL(QK_ERR_INVALID, "%s: CMP_COL_COL needs two integer columns", who);
                    if (cmp > QK_CMP_NE) QK_FAIL(QK_ERR_INVALID, "%s: bad compare code", who);
                    depth++; } break;
                default: QK_FAIL(QK_ERR_INVALID, "%s: unknown op %d", who, s.op);
            }
            if (depth > QK_MAX_STACK) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: expression needs more than %d stack slots", who, QK_MAX_STACK);
            P.nodes[n++] = d;
        }
        if (cnt > 0 && depth != 1) QK_FAIL(QK_ERR_INVALID, "%s: expression %d leaves %d values on the stack", who, k, depth);
    }
    P.off[1 + nexpr] = (int16_t)n;
    return 0;
}

// days since 1970-01-01 -> civil year / month / day (proleptic Gregorian; H. Hinnant's civil_from_days)
__device__ __forceinline__ long long civil_part(long long days, int part) {
    const long long z = days + 719468;
    const long long era = (z >= 0 ? z : z - 146096) / 146097;
    const long long doe = z - era * 146097;
    const long long yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;
    const long long doy = doe - (365 * yoe + yoe / 4 - yoe / 100);
    const long long mp = (5 * doy + 2) / 153;
    const long long d = doy - (153 * mp + 2) / 5 + 1;
    const long long m = mp < 10 ? mp + 3 : mp - 9;
    const long long y = yoe + era * 400 + (m <= 2 ? 1 : 0);
    return part == 0 ? y : part == 1 ? m : d;
}

// ---------------------------------------------------------------- the interpreter
__device__ __forceinline__ double eval_prog(const Programs& P, int k, int64_t row) {
    double st[QK_MAX_STACK];
    int sp = 0;
    const int end = P.off[k + 1];
    for (int pc = P.off[k]; pc < end; ++pc) {
        const PNode nd = P.nodes[pc];
        switch (nd.op) {
            case QK_OP_COL: st[sp++] = load_f64(P.cols[nd.a0].p, P.cols[nd.a0].dt, row); break;
            case QK_OP_CONST: st[sp++] = nd.imm; break;
            case QK_OP_ADD: sp--; st[sp - 1] = st[sp - 1] + st[sp]; break;
            case QK_OP_SUB: sp--; st[sp - 1] = st[sp - 1] - st[sp]; break;
            case QK_OP_MUL: sp--; st[sp - 1] = st[sp - 1] * st[sp]; break;
            case QK_OP_DIV: sp--; st[sp - 1] = st[sp - 1] / st[sp]; break;
            case QK_OP_NEG: st[sp - 1] = -st[sp - 1]; break;
            case QK_OP_LT: sp--; st[sp - 1] = st[sp - 1] < st[sp] ? 1.0 : 0.0; break;
            case QK_OP_LE: sp--; st[sp - 1] = st[sp - 1] <= st[sp] ? 1.0 : 0.0; break;
            case QK_OP_GT: sp--; st[sp - 1] = st[sp - 1] > st[sp] ? 1.0 : 0.0; break;
            case QK_OP_GE: sp--; st[sp - 1] = st[sp - 1] >= st[sp] ? 1.0 : 0.0; break;
            case QK_OP_EQ: sp--; st[sp - 1] = st[sp - 1] == st[sp] ? 1.0 : 0.0; break;
            case QK_OP_NE: sp--; st[sp - 1] = st[sp - 1] != st[sp] ? 1.0 : 0.0; break;
            case QK_OP_AND: sp--; st[sp - 1] = (st[sp - 1] != 0.0 && st[sp] != 0.0) ? 1.0 : 0.0; break;
            case QK_OP_OR: sp--; st[sp - 1] = (st[sp - 1] != 0.0 || st[sp] != 0.0) ? 1.0 : 0.0; break;
            case QK_OP_NOT: st[sp - 1] = st[sp - 1] == 0.0 ? 1.0 : 0.0; break;
            case QK_OP_RINT: st[sp - 1] = rint(st[sp - 1]); break;
            case QK_OP_EXTRACT: st[sp - 1] = (double)civil_part((long long)st[sp - 1], nd.a1); break;
            case QK_OP_SELECT: sp -= 2; st[sp - 1] = st[sp - 1] != 0.0 ? st[sp] : st[sp + 1]; break;
            case QK_OP_IN_SET: {
                const int64_t code = load_i64(P.cols[nd.a0].p, P.cols[nd.a0].dt, row);
                bool in = false;
                if (code >= 0 && code < (int64_t)nd.a1)
                    in = nd.a1 <= 64 ? ((unsigned long long)nd.imm_i >> code) & 1ull
                                     : (__ldg((const unsigned*)(uintptr_t)nd.imm_i + (code >> 5)) >> (code & 31)) & 1u;
                st[sp++] = in ? 1.0 : 0.0;
            } break;
            case QK_OP_CMP_COL_IMM:
                st[sp++] = cmp_i64(load_i64(P.cols[nd.a0].p, P.cols[nd.a0].dt, row), nd.a1, nd.imm_i) ? 1.0 : 0.0;
                break;
            case QK_OP_RANGE_COL_IMM: {
                const long long x = load_i64(P.cols[nd.a0].p, P.cols[nd.a0].dt, row);
                st[sp++] = (((x >= nd.imm_i) & (x <= nd.imm2)) != (nd.a1 != 0)) ? 1.0 : 0.0;
            } break;
            default: {  // QK_OP_CMP_COL_COL
                const int b = nd.a1 >> 8;
                st[sp++] = cmp_i64(load_i64(P.cols[nd.a0].p, P.cols[nd.a0].dt, row), nd.a1 & 0xff,
                                   load_i64(P.cols[b].p, P.cols[b].dt, row)) ? 1.0 : 0.0;
            } break;
        }
    }
    return st[0];
}
__device__ __forceinline__ bool eval_pred(const Programs& P, int64_t row) {
    return P.off[1] == P.off[0] ? true : eval_prog(P, 0, row) != 0.0;
}

// ---------------------------------------------------------------- projection output
struct ProjOut {
    void* out[QK_MAX_PROJ];
    int8_t pass_col[QK_MAX_PROJ];   // >= 0: verbatim copy of that column slot; -1: fp64 expression
};

__device__ __forceinline__ void write_proj(const Programs& P, const ProjOut& O, int nproj, int64_t row, int64_t pos) {
    for (int j = 0; j < nproj; ++j) {
        const int pc = O.pass_col[j];
        if (pc >= 0) {
            const ColRef c = P.cols[pc];
            switch (c.dt) {
                case QK_U8: ((uint8_t*)O.out[j])[pos] = ((const uint8_t*)c.p)[row]; break;
                case QK_I32: case QK_F32: ((uint32_t*)O.out[j])[pos] = ((const uint32_t*)c.p)[row]; break;
                default: ((uint64_t*)O.out[j])[pos] = ((const uint64_t*)c.p)[row]; break;
            }
        } else {
            ((double*)O.out[j])[pos] = eval_prog(P, 1 + j, row);
        }
    }
}

// unordered compaction: one atomic per warp, arrival order
__global__ void __launch_bounds__(256) k_filter_project_unordered(const __grid_constant__ Programs P,
                                                                  const __grid_constant__ ProjOut O, int nproj,
                                                                  int64_t nrows, unsigned long long* out_rows) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    const int64_t nround = (nrows + 31) / 32 * 32;
    for (int64_t row = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; row < nround; row += stride) {
        const bool pass = row < nrows && eval_pred(P, row);
        const unsigned m = __ballot_sync(0xffffffffu, pass);
        if (m == 0) continue;
        unsigned long long base = 0;
        if (lane_id() == 0) base = atomicAdd(out_rows, (unsigned long long)__popc(m));
        base = __shfl_sync(0xffffffffu, base, 0);
        if (pass) write_proj(P, O, nproj, row, (int64_t)base + __popc(m & lanemask_lt()));
    }
}

// stable compaction, pass 1: passing rows per CHUNK
constexpr int STABLE_CHUNK = 2048;
__global__ void __launch_bounds__(256) k_filter_count(const __grid_constant__ Programs P, int64_t nrows, int32_t* chunk_counts) {
    __shared__ int wsum[8];
    for (int64_t chunk = blockIdx.x; chunk * STABLE_CHUNK < nrows; chunk += gridDim.x) {
        int cnt = 0;
        const int64_t base = chunk * STABLE_CHUNK;
        for (int t = threadIdx.x; t < STABLE_CHUNK; t += 256) {
            const int64_t row = base + t;
            cnt += (row < nrows && eval_pred(P, row)) ? 1 : 0;
        }
        for (int o = 16; o; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
        if (lane_id() == 0) wsum[threadIdx.x >> 5] = cnt;
        __syncthreads();
        if (threadIdx.x == 0) {
            int s = 0;
            for (int w = 0; w < 8; ++w) s += wsum[w];
            chunk_counts[chunk] = s;
        }
        __syncthreads();
    }
}
// exclusive scan of chunk counts (single CTA, sequential over 1024-wide tiles), total -> out_rows
__global__ void __launch_bounds__(1024) k_scan_counts(const int32_t* counts, int64_t n, int64_t* offsets, int64_t* out_rows) {
    __shared__ int64_t wtot[32];
    __shared__ int64_t carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (int64_t base = 0; base < n; base += 1024) {
        const int64_t i = base + threadIdx.x;
        int64_t v = i < n ? counts[i] : 0, x = v;
        for (int o = 1; o < 32; o <<= 1) {
            int64_t y = __shfl_up_sync(0xffffffffu, x, o);
            if (lane_id() >= o) x += y;
        }
        if (lane_id() == 31) wtot[threadIdx.x >> 5] = x;
        __syncthreads();
        if (threadIdx.x < 32) {
            int64_t w = wtot[threadIdx.x], s = w;
            for (int o = 1; o < 32; o <<= 1) {
                int64_t y = __shfl_up_sync(0xffffffffu, s, o);
                if (lane_id() >= o) s += y;
            }
            wtot[threadIdx.x] = s - w;     // exclusive warp offsets
        }
        __syncthreads();
        const int64_t excl = carry + wtot[threadIdx.x >> 5] + x - v;
        if (i < n) offsets[i] = excl;
        __syncthreads();
        if (threadIdx.x == 1023) carry = excl + v;
        __syncthreads();
    }
    if (threadIdx.x == 0) *out_rows = carry;
}
// stable compaction, pass 2
__global__ void __launch_bounds__(256) k_filter_project_stable(const __grid_constant__ Programs P, const __grid_constant__ ProjOut O,
                                                               int nproj, int64_t nrows, const int64_t* chunk_offsets) {
    __shared__ int wcnt[8];
    for (int64_t chunk = blockIdx.x; chunk * STABLE_CHUNK < nrows; chunk += gridDim.x) {
        int64_t running = chunk_offsets[chunk];
        const int64_t base = chunk * STABLE_CHUNK;
        for (int t0 = 0; t0 < STABLE_CHUNK; t0 += 256) {
            const int64_t row = base + t0 + threadIdx.x;
            const bool pass = row < nrows && eval_pred(P, row);
            const unsigned m = __ballot_sync(0xffffffffu, pass);
            if (lane_id() == 0) wcnt[threadIdx.x >> 5] = __popc(m);
            __syncthreads();
            int before = 0, total = 0;
            for (int w = 0; w < 8; ++w) {
                const int c = wcnt[w];
                if (w < (int)(threadIdx.x >> 5)) before += c;
                total += c;
            }
            if (pass) write_proj(P, O, nproj, row, running + before + __popc(m & lanemask_lt()));
            running += total;
            __syncthreads();
        }
    }
}

// ---------------------------------------------------------------- dense aggregate, generic (variant 1)
struct DenseArgs {
    int32_t group_col[4];
    int32_t group_stride[4];
    int32_t ngroup_cols;
    int32_t n_groups;
    int32_t nagg;
    int32_t agg_op[QK_MAX_AGGS];
};

__device__ __forceinline__ double agg_identity(int op) {
    return op == QK_AGG_MIN ? __longlong_as_double(0x7ff0000000000000LL)
         : op == QK_AGG_MAX ? __longlong_as_double(0xfff0000000000000LL) : 0.0;
}
__device__ __forceinline__ double agg_combine(int op, double a, double b) {
    return op == QK_AGG_MIN ? fmin(a, b) : op == QK_AGG_MAX ? fmax(a, b) : a + b;
}

// CTA epilogue shared by all variants: reduce the NT lane-private copies of every slot and store the
// CTA partial.  acc layout: acc[(slot) * NT + tid], cnt[(g) * NT + tid].
template <int NT>
__device__ __forceinline__ void cta_flush(const double* acc, const unsigned* cnt, const DenseArgs& A,
                                          double* part_acc, long long* part_cnt) {
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = lane_id();
    const int nslots = A.n_groups * A.nagg;
    for (int s = warp; s < nslots; s += NT / 32) {
        const int op = A.agg_op[s % A.nagg];
        double v = agg_identity(op);
        for (int j = lane; j < NT; j += 32) v = agg_combine(op, v, acc[s * NT + j]);
        for (int o = 16; o; o >>= 1) v = agg_combine(op, v, __shfl_xor_sync(0xffffffffu, v, o));
        if (lane == 0) part_acc[(size_t)blockIdx.x * nslots + s] = v;
    }
    for (int g = warp; g < A.n_groups; g += NT / 32) {
        long long c = 0;
        for (int j = lane; j < NT; j += 32) c += cnt[g * NT + j];
        for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
        if (lane == 0) part_cnt[(size_t)blockIdx.x * A.n_groups + g] = c;
    }
}

template <int NT>
__device__ __forceinline__ void cta_init(double* acc, unsigned* cnt, const DenseArgs& A) {
    const int nslots = A.n_groups * A.nagg;
    for (int s = 0; s < nslots; ++s) acc[s * NT + threadIdx.x] = agg_identity(A.agg_op[s % A.nagg]);
    for (int g = 0; g < A.n_groups; ++g) cnt[g * NT + threadIdx.x] = 0u;
}

constexpr int GEN_NT = 256;
__global__ void __launch_bounds__(GEN_NT) k_dense_agg_generic(const __grid_constant__ Programs P, const __grid_constant__ DenseArgs A,
                                                              int64_t nrows, double* part_acc, long long* part_cnt) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    double* acc = (double*)smem_raw;
    unsigned* cnt = (unsigned*)(acc + (size_t)A.n_groups * A.nagg * GEN_NT);
    cta_init<GEN_NT>(acc, cnt, A);
    const int64_t stride = (int64_t)gridDim.x * GEN_NT;
    for (int64_t row = blockIdx.x * (int64_t)GEN_NT + threadIdx.x; row < nrows; row += stride) {
        if (!eval_pred(P, row)) continue;
        int g = 0;
        for (int k = 0; k < A.ngroup_cols; ++k)
            g += (int)load_i64(P.cols[A.group_col[k]].p, P.cols[A.group_col[k]].dt, row) * A.group_stride[k];
        g = min(max(g, 0), A.n_groups - 1);
        for (int j = 0; j < A.nagg; ++j) {
            double* a = &acc[(g * A.nagg + j) * GEN_NT + threadIdx.x];
            *a = agg_combine(A.agg_op[j], *a, eval_prog(P, 1 + j, row));
        }
        cnt[g * GEN_NT + threadIdx.x] += 1u;
    }
    cta_flush<GEN_NT>(acc, cnt, A, part_acc, part_cnt);
}

// fold per-CTA partials in a fixed order into the caller's running state
__global__ void k_dense_finalize(const double* part_acc, const long long* part_cnt, int nblocks,
                                 const __grid_constant__ DenseArgs A, double* acc, long long* cnt) {
    const int nslots = A.n_groups * A.nagg;
    for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < nslots + A.n_groups; s += gridDim.x * blockDim.x) {
        if (s < nslots) {
            const int op = A.agg_op[s % A.nagg];
            double v = agg_identity(op);
            for (int b = 0; b < nblocks; ++b) v = agg_combine(op, v, part_acc[(size_t)b * nslots + s]);
            // MIN/MAX states start at 0 in a zero-initialised caller buffer only if the group was never
            // seen; combine with the stored value only when the group already has rows
            const int g = s / A.nagg;
            long long seen = cnt[g];
            acc[s] = (op == QK_AGG_SUM || seen > 0) ? agg_combine(op, acc[s], v) : v;
        }
    }
    // counts are updated by a second launch-free phase: a grid-wide dependency is avoided by letting
    // the threads that own the count slots run after all acc slots of that group were read above is
    // NOT guaranteed across CTAs -> counts are folded by a separate kernel (k_dense_finalize_cnt).
}
__global__ void k_dense_finalize_cnt(const long long* part_cnt, int nblocks, int n_groups, long long* cnt) {
    for (int g = blockIdx.x * blockDim.x + threadIdx.x; g < n_groups; g += gridDim.x * blockDim.x) {
        long long c = 0;
        for (int b = 0; b < nblocks; ++b) c += part_cnt[(size_t)b * n_groups + g];
        cnt[g] += c;
    }
}

// ---------------------------------------------------------------- fused template plans (variants 2, 3)
// Operand kinds of an aggregate argument written as a product of affine factors of fp64 columns:
//   Col<S>        v[S]
//   KMinus<S,P>   par[P] - v[S]          (e.g. 1 - l_discount)
//   KPlus<S,P>    par[P] + v[S]          (e.g. 1 + l_tax)
// S indexes the plan's fp64 slots, P the constants in order of appearance.  pattern() emits the postfix
// token sequence the host compiler produces for the same expression, used to match a request to a plan.
struct Tok { int op; int slot; int par; };

template <int S> struct Col {
    template <class V> __device__ static __forceinline__ double eval(const V& v, const double*) { return v.f[S]; }
    static void pattern(std::vector<Tok>& t) { t.push_back({QK_OP_COL, S, -1}); }
};
template <int S, int P> struct KMinus {
    template <class V> __device__ static __forceinline__ double eval(const V& v, const double* par) { return par[P] - v.f[S]; }
    static void pattern(std::vector<Tok>& t) { t.push_back({QK_OP_CONST, -1, P}); t.push_back({QK_OP_COL, S, -1}); t.push_back({QK_OP_SUB, -1, -1}); }
};
template <int S, int P> struct KPlus {
    template <class V> __device__ static __forceinline__ double eval(const V& v, const double* par) { return par[P] + v.f[S]; }
    static void pattern(std::vector<Tok>& t) { t.push_back({QK_OP_CONST, -1, P}); t.push_back({QK_OP_COL, S, -1}); t.push_back({QK_OP_ADD, -1, -1}); }
};
template <class F0, class... Fs> struct Prod {
    template <class V> __device__ static __forceinline__ double eval(const V& v, const double* par) {
        double r = F0::eval(v, par);
        ((r = r * Fs::eval(v, par)), ...);          // left to right, like the postfix program
        return r;
    }
    static void pattern(std::vector<Tok>& t) {
        F0::pattern(t);
        ((Fs::pattern(t), t.push_back({QK_OP_MUL, -1, -1})), ...);
    }
};
template <class... As> struct AggList {
    static constexpr int N = sizeof...(As);
    template <class V, class F> __device__ static __forceinline__ void for_each(const V& v, const double* par, F&& f) {
        int j = 0;
        ((f(j++, As::eval(v, par))), ...);
    }
    static void patterns(std::vector<std::vector<Tok>>& out) {
        (([&] { std::vector<Tok> t; As::pattern(t); out.push_back(t); }()), ...);
    }
};

// A dense plan: optional predicate `icol <cmp> imm` on one integer column (dtype PRED_DT, 0 = none),
// NG group code columns (u8), NF fp64 measure columns, SUM aggregates from AggList.
template <int PRED_DT_, int NG_, int NF_, class Aggs_, int NPAR_>
struct DensePlan {
    static constexpr int PRED_DT = PRED_DT_, NG = NG_, NF = NF_, NAGG = Aggs_::N;
    static_assert(NPAR_ >= 0 && NPAR_ <= 8, "at most 8 constants");
    using Aggs = Aggs_;
};

struct FusedArgs {
    const void* pred_col;
    const uint8_t* gcol[2];
    const double* fcol[8];
    int32_t gstride[2];
    int32_t pred_neg;              // predicate = ((lo <= x) & (x <= hi)) != neg   (branch-free form of col <cmp> imm)
    int64_t pred_lo, pred_hi;
    double par[8];
};

// col <cmp> imm  ->  closed range [lo, hi] (+ negation for !=), clamped to the column's integer width
void range_of(int cmp, int64_t imm, int dt, FusedArgs& F) {
    const int64_t tmin = dt == QK_I32 ? INT32_MIN : INT64_MIN, tmax = dt == QK_I32 ? INT32_MAX : INT64_MAX;
    int64_t lo = tmin, hi = tmax;
    bool empty = false;
    F.pred_neg = 0;
    switch (cmp) {
        case QK_CMP_LT: if (imm <= tmin) empty = true; else hi = imm > tmax ? tmax : imm - 1; break;
        case QK_CMP_LE: if (imm < tmin) empty = true; else hi = imm > tmax ? tmax : imm; break;
        case QK_CMP_GT: if (imm >= tmax) empty = true; else lo = imm < tmin ? tmin : imm + 1; break;
        case QK_CMP_GE: if (imm > tmax) empty = true; else lo = imm < tmin ? tmin : imm; break;
        case QK_CMP_EQ: if (imm < tmin || imm > tmax) empty = true; else lo = hi = imm; break;
        default: F.pred_neg = 1; if (imm < tmin || imm > tmax) empty = true; else lo = hi = imm; break;   // !=
    }
    if (empty) { lo = 1; hi = 0; }
    F.pred_lo = lo; F.pred_hi = hi;
}

// closed range [lo, hi] (+ negation), clamped to the column's integer width
void range_closed(int64_t lo, int64_t hi, bool neg, int dt, FusedArgs& F) {
    const int64_t tmin = dt == QK_I32 ? INT32_MIN : INT64_MIN, tmax = dt == QK_I32 ? INT32_MAX : INT64_MAX;
    if (lo > tmax || hi < tmin || lo > hi) { lo = 1; hi = 0; }
    else { if (lo < tmin) lo = tmin; if (hi > tmax) hi = tmax; }
    F.pred_lo = lo; F.pred_hi = hi; F.pred_neg = neg ? 1 : 0;
}

template <int NF> struct RowVals { double f[NF]; };

constexpr int F_NT = 256;      // threads per CTA
constexpr int F_V = 4;         // rows per thread per tile
constexpr int F_TILE = F_NT * F_V;

__device__ __forceinline__ int4 ldg_nc_v4(const void* p) {
    int4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.s32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ unsigned ldg_nc_u32(const void* p) {
    unsigned r;
    asm volatile("ld.global.nc.L1::no_allocate.u32 %0, [%1];" : "=r"(r) : "l"(p));
    return r;
}

template <class Plan>
__device__ __forceinline__ bool pred_i32(int x, const FusedArgs& F) {
    return ((x >= (int)F.pred_lo) & (x <= (int)F.pred_hi)) != (F.pred_neg != 0);
}
template <class Plan>
__device__ __forceinline__ bool pred_i64(long long x, const FusedArgs& F) {
    return ((x >= F.pred_lo) & (x <= F.pred_hi)) != (F.pred_neg != 0);
}

// Branch-free: a row that fails the predicate adds 0.0 / 0 to its group, so the rows of a tile form one
// basic block and their loads are issued together.
template <class Plan, int NT>
__device__ __forceinline__ void accumulate_row(bool pass, int g, const RowVals<Plan::NF>& v, const FusedArgs& F,
                                               double* acc, unsigned* cnt) {
    Plan::Aggs::for_each(v, F.par, [&](int j, double x) {
        double* a = &acc[(g * Plan::NAGG + j) * NT + threadIdx.x];
        *a += pass ? x : 0.0;
    });
    cnt[g * NT + threadIdx.x] += pass ? 1u : 0u;
}

// variant 2: direct vector loads, 4 consecutive rows per thread
template <class Plan>
__global__ void __launch_bounds__(F_NT, 3) k_dense_agg_fused_ldg(const __grid_constant__ FusedArgs F, const __grid_constant__ DenseArgs A,
                                                                  int64_t nrows, double* part_acc, long long* part_cnt) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    double* acc = (double*)smem_raw;
    unsigned* cnt = (unsigned*)(acc + (size_t)A.n_groups * Plan::NAGG * F_NT);
    cta_init<F_NT>(acc, cnt, A);
    const int64_t ntiles = (nrows + F_TILE - 1) / F_TILE;
    for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int64_t base = tile * F_TILE + (int64_t)threadIdx.x * F_V;
        if (base + F_V <= nrows) {
            // ---- full vector path: issue every load before the first use
            int4 pv = make_int4(0, 0, 0, 0);
            int4 pw[2];
            if constexpr (Plan::PRED_DT == QK_I32) pv = ldg_nc_v4((const int32_t*)F.pred_col + base);
            if constexpr (Plan::PRED_DT == QK_I64) {
                pw[0] = ldg_nc_v4((const int64_t*)F.pred_col + base);
                pw[1] = ldg_nc_v4((const int64_t*)F.pred_col + base + 2);
            }
            unsigned gv[Plan::NG > 0 ? Plan::NG : 1];
#pragma unroll
            for (int k = 0; k < Plan::NG; ++k) gv[k] = ldg_nc_u32(F.gcol[k] + base);
            int4 fv[Plan::NF][2];
#pragma unroll
            for (int s = 0; s < Plan::NF; ++s) {
                fv[s][0] = ldg_nc_v4(F.fcol[s] + base);
                fv[s][1] = ldg_nc_v4(F.fcol[s] + base + 2);
            }
#pragma unroll
            for (int r = 0; r < F_V; ++r) {
                bool pass = true;
                if constexpr (Plan::PRED_DT == QK_I32) pass = pred_i32<Plan>(r == 0 ? pv.x : r == 1 ? pv.y : r == 2 ? pv.z : pv.w, F);
                if constexpr (Plan::PRED_DT == QK_I64) {
                    const int4 q = pw[r >> 1];
                    const long long x = (r & 1) ? (((long long)(unsigned)q.w << 32) | (unsigned)q.z) : (((long long)(unsigned)q.y << 32) | (unsigned)q.x);
                    pass = pred_i64<Plan>(x, F);
                }
                int g = 0;
#pragma unroll
                for (int k = 0; k < Plan::NG; ++k) g += (int)((gv[k] >> (8 * r)) & 0xffu) * F.gstride[k];
                g = min(g, A.n_groups - 1);
                RowVals<Plan::NF> v;
#pragma unroll
                for (int s = 0; s < Plan::NF; ++s) {
                    const int4 q = fv[s][r >> 1];
                    v.f[s] = (r & 1) ? __hiloint2double(q.w, q.z) : __hiloint2double(q.y, q.x);
                }
                accumulate_row<Plan, F_NT>(pass, g, v, F, acc, cnt);
            }
        } else {
            for (int r = 0; r < F_V; ++r) {
                const int64_t row = base + r;
                if (row >= nrows) break;
                bool pass = true;
                if constexpr (Plan::PRED_DT == QK_I32) pass = pred_i32<Plan>(((const int32_t*)F.pred_col)[row], F);
                if constexpr (Plan::PRED_DT == QK_I64) pass = pred_i64<Plan>(((const int64_t*)F.pred_col)[row], F);
                int g = 0;
#pragma unroll
                for (int k = 0; k < Plan::NG; ++k) g += (int)F.gcol[k][row] * F.gstride[k];
                g = min(g, A.n_groups - 1);
                RowVals<Plan::NF> v;
#pragma unroll
                for (int s = 0; s < Plan::NF; ++s) v.f[s] = F.fcol[s][row];
                accumulate_row<Plan, F_NT>(pass, g, v, F, acc, cnt);
            }
        }
    }
    cta_flush<F_NT>(acc, cnt, A, part_acc, part_cnt);
}

// variant 3+: TMA-engine (cp.async.bulk) staging of column tiles into shared memory.
// Shared-memory tile of TILE rows: fp64 columns first (8-byte aligned), then the predicate column, then
// the 1-byte group-code columns.  Every sub-array starts on a 16-byte boundary (TILE is a multiple of 16).
template <class Plan, int TILE> struct TileLayout {
    static constexpr int pred_bytes = Plan::PRED_DT == QK_I32 ? 4 : Plan::PRED_DT == QK_I64 ? 8 : 0;
    static constexpr int row_bytes = pred_bytes + Plan::NG + 8 * Plan::NF;
    static constexpr int off_f = 0;
    static constexpr int off_pred = 8 * Plan::NF * TILE;
    static constexpr int off_g = off_pred + pred_bytes * TILE;
    static constexpr int stage_bytes = row_bytes * TILE;
    static_assert(TILE % 16 == 0, "bulk copies need 16-byte multiples");
};

template <class Plan, int TILE>
__device__ __forceinline__ void tma_issue_tile(const FusedArgs& F, int64_t tile, unsigned char* stage, unsigned bar) {
    using L = TileLayout<Plan, TILE>;
    const int64_t base = tile * TILE;
    mbar_expect_tx(bar, (unsigned)L::stage_bytes);
#pragma unroll
    for (int s = 0; s < Plan::NF; ++s) bulk_g2s(smem_u32(stage + L::off_f + s * 8 * TILE), F.fcol[s] + base, 8 * TILE, bar);
    if constexpr (L::pred_bytes > 0)
        bulk_g2s(smem_u32(stage + L::off_pred), (const unsigned char*)F.pred_col + base * L::pred_bytes, L::pred_bytes * TILE, bar);
#pragma unroll
    for (int k = 0; k < Plan::NG; ++k) bulk_g2s(smem_u32(stage + L::off_g + k * TILE), F.gcol[k] + base, TILE, bar);
}

template <class Plan, int NT, int V, int STAGES>
__global__ void __launch_bounds__(NT, 1) k_dense_agg_fused_tma(const __grid_constant__ FusedArgs F, const __grid_constant__ DenseArgs A,
                                                               int64_t nrows, double* part_acc, long long* part_cnt) {
    constexpr int TILE = NT * V;
    using L = TileLayout<Plan, TILE>;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    __shared__ __align__(8) unsigned long long bars[STAGES];
    unsigned char* stages = smem_raw;                                        // STAGES * stage_bytes
    double* acc = (double*)(smem_raw + (size_t)STAGES * L::stage_bytes);
    unsigned* cnt = (unsigned*)(acc + (size_t)A.n_groups * Plan::NAGG * NT);
    cta_init<NT>(acc, cnt, A);
    const int64_t nfull = nrows / TILE;                                      // full tiles go through TMA
    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; ++s) mbar_init(smem_u32(&bars[s]), 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    // my tiles: blockIdx.x, +gridDim.x, ...
    const int64_t my_n = nfull > blockIdx.x ? (nfull - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES && s < my_n; ++s)
            tma_issue_tile<Plan, TILE>(F, blockIdx.x + (int64_t)s * gridDim.x, stages + (size_t)s * L::stage_bytes, smem_u32(&bars[s]));
    }
    int s = 0;
    unsigned parity = 0;
    for (int64_t it = 0; it < my_n; ++it) {
        mbar_wait(smem_u32(&bars[s]), parity);
        const unsigned char* st = stages + (size_t)s * L::stage_bytes;
        // gather the thread's V rows (strided by NT: conflict-free shared loads) before touching the states
        bool pass[V];
        int g[V];
        RowVals<Plan::NF> v[V];
#pragma unroll
        for (int r = 0; r < V; ++r) {
            const int t = r * NT + threadIdx.x;
            pass[r] = true;
            if constexpr (Plan::PRED_DT == QK_I32) pass[r] = pred_i32<Plan>(((const int32_t*)(st + L::off_pred))[t], F);
            if constexpr (Plan::PRED_DT == QK_I64) pass[r] = pred_i64<Plan>(((const int64_t*)(st + L::off_pred))[t], F);
            int gg = 0;
#pragma unroll
            for (int k = 0; k < Plan::NG; ++k) gg += (int)st[L::off_g + k * TILE + t] * F.gstride[k];
            g[r] = min(gg, A.n_groups - 1);
#pragma unroll
            for (int q = 0; q < Plan::NF; ++q) v[r].f[q] = ((const double*)(st + L::off_f + q * 8 * TILE))[t];
        }
#pragma unroll
        for (int r = 0; r < V; ++r) accumulate_row<Plan, NT>(pass[r], g[r], v[r], F, acc, cnt);
        __syncthreads();                                   // every thread is done with stage s
        if (threadIdx.x == 0 && it + STAGES < my_n)
            tma_issue_tile<Plan, TILE>(F, blockIdx.x + (it + STAGES) * gridDim.x, stages + (size_t)s * L::stage_bytes, smem_u32(&bars[s]));
        if (++s == STAGES) { s = 0; parity ^= 1u; }
    }
    // ragged tail (< TILE rows): plain loads, handled by CTA 0
    if (blockIdx.x == 0) {
        for (int64_t row = nfull * TILE + threadIdx.x; row < nrows; row += NT) {
            bool pass = true;
            if constexpr (Plan::PRED_DT == QK_I32) pass = pred_i32<Plan>(((const int32_t*)F.pred_col)[row], F);
            if constexpr (Plan::PRED_DT == QK_I64) pass = pred_i64<Plan>(((const int64_t*)F.pred_col)[row], F);
            int g = 0;
#pragma unroll
            for (int k = 0; k < Plan::NG; ++k) g += (int)F.gcol[k][row] * F.gstride[k];
            g = min(g, A.n_groups - 1);
            RowVals<Plan::NF> v;
#pragma unroll
            for (int q = 0; q < Plan::NF; ++q) v.f[q] = F.fcol[q][row];
            accumulate_row<Plan, NT>(pass, g, v, F, acc, cnt);
        }
    }
    cta_flush<NT>(acc, cnt, A, part_acc, part_cnt);
}

// ---------------------------------------------------------------- plan registry + matcher
struct Request {           // what the caller asked for, in host terms
    const qk_column* cols; int ncols; int64_t nrows;
    const qk_expr* pred;
    const int32_t* group_cols; const int32_t* group_card; int ngroup_cols;
    const qk_expr* agg_expr; const int32_t* agg_op; int nagg;
};

template <class Plan>
bool match_plan(const Request& R, FusedArgs& F) {
    if (R.nagg != Plan::NAGG || R.ngroup_cols != Plan::NG) return false;
    for (int j = 0; j < R.nagg; ++j) if (R.agg_op[j] != QK_AGG_SUM) return false;
    // predicate: none, or exactly one CMP_COL_IMM on a column of the plan's predicate dtype
    const int npred = R.pred ? R.pred->n_nodes : 0;
    if (Plan::PRED_DT == 0) { if (npred != 0) return false; }
    else {
        if (npred != 1 || (R.pred->nodes[0].op != QK_OP_CMP_COL_IMM && R.pred->nodes[0].op != QK_OP_RANGE_COL_IMM)) return false;
        const qk_expr_node& nd = R.pred->nodes[0];
        if (R.cols[nd.a0].dtype != Plan::PRED_DT) return false;
        F.pred_col = R.cols[nd.a0].data;
        if (nd.op == QK_OP_CMP_COL_IMM) range_of(nd.a1, nd.imm_i, Plan::PRED_DT, F);
        else range_closed(nd.imm_i, (int64_t)nd.imm, nd.a1 != 0, Plan::PRED_DT, F);
    }
    int stride = 1;
    for (int k = Plan::NG - 1; k >= 0; --k) {      // row-major group id: first key most significant
        const qk_column& c = R.cols[R.group_cols[k]];
        if (c.dtype != QK_U8) return false;
        F.gcol[k] = (const uint8_t*)c.data; F.gstride[k] = stride; stride *= R.group_card[k];
    }
    std::vector<std::vector<Tok>> pats;
    Plan::Aggs::patterns(pats);
    int slot_col[8]; for (int s = 0; s < 8; ++s) slot_col[s] = -1;
    for (int j = 0; j < R.nagg; ++j) {
        const qk_expr& e = R.agg_expr[j];
        if ((int)pats[j].size() != e.n_nodes) return false;
        for (int i = 0; i < e.n_nodes; ++i) {
            const Tok& t = pats[j][i]; const qk_expr_node& nd = e.nodes[i];
            if (t.op != nd.op) return false;
            if (t.op == QK_OP_COL) {
                if (R.cols[nd.a0].dtype != QK_F64) return false;
                if (slot_col[t.slot] == -1) {
                    for (int s = 0; s < 8; ++s) if (slot_col[s] == nd.a0) return false;   // injective
                    slot_col[t.slot] = nd.a0;
                } else if (slot_col[t.slot] != nd.a0) return false;
            } else if (t.op == QK_OP_CONST) F.par[t.par] = nd.imm;
        }
    }
    for (int s = 0; s < Plan::NF; ++s) { if (slot_col[s] < 0) return false; F.fcol[s] = (const double*)R.cols[slot_col[s]].data; }
    // vector loads need 16-byte aligned column bases
    auto al = [](const void* p) { return ((uintptr_t)p & 15) == 0; };
    if (Plan::PRED_DT && !al(F.pred_col)) return false;
    for (int k = 0; k < Plan::NG; ++k) if (!al(F.gcol[k])) return false;
    for (int s = 0; s < Plan::NF; ++s) if (!al(F.fcol[s])) return false;
    return true;
}

// --- the instantiated plans -------------------------------------------------------------------
// Q1 (apps/tpc-h/tpch.py:108-117 after de-duplicating the AVG partial sums): pred on a date32 column,
// 2 code keys, fp64 slots {0: qty, 1: extendedprice, 2: discount, 3: tax}
using PlanQ1 = DensePlan<QK_I32, 2, 4,
    AggList<Prod<Col<0>>, Prod<Col<1>>, Prod<Col<1>, KMinus<2, 0>>, Prod<Col<1>, KMinus<2, 1>, KPlus<3, 2>>, Prod<Col<2>>>, 3>;
// sum(a * (k - b)) by one code key, optional date predicate (Q5 / Q3-style revenue by a dictionary key)
using PlanRev1 = DensePlan<QK_I32, 1, 2, AggList<Prod<Col<0>, KMinus<1, 0>>>, 1>;
// sum(a * b) ungrouped with a date predicate is Q6-like; grouped by one key here
using PlanMul1 = DensePlan<QK_I32, 1, 2, AggList<Prod<Col<0>, Col<1>>>, 0>;

thread_local std::string g_variant, g_variant_cfg;

template <class Plan, int NT, int V, int STAGES>
int launch_tma(const FusedArgs& F, const DenseArgs& A, int64_t nrows, double* part_acc, long long* part_cnt,
               int* nblocks_out, cudaStream_t st, const char* name) {
    using L = TileLayout<Plan, NT * V>;
    const size_t acc_bytes = (size_t)A.n_groups * (Plan::NAGG * 8 + 4) * NT;
    const size_t smem = (size_t)STAGES * L::stage_bytes + acc_bytes;
    if (smem > 227 * 1024 - 64) return 1;     // does not fit: caller tries the next configuration
    auto kern = k_dense_agg_fused_tma<Plan, NT, V, STAGES>;
    QK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int sms = sm_count();
    const int64_t nfull = nrows / (NT * V);
    int nb = (int)(nfull < sms ? (nfull > 0 ? nfull : 1) : sms);       // persistent: one CTA per SM
    kern<<<nb, NT, smem, st>>>(F, A, nrows, part_acc, part_cnt);
    QK_LAUNCH_CHECK("k_dense_agg_fused_tma");
    *nblocks_out = nb;
    char buf[96];
    snprintf(buf, sizeof buf, "fused_tma:%s", name);
    g_variant = buf;
    g_variant_cfg = std::string("nt") + std::to_string(NT) + "v" + std::to_string(V) + "s" + std::to_string(STAGES);
    return 0;
}

template <class Plan>
int launch_fused(const FusedArgs& F, const DenseArgs& A, int64_t nrows, int variant, double* part_acc,
                 long long* part_cnt, int* nblocks_out, cudaStream_t st, const char* name) {
    // variant 3 = default TMA configuration; 4..6 = alternative (threads, rows/thread, stages) shapes kept
    // selectable for profiling
    switch (variant) {
        case 3: {   // default shape: 256 threads x 4 rows, 3 stages
            int rc = launch_tma<Plan, 256, 4, 3>(F, A, nrows, part_acc, part_cnt, nblocks_out, st, name);
            if (rc == 1) rc = launch_tma<Plan, 256, 2, 3>(F, A, nrows, part_acc, part_cnt, nblocks_out, st, name);
            if (rc == 1) rc = launch_tma<Plan, 256, 1, 3>(F, A, nrows, part_acc, part_cnt, nblocks_out, st, name);
            return rc;
        }
        case 4: return launch_tma<Plan, 512, 2, 2>(F, A, nrows, part_acc, part_cnt, nblocks_out, st, name);
        case 5: return launch_tma<Plan, 512, 1, 4>(F, A, nrows, part_acc, part_cnt, nblocks_out, st, name);
        case 6: return launch_tma<Plan, 256, 2, 6>(F, A, nrows, part_acc, part_cnt, nblocks_out, st, name);
        default: break;
    }
    const size_t acc_bytes = (size_t)A.n_groups * (Plan::NAGG * 8 + 4) * F_NT;
    const int sms = sm_count();
    if (acc_bytes > 110 * 1024) return 1;
    auto kern = k_dense_agg_fused_ldg<Plan>;
    QK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)acc_bytes));
    const int64_t ntiles = (nrows + F_TILE - 1) / F_TILE;
    int per_sm = (int)((220 * 1024) / (acc_bytes + 1024));      // resident CTAs per SM (shared-memory bound)
    if (per_sm > 3) per_sm = 3;
    if (per_sm < 1) per_sm = 1;
    int nb = (int)(ntiles < (int64_t)per_sm * sms ? (ntiles > 0 ? ntiles : 1) : per_sm * sms);
    kern<<<nb, F_NT, acc_bytes, st>>>(F, A, nrows, part_acc, part_cnt);
    QK_LAUNCH_CHECK("k_dense_agg_fused_ldg");
    *nblocks_out = nb;
    g_variant = std::string("fused_ldg:") + name;
    g_variant_cfg = "nt256v4";
    return 0;
}


// ---------------------------------------------------------------- dynamic fused plan (variant 3 for every other shape)
// The typed plans above cover the headline query at the speed of light; every OTHER aggregate of the grammar
//     predicate  = AND of terms:  int column <cmp> constant | fp column <cmp> constant | code column IN set | NOT term
//     group keys = 0..4 code columns
//     aggregate  = SUM / MIN / MAX of  f1 * f2 * f3,  f = k0 + k1 * column,  optionally gated: CASE WHEN term THEN .. ELSE 0
// (Q6, Q14, Q19-, Q12-shaped partial aggregates) runs through the SAME TMA tile ring with a runtime-described plan
// instead of the per-row postfix interpreter: the columns a plan touches are staged tile by tile with cp.async.bulk, a
// row costs one shared-memory read per factor / term, and the partial states are the same lane-private accumulators.
constexpr int DY_MAXCOLS = 10;
constexpr int DY_MAXTERMS = 6;
constexpr int DY_MAXFACT = 3;
struct DyTerm {
    int8_t col, kind, neg, lo_open, hi_open;         // kind 0: integer range, 1: fp64 range, 2: set membership, 3: column <cmp> column
    int8_t col2, cmp, w;                             // kind 3: the other column and the QK_CMP_* code; w: byte width of the integer column(s)
    int32_t nbits;
    int32_t soff;                                    // byte offset of the column's tile inside a stage (= off[col])
    long long ilo, ihi;
    double flo, fhi;
    unsigned long long bits;                         // inline bitmap (nbits <= 64) or device pointer
    int32_t soff2, pad2;                             // kind 3: off[col2]
};
struct DyFactor { double k0, k1; int32_t col; int32_t soff; };     // col < 0: the constant k0; soff = off[col]
struct DyAgg {
    DyFactor f[DY_MAXFACT]; int32_t nfact; int32_t gate;              // gate: index of a DyTerm or -1
    int32_t start, pad;                                              // typed tile walk: factors [0, start) are the previous aggregate's
};                                                                   // whole product (Q1: price*(1-disc) then *(1+tax)) -- continue from it
struct DyArgs {
    const unsigned char* src[DY_MAXCOLS];
    int32_t off[DY_MAXCOLS];                         // byte offset of the column's tile inside a stage
    int8_t width[DY_MAXCOLS], dtype[DY_MAXCOLS];
    int32_t ncols, stage_bytes, nterms;
    DyTerm term[DY_MAXTERMS + QK_MAX_AGGS];
    int32_t gcol[4], goff[4];                        // goff = off[gcol]
    int8_t gw[4];                                    // byte width of the key columns (typed walk: 1 or 4)
    DyAgg agg[QK_MAX_AGGS];
};

// staged: column c of the tile lives at stage + off[c]; unstaged (ragged tail): straight from global memory
__device__ __forceinline__ const unsigned char* dy_base(const DyArgs& D, const unsigned char* stage, int c) {
    return stage ? stage + D.off[c] : D.src[c];
}
// FAST = the column types every TPC-H-shaped plan has (int32 range terms, fp64 compare terms and factors, uint8 code columns for
// sets and group keys): typed loads instead of a dtype switch per access.
template <bool FAST = false>
__device__ __forceinline__ bool dy_term(const DyArgs& D, const DyTerm& T, const unsigned char* stage, int64_t i) {
    const unsigned char* p = dy_base(D, stage, T.col);
    const int dt = D.dtype[T.col];
    bool r;
    if (T.kind == 0) {
        if constexpr (FAST) {
            const int x = ((const int*)p)[i];
            r = (x >= (int)T.ilo) & (x <= (int)T.ihi);
        } else {
            const long long x = load_i64(p, dt, i);
            r = (x >= T.ilo) & (x <= T.ihi);
        }
    } else if (T.kind == 1) {
        const double v = FAST ? ((const double*)p)[i] : load_f64(p, dt, i);
        r = (T.lo_open ? v > T.flo : v >= T.flo) & (T.hi_open ? v < T.fhi : v <= T.fhi);
    } else if (T.kind == 3) {
        r = cmp_i64(load_i64(p, dt, i), T.cmp, load_i64(dy_base(D, stage, T.col2), D.dtype[T.col2], i));
    } else {
        const long long code = FAST ? (long long)p[i] : load_i64(p, dt, i);
        r = false;
        if (code >= 0 && code < (long long)T.nbits)
            r = T.nbits <= 64 ? ((T.bits >> code) & 1ull) != 0 : ((__ldg((const unsigned*)(uintptr_t)T.bits + (code >> 5)) >> (code & 31)) & 1u) != 0;
    }
    return r != (T.neg != 0);
}

template <int NT>
__device__ __forceinline__ void dy_row(const DyArgs& D, const DenseArgs& A, const unsigned char* stage, int64_t i, double* acc, unsigned* cnt) {
    bool pass = true;
    for (int k = 0; k < D.nterms; ++k) pass &= dy_term(D, D.term[k], stage, i);
    int g = 0;
    for (int k = 0; k < A.ngroup_cols; ++k)
        g += (int)load_i64(dy_base(D, stage, D.gcol[k]), D.dtype[D.gcol[k]], i) * A.group_stride[k];
    g = min(max(g, 0), A.n_groups - 1);
    for (int j = 0; j < A.nagg; ++j) {
        const DyAgg& G = D.agg[j];
        double x = 1.0;
        for (int f = 0; f < G.nfact; ++f) {
            const DyFactor& F = G.f[f];
            double v = F.k0;
            if (F.col >= 0) {
                const double c = load_f64(dy_base(D, stage, F.col), D.dtype[F.col], i);
                v = (F.k0 == 0.0 && F.k1 == 1.0) ? c : F.k0 + F.k1 * c;
            }
            x = f == 0 ? v : x * v;
        }
        if (G.gate >= 0 && !dy_term(D, D.term[G.gate], stage, i)) x = 0.0;
        double* a = &acc[(g * A.nagg + j) * NT + threadIdx.x];
        const int op = A.agg_op[j];
        if (op == QK_AGG_SUM) *a += pass ? x : 0.0;
        else if (pass) *a = agg_combine(op, *a, x);
    }
    cnt[g * NT + threadIdx.x] += pass ? 1u : 0u;
}

// V rows of one thread at once, every step over all V rows before the next step: the loads of a step (one per row) are
// independent, so V of them are in flight per thread instead of one dependent chain per row (with 8 warps per SM and a
// serial per-row walk the kernel is bound by shared-memory latency, not by HBM).  Rows are idx0 + r * stride.
template <int NT, int V, bool FAST>
__device__ __forceinline__ void dy_rows(const DyArgs& D, const DenseArgs& A, const unsigned char* stage, int64_t idx0, int64_t stride,
                                        double* acc, unsigned* cnt) {
    bool pass[V];
    int g[V];
#pragma unroll
    for (int r = 0; r < V; ++r) { pass[r] = true; g[r] = 0; }
    for (int k = 0; k < D.nterms; ++k) {
#pragma unroll
        for (int r = 0; r < V; ++r) pass[r] &= dy_term<FAST>(D, D.term[k], stage, idx0 + r * stride);
    }
    for (int k = 0; k < A.ngroup_cols; ++k) {
        const unsigned char* p = dy_base(D, stage, D.gcol[k]);
        const int dt = D.dtype[D.gcol[k]], gs = A.group_stride[k];
#pragma unroll
        for (int r = 0; r < V; ++r) g[r] += (FAST ? (int)p[idx0 + r * stride] : (int)load_i64(p, dt, idx0 + r * stride)) * gs;
    }
#pragma unroll
    for (int r = 0; r < V; ++r) g[r] = min(max(g[r], 0), A.n_groups - 1);
    for (int j = 0; j < A.nagg; ++j) {
        const DyAgg& G = D.agg[j];
        double x[V];
        for (int f = 0; f < G.nfact; ++f) {
            const DyFactor& F = G.f[f];
            const bool plain = F.k0 == 0.0 && F.k1 == 1.0;
            const unsigned char* p = F.col >= 0 ? dy_base(D, stage, F.col) : nullptr;
            const int dt = F.col >= 0 ? D.dtype[F.col] : 0;
#pragma unroll
            for (int r = 0; r < V; ++r) {
                double v = F.k0;
                if (p) {
                    const double c = FAST ? ((const double*)p)[idx0 + r * stride] : load_f64(p, dt, idx0 + r * stride);
                    v = plain ? c : F.k0 + F.k1 * c;
                }
                x[r] = f == 0 ? v : x[r] * v;
            }
        }
        if (G.gate >= 0) {
#pragma unroll
            for (int r = 0; r < V; ++r) if (!dy_term<FAST>(D, D.term[G.gate], stage, idx0 + r * stride)) x[r] = 0.0;
        }
        const int op = A.agg_op[j];
#pragma unroll
        for (int r = 0; r < V; ++r) {
            double* a = &acc[(g[r] * A.nagg + j) * NT + threadIdx.x];
            if (op == QK_AGG_SUM) *a += pass[r] ? x[r] : 0.0;
            else if (pass[r]) *a = agg_combine(op, *a, x[r]);
        }
    }
#pragma unroll
    for (int r = 0; r < V; ++r) cnt[g[r] * NT + threadIdx.x] += pass[r] ? 1u : 0u;
}

// ---- the typed tile walk (FAST plans: int32 range terms, fp64 compare terms and factors, uint8 sets and group keys)
// A descriptor (term / factor / key) is decoded ONCE per tile into registers and then applied to the thread's V rows, with
// 32-bit shared-memory addresses: the first version decoded per row through generic pointers and spent ~290 instructions per
// row, 2/3 of them IMAD / LDC / ISETP / BRA of the walk itself -- it was bound by issue slots.
__device__ __forceinline__ int lds_i32(unsigned a) { int v; asm volatile("ld.shared.s32 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
__device__ __forceinline__ unsigned lds_u8(unsigned a) { unsigned v; asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
__device__ __forceinline__ long long lds_i64(unsigned a) { long long v; asm volatile("ld.shared.s64 %0, [%1];" : "=l"(v) : "r"(a)); return v; }
__device__ __forceinline__ double lds_f64(unsigned a) { double v; asm volatile("ld.shared.f64 %0, [%1];" : "=d"(v) : "r"(a)); return v; }

template <int NT, int V>
__device__ __forceinline__ void dy_term_tile(const DyTerm& T, unsigned sb, bool (&ok)[V]) {
    const unsigned a = sb + (unsigned)T.soff;
    const bool neg = T.neg != 0;
    if (T.kind == 0) {
        if (T.w == 4) {
            const int lo = (int)T.ilo, hi = (int)T.ihi;
            const unsigned a0 = a + threadIdx.x * 4u;
#pragma unroll
            for (int r = 0; r < V; ++r) { const int x = lds_i32(a0 + r * NT * 4); ok[r] = ((x >= lo) & (x <= hi)) != neg; }
        } else {
            const long long lo = T.ilo, hi = T.ihi;
            const unsigned a0 = a + threadIdx.x * 8u;
#pragma unroll
            for (int r = 0; r < V; ++r) { const long long x = lds_i64(a0 + r * NT * 8); ok[r] = ((x >= lo) & (x <= hi)) != neg; }
        }
    } else if (T.kind == 3) {                              // column <cmp> column, both int32 or both int64 (Q5: c_nationkey = s_nationkey)
        const unsigned b = sb + (unsigned)T.soff2;
        const int cmp = T.cmp;
        if (T.w == 4) {
#pragma unroll
            for (int r = 0; r < V; ++r)
                ok[r] = cmp_i64(lds_i32(a + (threadIdx.x + r * NT) * 4u), cmp, lds_i32(b + (threadIdx.x + r * NT) * 4u)) != neg;
        } else {
#pragma unroll
            for (int r = 0; r < V; ++r)
                ok[r] = cmp_i64(lds_i64(a + (threadIdx.x + r * NT) * 8u), cmp, lds_i64(b + (threadIdx.x + r * NT) * 8u)) != neg;
        }
    } else if (T.kind == 1) {                              // bounds are closed here (match_dyn moves open ones by one ulp)
        const double lo = T.flo, hi = T.fhi;
        const unsigned a0 = a + threadIdx.x * 8u;
#pragma unroll
        for (int r = 0; r < V; ++r) { const double v = lds_f64(a0 + r * NT * 8); ok[r] = ((v >= lo) & (v <= hi)) != neg; }
    } else {
        const unsigned nbits = (unsigned)T.nbits, a0 = a + threadIdx.x;
        const unsigned long long bits = T.bits;
        if (nbits <= 64) {
#pragma unroll
            for (int r = 0; r < V; ++r) { const unsigned c = lds_u8(a0 + r * NT); ok[r] = ((c < nbits) & (((bits >> (c & 63u)) & 1ull) != 0)) != neg; }
        } else {
            const unsigned* words = (const unsigned*)(uintptr_t)bits;
#pragma unroll
            for (int r = 0; r < V; ++r) {
                const unsigned c = lds_u8(a0 + r * NT);
                ok[r] = (c < nbits && ((__ldg(words + (c >> 5)) >> (c & 31u)) & 1u) != 0) != neg;
            }
        }
    }
}

template <int NT, int V>
__device__ __forceinline__ void dy_tile_fast(const DyArgs& D, const DenseArgs& A, unsigned sb, double* acc, unsigned* cnt) {
    bool pass[V], ok[V];
    int g[V];
#pragma unroll
    for (int r = 0; r < V; ++r) { pass[r] = true; g[r] = 0; }
    const int nterms = D.nterms, ngc = A.ngroup_cols, nagg = A.nagg;
    for (int k = 0; k < nterms; ++k) {
        dy_term_tile<NT, V>(D.term[k], sb, ok);
#pragma unroll
        for (int r = 0; r < V; ++r) pass[r] &= ok[r];
    }
    if (ngc > 0) {
        for (int k = 0; k < ngc; ++k) {
            const int gs = A.group_stride[k];
            if (D.gw[k] == 1) {
                const unsigned a0 = sb + (unsigned)D.goff[k] + threadIdx.x;
#pragma unroll
                for (int r = 0; r < V; ++r) g[r] += (int)lds_u8(a0 + r * NT) * gs;
            } else {
                const unsigned a0 = sb + (unsigned)D.goff[k] + threadIdx.x * 4u;
#pragma unroll
                for (int r = 0; r < V; ++r) g[r] += lds_i32(a0 + r * NT * 4) * gs;
            }
        }
        const int top = A.n_groups - 1;
#pragma unroll
        for (int r = 0; r < V; ++r) g[r] = min(max(g[r], 0), top);
    }
    double x[V];
    for (int j = 0; j < nagg; ++j) {
        const DyAgg& G = D.agg[j];
        const int nfact = G.nfact;
        for (int f = G.start; f < nfact; ++f) {
            const DyFactor& F = G.f[f];
            const double k0 = F.k0, k1 = F.k1;
            double v[V];
            if (F.col < 0) {
#pragma unroll
                for (int r = 0; r < V; ++r) v[r] = k0;
            } else {
                const unsigned a0 = sb + (unsigned)F.soff + threadIdx.x * 8u;
                if (k0 == 0.0 && k1 == 1.0) {
#pragma unroll
                    for (int r = 0; r < V; ++r) v[r] = lds_f64(a0 + r * NT * 8);
                } else {
#pragma unroll
                    for (int r = 0; r < V; ++r) v[r] = k0 + k1 * lds_f64(a0 + r * NT * 8);
                }
            }
            if (f == 0) {
#pragma unroll
                for (int r = 0; r < V; ++r) x[r] = v[r];
            } else {
#pragma unroll
                for (int r = 0; r < V; ++r) x[r] *= v[r];
            }
        }
        bool on[V];
#pragma unroll
        for (int r = 0; r < V; ++r) on[r] = pass[r];
        if (G.gate >= 0) {                                 // CASE WHEN term THEN product ELSE 0 (SUM only): the row adds 0
            dy_term_tile<NT, V>(D.term[G.gate], sb, ok);
#pragma unroll
            for (int r = 0; r < V; ++r) on[r] &= ok[r];
        }
        const int op = A.agg_op[j];
        double* aj = acc + (size_t)j * NT + threadIdx.x;
        if (op == QK_AGG_SUM) {
#pragma unroll
            for (int r = 0; r < V; ++r) { double* a = aj + g[r] * nagg * NT; *a += on[r] ? x[r] : 0.0; }
        } else {
#pragma unroll
            for (int r = 0; r < V; ++r) if (on[r]) { double* a = aj + g[r] * nagg * NT; *a = agg_combine(op, *a, x[r]); }
        }
    }
#pragma unroll
    for (int r = 0; r < V; ++r) cnt[g[r] * NT + threadIdx.x] += pass[r] ? 1u : 0u;
}

template <int NT, int V, int STAGES, bool FAST>
__global__ void __launch_bounds__(NT, 1) k_dense_agg_dyn_tma(const __grid_constant__ DyArgs D, const __grid_constant__ DenseArgs A,
                                                             int64_t nrows, double* part_acc, long long* part_cnt) {
    constexpr int TILE = NT * V;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    __shared__ __align__(8) unsigned long long bars[STAGES];
    unsigned char* stages = smem_raw;
    double* acc = (double*)(smem_raw + (size_t)STAGES * D.stage_bytes);
    unsigned* cnt = (unsigned*)(acc + (size_t)A.n_groups * A.nagg * NT);
    cta_init<NT>(acc, cnt, A);
    const int64_t nfull = nrows / TILE;
    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; ++s) mbar_init(smem_u32(&bars[s]), 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const int64_t my_n = nfull > blockIdx.x ? (nfull - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
    auto issue = [&](int64_t tile, int s) {
        const unsigned bar = smem_u32(&bars[s]);
        unsigned char* st = stages + (size_t)s * D.stage_bytes;
        mbar_expect_tx(bar, (unsigned)D.stage_bytes);
        for (int c = 0; c < D.ncols; ++c)
            bulk_g2s(smem_u32(st + D.off[c]), D.src[c] + tile * TILE * D.width[c], (unsigned)(TILE * D.width[c]), bar);
    };
    if (threadIdx.x == 0)
        for (int s = 0; s < STAGES && s < my_n; ++s) issue(blockIdx.x + (int64_t)s * gridDim.x, s);
    int s = 0;
    unsigned parity = 0;
    for (int64_t it = 0; it < my_n; ++it) {
        mbar_wait(smem_u32(&bars[s]), parity);
        const unsigned char* st = stages + (size_t)s * D.stage_bytes;
        if constexpr (FAST) dy_tile_fast<NT, V>(D, A, smem_u32(st), acc, cnt);
        else dy_rows<NT, V, false>(D, A, st, threadIdx.x, NT, acc, cnt);
        __syncthreads();
        if (threadIdx.x == 0 && it + STAGES < my_n) issue(blockIdx.x + (it + STAGES) * gridDim.x, s);
        if (++s == STAGES) { s = 0; parity ^= 1u; }
    }
    if (blockIdx.x == 0)
        for (int64_t row = nfull * TILE + threadIdx.x; row < nrows; row += NT) dy_row<NT>(D, A, nullptr, row, acc, cnt);
    cta_flush<NT>(acc, cnt, A, part_acc, part_cnt);
}

// ---- host: postfix programs -> DyArgs
struct ExNode { int op, a0, a1; double imm; long long imm_i; int l, r, c; };
static bool ex_tree(const qk_expr* e, std::vector<ExNode>& out, int* root) {
    std::vector<int> st;
    const int n = e ? e->n_nodes : 0;
    for (int i = 0; i < n; ++i) {
        const qk_expr_node& nd = e->nodes[i];
        ExNode x{nd.op, nd.a0, nd.a1, nd.imm, nd.imm_i, -1, -1, -1};
        switch (nd.op) {
            case QK_OP_COL: case QK_OP_CONST: case QK_OP_CMP_COL_IMM: case QK_OP_CMP_COL_COL: case QK_OP_IN_SET: case QK_OP_RANGE_COL_IMM: break;
            case QK_OP_NEG: case QK_OP_NOT: case QK_OP_RINT: case QK_OP_EXTRACT:
                if (st.empty()) return false;
                x.l = st.back(); st.pop_back(); break;
            case QK_OP_SELECT:
                if (st.size() < 3) return false;
                x.c = st[st.size() - 3]; x.l = st[st.size() - 2]; x.r = st[st.size() - 1];
                st.resize(st.size() - 3); break;
            default:
                if (st.size() < 2) return false;
                x.l = st[st.size() - 2]; x.r = st[st.size() - 1];
                st.resize(st.size() - 2); break;
        }
        out.push_back(x);
        st.push_back((int)out.size() - 1);
    }
    if (st.size() != 1) return false;
    *root = st[0];
    return true;
}

struct DyBuilder {
    const Request& R;
    DyArgs& D;
    int slot_of[QK_MAX_COLS];
    explicit DyBuilder(const Request& r, DyArgs& d) : R(r), D(d) { for (int& s : slot_of) s = -1; D.ncols = 0; }
    int slot(int col) {                      // staged slot of input column `col` (-1: does not fit)
        if (col < 0 || col >= R.ncols) return -1;
        if (slot_of[col] >= 0) return slot_of[col];
        if (D.ncols >= DY_MAXCOLS || ((uintptr_t)R.cols[col].data & 15)) return -1;
        const int s = D.ncols++;
        D.src[s] = (const unsigned char*)R.cols[col].data;
        D.width[s] = (int8_t)dtype_size(R.cols[col].dtype); D.dtype[s] = (int8_t)R.cols[col].dtype;
        return slot_of[col] = s;
    }
    bool term(const std::vector<ExNode>& T, int i, DyTerm& out) {
        const ExNode& x = T[i];
        out = DyTerm{};
        if (x.op == QK_OP_NOT) {
            if (!term(T, x.l, out)) return false;
            out.neg = !out.neg;
            return true;
        }
        if (x.op == QK_OP_CMP_COL_IMM) {
            const int s = slot(x.a0);
            if (s < 0) return false;
            FusedArgs F{};
            range_of(x.a1, x.imm_i, R.cols[x.a0].dtype == QK_I32 ? QK_I32 : QK_I64, F);
            if (R.cols[x.a0].dtype == QK_U8) { if (F.pred_lo < 0) F.pred_lo = 0; }
            out.col = (int8_t)s; out.kind = 0; out.neg = (int8_t)F.pred_neg; out.ilo = F.pred_lo; out.ihi = F.pred_hi;
            return true;
        }
        if (x.op == QK_OP_RANGE_COL_IMM) {
            const int s = slot(x.a0);
            if (s < 0) return false;
            FusedArgs F{};
            range_closed(x.imm_i, (int64_t)x.imm, x.a1 != 0, R.cols[x.a0].dtype == QK_I32 ? QK_I32 : QK_I64, F);
            out.col = (int8_t)s; out.kind = 0; out.neg = (int8_t)F.pred_neg; out.ilo = F.pred_lo; out.ihi = F.pred_hi;
            return true;
        }
        if (x.op == QK_OP_CMP_COL_COL) {
            const int a = slot(x.a0), b = slot(x.a1 >> 8);
            if (a < 0 || b < 0) return false;
            out.col = (int8_t)a; out.col2 = (int8_t)b; out.kind = 3; out.cmp = (int8_t)(x.a1 & 0xff);
            return true;
        }
        if (x.op == QK_OP_IN_SET) {
            const int s = slot(x.a0);
            if (s < 0) return false;
            out.col = (int8_t)s; out.kind = 2; out.nbits = x.a1; out.bits = (unsigned long long)x.imm_i;
            return true;
        }
        if (x.op >= QK_OP_LT && x.op <= QK_OP_NE) {
            int op = x.op, ci = x.l, ki = x.r;
            if (T[ci].op != QK_OP_COL) {                                  // constant <cmp> column: flip
                std::swap(ci, ki);
                op = op == QK_OP_LT ? QK_OP_GT : op == QK_OP_LE ? QK_OP_GE : op == QK_OP_GT ? QK_OP_LT : op == QK_OP_GE ? QK_OP_LE : op;
            }
            if (T[ci].op != QK_OP_COL || T[ki].op != QK_OP_CONST) return false;
            const int s = slot(T[ci].a0);
            if (s < 0) return false;
            const double c = T[ki].imm, inf = __builtin_inf();
            out.col = (int8_t)s; out.kind = 1; out.flo = -inf; out.fhi = inf;
            switch (op) {
                case QK_OP_LT: out.fhi = c; out.hi_open = 1; break;
                case QK_OP_LE: out.fhi = c; break;
                case QK_OP_GT: out.flo = c; out.lo_open = 1; break;
                case QK_OP_GE: out.flo = c; break;
                case QK_OP_EQ: out.flo = out.fhi = c; break;
                default: out.flo = out.fhi = c; out.neg = 1; break;
            }
            // the kernels compare against CLOSED bounds: v > c  <=>  v >= the next double above c (exact for every non-NaN v, and a
            // NaN fails both forms); an open bound at +-infinity admits nothing, which a NaN bound expresses
            if (out.lo_open) { out.flo = out.flo == inf ? __builtin_nan("") : std::nextafter(out.flo, inf); out.lo_open = 0; }
            if (out.hi_open) { out.fhi = out.fhi == -inf ? __builtin_nan("") : std::nextafter(out.fhi, -inf); out.hi_open = 0; }
            return true;                         // NaN: every compare false, NE true -- same as the interpreter
        }
        return false;
    }
    bool conj(const std::vector<ExNode>& T, int i) {
        if (T[i].op == QK_OP_AND) return conj(T, T[i].l) && conj(T, T[i].r);
        if (D.nterms >= DY_MAXTERMS) return false;
        return term(T, i, D.term[D.nterms]) && (++D.nterms, true);
    }
    // f = k0 + k1 * column (or a constant)
    bool affine(const std::vector<ExNode>& T, int i, DyFactor& f) {
        const ExNode& x = T[i];
        if (x.op == QK_OP_COL) { const int s = slot(x.a0); if (s < 0) return false; f = DyFactor{0.0, 1.0, s, 0}; return true; }
        if (x.op == QK_OP_CONST) { f = DyFactor{x.imm, 0.0, -1, 0}; return true; }
        if (x.op == QK_OP_NEG) { if (!affine(T, x.l, f)) return false; f.k0 = -f.k0; f.k1 = -f.k1; return true; }
        if (x.op == QK_OP_ADD || x.op == QK_OP_SUB) {
            DyFactor a, b;
            if (!affine(T, x.l, a) || !affine(T, x.r, b)) return false;
            const double sg = x.op == QK_OP_SUB ? -1.0 : 1.0;
            // exact only when one side is a pure constant and the column's coefficient stays +-1 (k0 + (+-1) * c is ONE rounding,
            // like the interpreter's c + k / k - c); anything else keeps the interpreter
            if (a.col >= 0 && b.col >= 0) return false;
            if (a.col < 0 && b.col < 0) { f = DyFactor{a.k0 + sg * b.k0, 0.0, -1, 0}; return true; }
            if (a.col >= 0) { if (a.k0 != 0.0 || (a.k1 != 1.0 && a.k1 != -1.0)) return false; f = DyFactor{sg * b.k0, a.k1, a.col, 0}; return true; }
            if (b.k0 != 0.0 || (b.k1 != 1.0 && b.k1 != -1.0)) return false;
            f = DyFactor{a.k0, sg * b.k1, b.col, 0};
            return true;
        }
        return false;
    }
    bool product(const std::vector<ExNode>& T, int i, DyAgg& G) {
        if (T[i].op == QK_OP_MUL) return product(T, T[i].l, G) && product(T, T[i].r, G);
        if (G.nfact >= DY_MAXFACT) return false;
        return affine(T, i, G.f[G.nfact]) && (++G.nfact, true);
    }
    bool left_deep(const std::vector<ExNode>& T, int i) {     // a * b * c as ((a * b) * c): the order the accumulator multiplies in
        return T[i].op != QK_OP_MUL || (T[T[i].r].op != QK_OP_MUL && left_deep(T, T[i].l));
    }
    bool aggregate(const std::vector<ExNode>& T, int root, int j) {
        DyAgg& G = D.agg[j];
        G = DyAgg{};
        G.gate = -1;
        int body = root;
        if (T[root].op == QK_OP_SELECT) {                        // CASE WHEN term THEN body ELSE 0
            if (T[T[root].r].op != QK_OP_CONST || T[T[root].r].imm != 0.0 || R.agg_op[j] != QK_AGG_SUM) return false;
            G.gate = DY_MAXTERMS + j;
            if (!term(T, T[root].c, D.term[G.gate])) return false;
            body = T[root].l;
        }
        return left_deep(T, body) && product(T, body, G) && G.nfact >= 1;
    }
};

static bool match_dyn(const Request& R, DyArgs& D, const DenseArgs& A) {
    DyBuilder B(R, D);
    D.nterms = 0;
    if (R.pred && R.pred->n_nodes > 0) {
        std::vector<ExNode> T; int root;
        if (!ex_tree(R.pred, T, &root) || !B.conj(T, root)) return false;
    }
    for (int k = 0; k < R.ngroup_cols; ++k) {
        const int s = B.slot(R.group_cols[k]);
        if (s < 0) return false;
        D.gcol[k] = s;
    }
    for (int j = 0; j < R.nagg; ++j) {
        std::vector<ExNode> T; int root;
        if (!ex_tree(&R.agg_expr[j], T, &root) || !B.aggregate(T, root, j)) return false;
    }
    if (D.ncols == 0) return false;
    for (int j = 0; j < R.nagg; ++j) {                     // product prefix shared with the previous aggregate
        D.agg[j].start = 0;
        if (j == 0 || D.agg[j - 1].nfact >= D.agg[j].nfact) continue;
        bool same = true;
        for (int f = 0; f < D.agg[j - 1].nfact && same; ++f) {
            const DyFactor &a = D.agg[j - 1].f[f], &b = D.agg[j].f[f];
            same = a.col == b.col && a.k0 == b.k0 && a.k1 == b.k1;
        }
        if (same) D.agg[j].start = D.agg[j - 1].nfact;
    }
    return true;
}

// resident CTAs per SM the plan's shared memory allows with NT threads x V rows per tile (0: does not fit at all)
static int dyn_ctas_per_sm(const DyArgs& D, const DenseArgs& A, int NT, int V) {
    int row_bytes = 0;
    for (int c = 0; c < D.ncols; ++c) row_bytes += D.width[c];
    const size_t smem = (size_t)3 * row_bytes * NT * V + (size_t)A.n_groups * (A.nagg * 8 + 4) * NT;
    if (smem > 227 * 1024 - 64) return 0;
    int n = (int)((size_t)(227 * 1024) / (smem + 1024));
    const int by_threads = 2048 / NT;
    if (n > by_threads) n = by_threads;
    return n > 6 ? 6 : n;                                  // <= 888 CTAs: the per-CTA partial states have MAX_PART_BLOCKS slots
}

template <int NT, int V>
static int launch_dyn_v(DyArgs& D, const DenseArgs& A, int64_t nrows, double* part_acc, long long* part_cnt, int* nblocks_out, cudaStream_t st) {
    constexpr int STAGES = 3, TILE = NT * V;
    int off = 0;
    for (int w : {8, 4, 1})                                              // widest first: every sub-array stays 16-byte aligned
        for (int c = 0; c < D.ncols; ++c) if (D.width[c] == w) { D.off[c] = off; off += w * TILE; }
    D.stage_bytes = off;
    for (DyTerm& T : D.term) { T.soff = D.off[T.col]; T.soff2 = D.off[T.col2]; T.w = D.width[T.col]; }
    for (int k = 0; k < A.ngroup_cols; ++k) { D.goff[k] = D.off[D.gcol[k]]; D.gw[k] = D.width[D.gcol[k]]; }
    for (int j = 0; j < A.nagg; ++j)
        for (int f = 0; f < D.agg[j].nfact; ++f) if (D.agg[j].f[f].col >= 0) D.agg[j].f[f].soff = D.off[D.agg[j].f[f].col];
    const size_t smem = (size_t)STAGES * off + (size_t)A.n_groups * (A.nagg * 8 + 4) * NT;
    if (smem > 227 * 1024 - 64) return 1;
    bool fast = true;                                                    // typed loads when every access has the common type
    auto term_ok = [&](const DyTerm& T) {
        const int dt = D.dtype[T.col];
        if (T.kind == 3) return (dt == QK_I32 || dt == QK_I64) && D.dtype[T.col2] == dt;
        return T.kind == 0 ? (dt == QK_I32 || dt == QK_I64) : T.kind == 1 ? dt == QK_F64 : dt == QK_U8;
    };
    for (int k = 0; k < D.nterms && fast; ++k) fast = term_ok(D.term[k]);
    for (int j = 0; j < A.nagg && fast; ++j) if (D.agg[j].gate >= 0) fast = term_ok(D.term[D.agg[j].gate]);
    for (int k = 0; k < A.ngroup_cols && fast; ++k) fast = D.dtype[D.gcol[k]] == QK_U8 || D.dtype[D.gcol[k]] == QK_I32;
    for (int j = 0; j < A.nagg && fast; ++j)
        for (int f = 0; f < D.agg[j].nfact && fast; ++f) if (D.agg[j].f[f].col >= 0) fast = D.dtype[D.agg[j].f[f].col] == QK_F64;
    // persistent grid: as many CTAs per SM as the plan's shared memory allows -- with one CTA per SM the kernel is bound by
    // shared-memory latency (few warps active)
    const int sms = sm_count(), per_sm = dyn_ctas_per_sm(D, A, NT, V);
    const int64_t nfull = nrows / TILE, want = (int64_t)sms * (per_sm > 0 ? per_sm : 1);
    const int nb = (int)(nfull < want ? (nfull > 0 ? nfull : 1) : want);
    if (fast) {
        auto kern = k_dense_agg_dyn_tma<NT, V, STAGES, true>;
        QK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        kern<<<nb, NT, smem, st>>>(D, A, nrows, part_acc, part_cnt);
    } else {
        auto kern = k_dense_agg_dyn_tma<NT, V, STAGES, false>;
        QK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        kern<<<nb, NT, smem, st>>>(D, A, nrows, part_acc, part_cnt);
    }
    QK_LAUNCH_CHECK("k_dense_agg_dyn_tma");
    *nblocks_out = nb;
    g_variant = "fused_tma:dyn";
    g_variant_cfg = std::string("nt") + std::to_string(NT) + "v" + std::to_string(V) + "s3c" + std::to_string(D.ncols) + (fast ? "t" : "") + "x" + std::to_string(per_sm);
    return 0;
}
static int launch_dyn(DyArgs& D, const DenseArgs& A, int64_t nrows, double* part_acc, long long* part_cnt, int* nblocks_out, cudaStream_t st) {
    // (threads, rows per thread) shapes in order of preference; the first whose tile ring + partial states leave at least two
    // CTAs per SM wins, else the one with the most rows in flight.  QK_DYN_SHAPE=<threads>x<rows> pins one (profiling).
    static const int shapes[][2] = {{128, 4}, {256, 4}, {256, 2}, {128, 8}, {128, 2}, {128, 1}};   // measured order on Q6 / Q1 (SF-100)
    int pick = -1, best_rows = 0;
    if (const char* e = getenv("QK_DYN_SHAPE")) {
        int nt = 0, v = 0;
        if (sscanf(e, "%dx%d", &nt, &v) == 2)
            for (int i = 0; i < 6; ++i) if (shapes[i][0] == nt && shapes[i][1] == v && dyn_ctas_per_sm(D, A, nt, v) > 0) pick = i;
    }
    if (pick < 0) {
        for (int i = 0; i < 6 && pick < 0; ++i) if (dyn_ctas_per_sm(D, A, shapes[i][0], shapes[i][1]) >= 2) pick = i;
    }
    if (pick < 0)
        for (int i = 0; i < 6; ++i) {
            const int rows = dyn_ctas_per_sm(D, A, shapes[i][0], shapes[i][1]) * shapes[i][0] * shapes[i][1];
            if (rows > best_rows) { best_rows = rows; pick = i; }
        }
    switch (pick) {
        case 0: return launch_dyn_v<128, 4>(D, A, nrows, part_acc, part_cnt, nblocks_out, st);
        case 1: return launch_dyn_v<256, 4>(D, A, nrows, part_acc, part_cnt, nblocks_out, st);
        case 2: return launch_dyn_v<256, 2>(D, A, nrows, part_acc, part_cnt, nblocks_out, st);
        case 3: return launch_dyn_v<128, 8>(D, A, nrows, part_acc, part_cnt, nblocks_out, st);
        case 4: return launch_dyn_v<128, 2>(D, A, nrows, part_acc, part_cnt, nblocks_out, st);
        case 5: return launch_dyn_v<128, 1>(D, A, nrows, part_acc, part_cnt, nblocks_out, st);
        default: return 1;                                 // no shape fits: the caller falls back to the interpreter
    }
}

constexpr int MAX_PART_BLOCKS = 1024;

}  // namespace
}  // namespace qk

using namespace qk;

namespace qk {
// compact.cu: TMA-staged filter + column compaction; returns 1 when the request does not fit the fast path
int try_filter_compact_tma(const qk_column* cols, int ncols, int64_t nrows, const qk_expr* pred, const qk_expr* proj, int nproj,
                           qk_column* out, int64_t* out_rows, void* workspace, size_t ws_bytes, const qk_bloom* bloom, cudaStream_t st);
int bloom_build(const qk_column* key, unsigned* bits, long long words_per_part, int nparts, cudaStream_t st);
}

extern "C" const char* qk_last_variant(void) { return g_variant.c_str(); }
extern "C" const char* qk_last_variant_config(void) { return g_variant_cfg.c_str(); }

extern "C" size_t qk_scan_workspace_bytes(int64_t nrows) {
    const int64_t nchunks = (nrows + STABLE_CHUNK - 1) / STABLE_CHUNK + 1;
    const size_t generic = align_up((size_t)nchunks * 4, 256) + align_up((size_t)nchunks * 8, 256);
    // chunk counts + offsets + the 1-bit-per-row survivor bitmap of the TMA compaction path
    const size_t compact = (size_t)(2 * 1024 + 8) * 8 + align_up((size_t)((nrows + 31) / 32 + 8) * 4, 256);
    return generic > compact ? generic : compact;
}

extern "C" int qk_bloom_build(const qk_column* key, uint32_t* bits, int64_t words_per_part, int32_t nparts, void* stream) {
    const char* who = "qk_bloom_build";
    if (int rc = check_col(key, who)) return rc;
    if (!dtype_is_int(key->dtype)) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: keys must be integer columns", who);
    if (!bits || words_per_part < 8 || (words_per_part & 7) || nparts < 1) QK_FAIL(QK_ERR_INVALID, "%s: bad filter geometry", who);
    return bloom_build(key, bits, words_per_part, nparts, (cudaStream_t)stream);
}

static int scan_filter_project_impl(const qk_column* cols, int32_t ncols, int64_t nrows, const qk_expr* pred,
                                    const qk_expr* proj, int32_t nproj, qk_column* out, int64_t* out_rows,
                                    int32_t stable, void* workspace, size_t ws_bytes, const qk_bloom* bloom, void* stream);

extern "C" int qk_scan_filter_project(const qk_column* cols, int32_t ncols, int64_t nrows, const qk_expr* pred,
                                      const qk_expr* proj, int32_t nproj, qk_column* out, int64_t* out_rows,
                                      int32_t stable, void* workspace, size_t ws_bytes, void* stream) {
    return scan_filter_project_impl(cols, ncols, nrows, pred, proj, nproj, out, out_rows, stable, workspace, ws_bytes, nullptr, stream);
}

extern "C" int qk_scan_filter_project_sj(const qk_column* cols, int32_t ncols, int64_t nrows, const qk_expr* pred,
                                         const qk_expr* proj, int32_t nproj, qk_column* out, int64_t* out_rows,
                                         const qk_bloom* bloom, void* workspace, size_t ws_bytes, void* stream) {
    if (!bloom || !bloom->bits) QK_FAIL(QK_ERR_INVALID, "qk_scan_filter_project_sj: null Bloom descriptor");
    return scan_filter_project_impl(cols, ncols, nrows, pred, proj, nproj, out, out_rows, 0, workspace, ws_bytes, bloom, stream);
}

static int scan_filter_project_impl(const qk_column* cols, int32_t ncols, int64_t nrows, const qk_expr* pred,
                                    const qk_expr* proj, int32_t nproj, qk_column* out, int64_t* out_rows,
                                    int32_t stable, void* workspace, size_t ws_bytes, const qk_bloom* bloom, void* stream) {
    static thread_local Programs P;
    if (!out_rows) QK_FAIL(QK_ERR_INVALID, "qk_scan_filter_project: out_rows is null");
    if (nproj < 0 || (nproj > 0 && (!proj || !out))) QK_FAIL(QK_ERR_INVALID, "qk_scan_filter_project: bad projection arguments");
    if (int rc = pack_programs(P, cols, ncols, nrows, pred, proj, nproj, "qk_scan_filter_project")) return rc;
    ProjOut O;
    for (int j = 0; j < nproj; ++j) {
        const bool pass = proj[j].n_nodes == 1 && proj[j].nodes[0].op == QK_OP_COL;
        O.pass_col[j] = pass ? (int8_t)proj[j].nodes[0].a0 : (int8_t)-1;
        const int want = pass ? cols[proj[j].nodes[0].a0].dtype : QK_F64;
        if (out[j].dtype != want) QK_FAIL(QK_ERR_INVALID, "qk_scan_filter_project: output %d must have dtype %d", j, want);
        if (out[j].length < nrows) QK_FAIL(QK_ERR_CAPACITY, "qk_scan_filter_project: output %d holds %lld rows, needs %lld", j, (long long)out[j].length, (long long)nrows);
        if (nrows > 0 && !out[j].data) QK_FAIL(QK_ERR_INVALID, "qk_scan_filter_project: output %d has no data", j);
        O.out[j] = (void*)out[j].data;
    }
    cudaStream_t st = (cudaStream_t)stream;
    QK_CUDA(cudaMemsetAsync(out_rows, 0, sizeof(int64_t), st));
    if (nrows == 0) return QK_OK;
    const int sms = sm_count();
    {
        // fast path (stable by construction): integer-range predicate + verbatim columns
        const int rc = try_filter_compact_tma(cols, ncols, nrows, pred, proj, nproj, out, out_rows, workspace, ws_bytes, bloom, st);
        if (rc == 0) { g_variant = bloom ? "compact_tma+bloom" : "compact_tma"; g_variant_cfg = "nt256s3"; }
        if (rc <= 0) return rc;                          // 0 = done by the fast path, < 0 = error
        if (bloom) QK_FAIL(QK_ERR_UNSUPPORTED, "qk_scan_filter_project_sj: needs an integer-range predicate and verbatim columns");
        g_variant = "filter_interpreter"; g_variant_cfg = "nt256";
    }
    if (!stable) {
        int64_t nb = (nrows + 255) / 256;
        if (nb > (int64_t)sms * 8) nb = (int64_t)sms * 8;
        k_filter_project_unordered<<<(unsigned)nb, 256, 0, st>>>(P, O, nproj, nrows, (unsigned long long*)out_rows);
        QK_LAUNCH_CHECK("k_filter_project_unordered");
        return QK_OK;
    }
    const int64_t nchunks = (nrows + STABLE_CHUNK - 1) / STABLE_CHUNK;
    if (ws_bytes < qk_scan_workspace_bytes(nrows) || !workspace) QK_FAIL(QK_ERR_CAPACITY, "qk_scan_filter_project: workspace too small (%zu < %zu)", ws_bytes, qk_scan_workspace_bytes(nrows));
    int32_t* counts = (int32_t*)workspace;
    int64_t* offsets = (int64_t*)((char*)workspace + align_up((size_t)(nchunks + 1) * 4, 256));
    int64_t nb = nchunks < (int64_t)sms * 8 ? nchunks : (int64_t)sms * 8;
    k_filter_count<<<(unsigned)nb, 256, 0, st>>>(P, nrows, counts);
    QK_LAUNCH_CHECK("k_filter_count");
    k_scan_counts<<<1, 1024, 0, st>>>(counts, nchunks, offsets, out_rows);
    QK_LAUNCH_CHECK("k_scan_counts");
    k_filter_project_stable<<<(unsigned)nb, 256, 0, st>>>(P, O, nproj, nrows, offsets);
    QK_LAUNCH_CHECK("k_filter_project_stable");
    return QK_OK;
}

extern "C" size_t qk_scan_agg_workspace_bytes(int32_t n_groups, int32_t nagg) {
    if (n_groups <= 0 || nagg < 0) return 0;
    return align_up((size_t)MAX_PART_BLOCKS * n_groups * (nagg > 0 ? nagg : 1) * 8, 256) + align_up((size_t)MAX_PART_BLOCKS * n_groups * 8, 256);
}

extern "C" int qk_scan_filter_agg_dense(const qk_column* cols, int32_t ncols, int64_t nrows, const qk_expr* pred,
                                        const int32_t* group_cols, const int32_t* group_card, int32_t ngroup_cols,
                                        const qk_expr* agg_expr, const int32_t* agg_op, int32_t nagg,
                                        double* acc, int64_t* cnt, void* workspace, size_t ws_bytes,
                                        int32_t variant, void* stream) {
    static thread_local Programs P;
    const char* who = "qk_scan_filter_agg_dense";
    if (ngroup_cols < 0 || ngroup_cols > 4 || nagg < 0 || nagg > QK_MAX_AGGS) QK_FAIL(QK_ERR_INVALID, "%s: ngroup_cols / nagg out of range", who);
    if (!cnt || (nagg > 0 && (!acc || !agg_expr || !agg_op))) QK_FAIL(QK_ERR_INVALID, "%s: null output / aggregate arguments", who);
    if (int rc = pack_programs(P, cols, ncols, nrows, pred, agg_expr, nagg, who)) return rc;
    DenseArgs A{};
    int64_t ng = 1;
    for (int k = 0; k < ngroup_cols; ++k) {
        if (group_cols[k] < 0 || group_cols[k] >= ncols || !dtype_is_int(cols[group_cols[k]].dtype)) QK_FAIL(QK_ERR_INVALID, "%s: group column %d must be an integer code column", who, k);
        if (group_card[k] <= 0) QK_FAIL(QK_ERR_INVALID, "%s: group cardinality must be positive", who);
        ng *= group_card[k];
        if (ng > 4096) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: more than 4096 dense groups; use the hash aggregate", who);
    }
    int stride = 1;
    for (int k = ngroup_cols - 1; k >= 0; --k) { A.group_col[k] = group_cols[k]; A.group_stride[k] = stride; stride *= group_card[k]; }
    A.ngroup_cols = ngroup_cols; A.n_groups = (int)ng; A.nagg = nagg;
    for (int j = 0; j < nagg; ++j) {
        if (agg_op[j] < QK_AGG_SUM || agg_op[j] > QK_AGG_MAX) QK_FAIL(QK_ERR_INVALID, "%s: bad aggregate op %d", who, agg_op[j]);
        A.agg_op[j] = agg_op[j];
    }
    if (nrows == 0) return QK_OK;
    if (!workspace || ws_bytes < qk_scan_agg_workspace_bytes((int)ng, nagg)) QK_FAIL(QK_ERR_CAPACITY, "%s: workspace too small", who);
    double* part_acc = (double*)workspace;
    long long* part_cnt = (long long*)((char*)workspace + align_up((size_t)MAX_PART_BLOCKS * ng * (nagg > 0 ? nagg : 1) * 8, 256));
    cudaStream_t st = (cudaStream_t)stream;
    int nblocks = 0;
    bool done = false;
    if (variant != 1) {
        Request R{cols, ncols, nrows, pred, group_cols, group_card, ngroup_cols, agg_expr, agg_op, nagg};
        FusedArgs F{};
        // auto: TMA-staged fused kernel first (measured faster), then the LDG one, then the interpreter
        const int order[2] = {variant == 0 ? 3 : variant, variant == 0 ? 2 : -1};
        int rc = 1;
        for (int a = 0; a < 2 && rc == 1 && order[a] > 0 && variant != 7; ++a) {
            const int v = order[a];
            if (match_plan<PlanQ1>(R, F)) rc = launch_fused<PlanQ1>(F, A, nrows, v, part_acc, part_cnt, &nblocks, st, "q1");
            else if (match_plan<PlanRev1>(R, F)) rc = launch_fused<PlanRev1>(F, A, nrows, v, part_acc, part_cnt, &nblocks, st, "rev1");
            else if (match_plan<PlanMul1>(R, F)) rc = launch_fused<PlanMul1>(F, A, nrows, v, part_acc, part_cnt, &nblocks, st, "mul1");
            else break;
        }
        if (rc < 0) return rc;
        done = rc == 0;
        if (!done && (variant == 0 || variant == 3 || variant == 7)) {
            // no typed plan: the runtime-described plan over the same TMA tile ring (any aggregate of the grammar above)
            static thread_local DyArgs D;
            if (match_dyn(R, D, A)) {
                rc = launch_dyn(D, A, nrows, part_acc, part_cnt, &nblocks, st);
                if (rc < 0) return rc;
                done = rc == 0;
            }
        }
        if (!done && variant != 0) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: no fused plan matches this request (variant %d forced)", who, variant);
    }
    if (!done) {
        const size_t smem = (size_t)ng * (nagg * 8 + 4) * GEN_NT;
        if (smem > 200 * 1024) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: %lld groups x %d aggregates exceed the shared-memory dense path; use the hash aggregate", who, (long long)ng, nagg);
        QK_CUDA(cudaFuncSetAttribute(k_dense_agg_generic, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        const int sms = sm_count();
        int per_sm = (int)((220 * 1024) / (smem + 1024));
        if (per_sm < 1) per_sm = 1;
        if (per_sm > 4) per_sm = 4;
        int64_t nb = (nrows + GEN_NT - 1) / GEN_NT;
        if (nb > (int64_t)sms * per_sm) nb = (int64_t)sms * per_sm;
        nblocks = (int)nb;
        k_dense_agg_generic<<<nblocks, GEN_NT, smem, st>>>(P, A, nrows, part_acc, part_cnt);
        QK_LAUNCH_CHECK("k_dense_agg_generic");
        g_variant = "generic"; g_variant_cfg = "nt256";
    }
    if (nblocks > MAX_PART_BLOCKS) QK_FAIL(QK_ERR_INVALID, "%s: internal: %d partial blocks", who, nblocks);
    if (nagg > 0) {
        k_dense_finalize<<<(A.n_groups * A.nagg + 127) / 128, 128, 0, st>>>(part_acc, part_cnt, nblocks, A, acc, (long long*)cnt);
        QK_LAUNCH_CHECK("k_dense_finalize");
    }
    k_dense_finalize_cnt<<<(A.n_groups + 127) / 128, 128, 0, st>>>(part_cnt, nblocks, A.n_groups, (long long*)cnt);
    QK_LAUNCH_CHECK("k_dense_finalize_cnt");
    return QK_OK;
}
