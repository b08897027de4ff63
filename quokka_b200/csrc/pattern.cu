// pattern.cu -- complex event recognition over a key-segmented, time-sorted stream: the search behind
// OrderedStream.pattern_recognize (pyquokka/orderedstream.py:37-53; the reference's CEPExecutor, executors/cep_executors.py:86-178,
// runs a per-batch DuckDB range join and a Python DFS).  The rows arrive segmented by key with the stable partition of
// partition.cu, so time order survives inside a segment.  The row-local conjuncts of every event were evaluated before by the
// scan kernel into a candidate mask (bit e of cand[r]: row r may bind event e); what is left here is the data-dependent part:
//   one warp per start row, starts handed out by an atomic counter to a persistent grid (the work per start is very uneven);
//   at level i the 32 lanes test 32 consecutive rows of the segment -- cand bit, t > t(i-1), t <= t0 + maxspan, the link
//   program of event i over the bound rows -- and a ballot picks the first passing row; a ballot on "past the span" ends the level;
//   backtracking resumes the level above after its bound row, except that a level no later link program reads is ended as
//   well (its later rows can only have fewer completions), which keeps row-local-only patterns at O(rows in the span) per start;
//   after the first complete match B the search goes on, accepting at level i only t <= B_i while the levels above equal B, and
//   keeps the lexicographically smallest time vector.
// Link programs are interpreted in fp64 (the library is built with -fmad=false), with the lane's stack and the values of the
// bound rows in shared memory, so the kernel has no local-memory stack.
#include "common.cuh"

#include <limits.h>

namespace qk {
namespace {

constexpr int PT_NT = 128;                       // 4 warps per CTA; >= 8 CTAs per SM lets ptxas use 64 registers (54, no spills)
constexpr int PT_WARPS = PT_NT / 32;
constexpr int PM = QK_PATTERN_MAX_EVENTS;
constexpr int PT_MAX_NODES = 128;                // all link programs of one call together

struct LNode { int16_t op; int8_t a0; int8_t a1; int32_t pad; double imm; };     // a0 = link column, a1 = event whose row is read
struct LCol { const void* p; const uint8_t* valid; int32_t dt; int32_t pad; };

struct PatArgs {
    LCol cols[QK_MAX_COLS];
    LNode nodes[PT_MAX_NODES];
    int16_t off[PM + 1];                         // program of event e = nodes[off[e], off[e + 1])
    int32_t m, nlink;
    uint32_t read;                               // bit i: a link program of a later event reads event i's row
    uint32_t indep;                              // bit i: ending a binding at level i ends level i (no later program reads it)
    const long long* time;
    const int32_t* by;
    const int64_t* seg;
    const uint8_t* cand;
    const int32_t* starts;
    int64_t n_starts, n;
    int32_t n_by;
    long long maxspan, budget;
    int32_t* out;
    unsigned long long* status;                  // [0] starts over budget, [1] n_starts - smallest such index, [2] work counter
    unsigned long long* tested;
};

struct WarpState {
    double val[PM][QK_MAX_COLS];                 // link columns of every bound row (staged once per binding)
    double stk[QK_MAX_STACK][32];                // the lanes' interpreter stacks
    long long tb[PM];                            // times of the bound rows
    long long best[PM];                          // times of the best complete match
    int32_t row[PM];                             // bound rows
    int32_t pos[PM];                             // next row to test, per level
    int32_t brow[PM];                            // rows of the best complete match
    uint32_t vmask[PM];                          // bit c: val[e][c] is not NULL
    unsigned long long tested;                   // rows tested by the warp over all its starts
};

__device__ __forceinline__ bool eval_link(const PatArgs& A, WarpState& S, int ev, int64_t r, int lane) {
    int sp = 0;
    const int end = A.off[ev + 1];
    for (int pc = A.off[ev]; pc < end; ++pc) {
        const LNode& nd = A.nodes[pc];
        switch (nd.op) {
            case QK_OP_COL: {
                double v;
                if (nd.a1 == ev) {
                    const LCol* c = &A.cols[nd.a0];
                    if (c->valid && !c->valid[r]) return false;          // a predicate that reads a NULL is false
                    v = load_f64(c->p, c->dt, r);
                } else {
                    if (!((S.vmask[nd.a1] >> nd.a0) & 1u)) return false;
                    v = S.val[nd.a1][nd.a0];
                }
                S.stk[sp++][lane] = v;
            } break;
            case QK_OP_CONST: S.stk[sp++][lane] = nd.imm; break;
            case QK_OP_NEG: S.stk[sp - 1][lane] = -S.stk[sp - 1][lane]; break;
            case QK_OP_NOT: S.stk[sp - 1][lane] = S.stk[sp - 1][lane] == 0.0 ? 1.0 : 0.0; break;
            case QK_OP_SELECT: {
                sp -= 2;
                const double c = S.stk[sp - 1][lane];
                S.stk[sp - 1][lane] = c != 0.0 ? S.stk[sp][lane] : S.stk[sp + 1][lane];
            } break;
            default: {
                const double b = S.stk[--sp][lane], a = S.stk[sp - 1][lane];
                double v;
                switch (nd.op) {
                    case QK_OP_ADD: v = a + b; break;
                    case QK_OP_SUB: v = a - b; break;
                    case QK_OP_MUL: v = a * b; break;
                    case QK_OP_DIV: v = a / b; break;
                    case QK_OP_LT: v = a < b ? 1.0 : 0.0; break;
                    case QK_OP_LE: v = a <= b ? 1.0 : 0.0; break;
                    case QK_OP_GT: v = a > b ? 1.0 : 0.0; break;
                    case QK_OP_GE: v = a >= b ? 1.0 : 0.0; break;
                    case QK_OP_EQ: v = a == b ? 1.0 : 0.0; break;
                    case QK_OP_NE: v = a != b ? 1.0 : 0.0; break;
                    case QK_OP_AND: v = (a != 0.0 && b != 0.0) ? 1.0 : 0.0; break;
                    default: v = (a != 0.0 || b != 0.0) ? 1.0 : 0.0; break;       // QK_OP_OR
                }
                S.stk[sp - 1][lane] = v;
            }
        }
    }
    return sp == 0 || S.stk[0][lane] != 0.0;
}

// the link columns of row r, bound to event e, into the warp's slab
__device__ __forceinline__ void stage(const PatArgs& A, WarpState& S, int e, int64_t r, int lane) {
    bool ok = true;
    if (lane < A.nlink) {
        const LCol* c = &A.cols[lane];
        ok = !c->valid || c->valid[r];
        S.val[e][lane] = ok ? load_f64(c->p, c->dt, r) : 0.0;
    }
    const unsigned vm = __ballot_sync(0xffffffffu, ok);
    if (lane == 0) S.vmask[e] = vm;
    __syncwarp();
}

__global__ void __launch_bounds__(PT_NT, 8) k_pattern_search(const __grid_constant__ PatArgs A) {
    __shared__ WarpState ws[PT_WARPS];
    const int lane = (int)lane_id();
    WarpState& S = ws[threadIdx.x >> 5];
    const int m = A.m;
    const unsigned all_levels = (1u << m) - 1u;
    if (lane == 0) S.tested = 0;
    for (;;) {
        long long si = 0;
        if (lane == 0) si = (long long)atomicAdd(&A.status[2], 1ull);
        si = __shfl_sync(0xffffffffu, si, 0);
        if (si >= A.n_starts) break;
        const int64_t s = A.starts[si];
        const int b = (s >= 0 && s < A.n) ? A.by[s] : -1;
        // a start outside its key's segment, or a segment past the columns, is a caller's error: no match, nothing read
        const bool inside = b >= 0 && b < A.n_by && A.seg[b] <= s && s < A.seg[b + 1] && A.seg[b + 1] <= A.n;
        if (!inside || !(A.cand[s] & 1u)) {
            if (lane < m) A.out[si * m + lane] = -1;
            continue;
        }
        const int64_t end = A.seg[b + 1];
        const long long t0 = A.time[s];
        const long long lim = t0 > LLONG_MAX - A.maxspan ? LLONG_MAX : t0 + A.maxspan;
        if (lane == 0) { S.row[0] = (int32_t)s; S.tb[0] = t0; S.pos[1] = (int32_t)(s + 1); }
        __syncwarp();
        if (A.read & 1u) stage(A, S, 0, s, lane);
        bool have = false;
        unsigned tight = all_levels;            // bit i: levels 1 .. i-1 equal the best match, so level i is capped by it
        long long tested = 0;
        int level = 1;
        while (level >= 1) {
            int64_t p = S.pos[level];
            const long long tprev = S.tb[level - 1];
            const long long cap = (have && ((tight >> level) & 1u)) ? min(lim, S.best[level]) : lim;
            int64_t found = -1;
            for (;;) {
                const int64_t r = p + lane;
                const bool in = r < end;
                const long long t = in ? A.time[r] : 0;
                const bool past = !in || t > cap;                      // monotone in r: time is sorted inside a segment
                const bool pass = !past && ((A.cand[r] >> level) & 1u) && t > tprev && eval_link(A, S, level, r, lane);
                const unsigned pm = __ballot_sync(0xffffffffu, past), om = __ballot_sync(0xffffffffu, pass);
                if (om) {
                    const int fl = __ffs(om) - 1;
                    found = p + fl;
                    tested += fl + 1;
                    break;
                }
                tested += pm ? __ffs(pm) - 1 : 32;
                if (pm || tested > A.budget) break;
                p += 32;
            }
            if (tested > A.budget) break;
            if (found >= 0) {
                if (lane == 0) { S.row[level] = (int32_t)found; S.pos[level] = (int32_t)(found + 1); S.tb[level] = A.time[found]; }
                __syncwarp();
                if (level < m - 1) {
                    if ((A.read >> level) & 1u) stage(A, S, level, found, lane);
                    const bool eq = have && S.tb[level] == S.best[level];
                    tight = ((tight >> level) & 1u) && eq ? tight | (1u << (level + 1)) : tight & ~(1u << (level + 1));
                    if (lane == 0) S.pos[level + 1] = (int32_t)(found + 1);
                    __syncwarp();
                    ++level;
                    continue;
                }
                // a complete match; the caps make it <= the best one, so it becomes the best
                if (lane < m) { S.best[lane] = S.tb[lane]; S.brow[lane] = S.row[lane]; }
                __syncwarp();
                have = true;
                tight = all_levels;
            }
            // level exhausted (or done after its first completion, at the last level): back to the level above, which ends
            // too when no later link program reads its row
            do { --level; } while (level >= 1 && ((A.indep >> level) & 1u));
        }
        if (lane == 0) S.tested += (unsigned long long)tested;
        const bool over = tested > A.budget;
        if (over && lane == 0) {
            atomicAdd(&A.status[0], 1ull);
            atomicMax(&A.status[1], (unsigned long long)(A.n_starts - si));
        }
        if (lane < m) A.out[si * m + lane] = (have && !over) ? S.brow[lane] : -1;
        __syncwarp();
    }
    if (A.tested && lane == 0 && S.tested) atomicAdd(A.tested, S.tested);
}

int check_link_col(const qk_column* c, int64_t n, const char* who, int k) {
    if (!c) QK_FAIL(QK_ERR_INVALID, "%s: null link column %d", who, k);
    if (c->lanes > 1 || c->dtype == QK_F16 || dtype_size(c->dtype) == 0)
        QK_FAIL(QK_ERR_UNSUPPORTED, "%s: link column %d must be a scalar u8 / i32 / i64 / f32 / f64 column", who, k);
    if (c->length != n) QK_FAIL(QK_ERR_INVALID, "%s: link column %d has %lld rows, expected %lld", who, k, (long long)c->length, (long long)n);
    if (n > 0 && !c->data) QK_FAIL(QK_ERR_INVALID, "%s: link column %d has null data", who, k);
    return 0;
}

}  // namespace
}  // namespace qk

using namespace qk;

extern "C" int qk_pattern_search(const qk_column* time, const qk_column* by, const int64_t* seg, int32_t n_by, const uint8_t* cand,
                                 const int32_t* starts, int64_t n_starts, int32_t m, int64_t maxspan, const qk_column* link_cols,
                                 int32_t nlink, const qk_expr* links, int64_t budget, int32_t* out_bound, uint64_t* status,
                                 uint64_t* rows_tested, void* stream) {
    const char* who = "qk_pattern_search";
    if (int rc = check_col(time, who)) return rc;
    if (int rc = check_col(by, who)) return rc;
    if (time->dtype != QK_I64 || by->dtype != QK_I32) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: time must be int64 and the key int32 codes", who);
    const int64_t n = time->length;
    if (by->length != n) QK_FAIL(QK_ERR_INVALID, "%s: time / key length mismatch", who);
    if (m < 2 || m > QK_PATTERN_MAX_EVENTS) QK_FAIL(QK_ERR_INVALID, "%s: %d events; a pattern has 2 to %d", who, m, QK_PATTERN_MAX_EVENTS);
    if (maxspan < 0) QK_FAIL(QK_ERR_INVALID, "%s: negative maxspan", who);
    if (budget < 1) QK_FAIL(QK_ERR_INVALID, "%s: the step budget must be >= 1", who);
    if (n_starts < 0 || n_starts > 0x7fffffffLL) QK_FAIL(QK_ERR_INVALID, "%s: n_starts %lld out of range", who, (long long)n_starts);
    if (!seg || n_by < 1) QK_FAIL(QK_ERR_INVALID, "%s: bad segments", who);
    if (!status) QK_FAIL(QK_ERR_INVALID, "%s: null status", who);
    if (n > 0 && !cand) QK_FAIL(QK_ERR_INVALID, "%s: null candidate mask", who);
    if (n_starts > 0 && (!starts || !out_bound)) QK_FAIL(QK_ERR_INVALID, "%s: null starts / output", who);
    if (nlink < 0 || nlink > QK_MAX_COLS) QK_FAIL(QK_ERR_INVALID, "%s: %d link columns; at most %d", who, nlink, QK_MAX_COLS);
    if (nlink > 0 && !link_cols) QK_FAIL(QK_ERR_INVALID, "%s: null link columns", who);
    if (!links) QK_FAIL(QK_ERR_INVALID, "%s: null link programs", who);
    PatArgs A{};
    for (int c = 0; c < nlink; ++c) {
        if (int rc = check_link_col(&link_cols[c], n, who, c)) return rc;
        A.cols[c] = LCol{link_cols[c].data, link_cols[c].validity, link_cols[c].dtype, 0};
    }
    int total = 0;
    uint32_t read = 0;
    for (int e = 0; e < m; ++e) {
        const qk_expr& x = links[e];
        A.off[e] = (int16_t)total;
        if (x.n_nodes < 0 || x.n_nodes > QK_MAX_EXPR_NODES) QK_FAIL(QK_ERR_INVALID, "%s: link program %d has %d nodes", who, e, x.n_nodes);
        if (x.n_nodes > 0 && !x.nodes) QK_FAIL(QK_ERR_INVALID, "%s: link program %d has null nodes", who, e);
        if (e == 0 && x.n_nodes != 0) QK_FAIL(QK_ERR_INVALID, "%s: event 0 has no link program (its predicate is row-local)", who);
        if (total + x.n_nodes > PT_MAX_NODES) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: link programs exceed %d nodes in total", who, PT_MAX_NODES);
        int depth = 0;
        for (int i = 0; i < x.n_nodes; ++i) {
            const qk_expr_node& s = x.nodes[i];
            LNode d{};
            d.op = (int16_t)s.op; d.imm = s.imm;
            switch (s.op) {
                case QK_OP_COL:
                    if (s.a0 < 0 || s.a0 >= nlink) QK_FAIL(QK_ERR_INVALID, "%s: link program %d reads column slot %d of %d", who, e, s.a0, nlink);
                    if (s.a1 < 0 || s.a1 > e) QK_FAIL(QK_ERR_INVALID, "%s: link program %d reads event %d (only events 0 .. %d)", who, e, s.a1, e);
                    d.a0 = (int8_t)s.a0; d.a1 = (int8_t)s.a1;
                    if (s.a1 < e) read |= 1u << s.a1;
                    depth++; break;
                case QK_OP_CONST: depth++; break;
                case QK_OP_ADD: case QK_OP_SUB: case QK_OP_MUL: case QK_OP_DIV: case QK_OP_LT: case QK_OP_LE:
                case QK_OP_GT: case QK_OP_GE: case QK_OP_EQ: case QK_OP_NE: case QK_OP_AND: case QK_OP_OR:
                    if (depth < 2) QK_FAIL(QK_ERR_INVALID, "%s: stack underflow in link program %d", who, e);
                    depth--; break;
                case QK_OP_NEG: case QK_OP_NOT:
                    if (depth < 1) QK_FAIL(QK_ERR_INVALID, "%s: stack underflow in link program %d", who, e);
                    break;
                case QK_OP_SELECT:
                    if (depth < 3) QK_FAIL(QK_ERR_INVALID, "%s: stack underflow in link program %d", who, e);
                    depth -= 2; break;
                default: QK_FAIL(QK_ERR_UNSUPPORTED, "%s: op %d is not supported in link programs", who, s.op);
            }
            if (depth > QK_MAX_STACK) QK_FAIL(QK_ERR_UNSUPPORTED, "%s: link program %d needs more than %d stack slots", who, e, QK_MAX_STACK);
            A.nodes[total++] = d;
        }
        if (x.n_nodes > 0 && depth != 1) QK_FAIL(QK_ERR_INVALID, "%s: link program %d leaves %d values on the stack", who, e, depth);
    }
    A.off[m] = (int16_t)total;
    A.m = m; A.nlink = nlink; A.read = read;
    A.indep = (~read | (1u << (m - 1))) & ((1u << m) - 1u);
    A.time = (const long long*)time->data; A.by = (const int32_t*)by->data; A.seg = seg; A.cand = cand; A.starts = starts;
    A.n_starts = n_starts; A.n = n; A.n_by = n_by; A.maxspan = maxspan; A.budget = budget;
    A.out = out_bound; A.status = (unsigned long long*)status; A.tested = (unsigned long long*)rows_tested;
    cudaStream_t st = (cudaStream_t)stream;
    QK_CUDA(cudaMemsetAsync(status, 0, QK_PATTERN_STATUS_WORDS * sizeof(uint64_t), st));
    if (n_starts == 0) return QK_OK;
    int per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_pattern_search, PT_NT, 0) != cudaSuccess || per_sm < 1) per_sm = 1;
    long long grid = (long long)sm_count() * per_sm;
    const long long need = (n_starts + PT_WARPS - 1) / PT_WARPS;
    if (grid > need) grid = need;
    k_pattern_search<<<(unsigned)grid, PT_NT, 0, st>>>(A);
    QK_LAUNCH_CHECK("k_pattern_search");
    return QK_OK;
}
