/* qk.h -- C-ABI of libqk.so: the sm_90a kernels behind Quokka's operator protocols.
 *
 * The reference (marsupialtail/quokka @ 1caf62e) has NO FFI on this path: its operators are Python
 * classes that delegate to Polars / DuckDB / Arrow.  Each entry point below replaces one of those
 * delegated native calls; the comment on each names the reference call site it stands in for.
 * INTEGRATION.md shows the ctypes binding a reference maintainer would add.
 *
 * Conventions
 *   - every pointer marked "device" is a CUDA device pointer owned by the caller (torch tensors);
 *     the library never allocates, frees or synchronises: all work is enqueued on `stream`
 *     (a cudaStream_t passed as void*; NULL = legacy default stream);
 *   - return value 0 = ok, negative = QK_ERR_*; qk_last_error() gives a thread-local message;
 *   - no nulls on the hot path: qk_column.validity must be NULL (QK_ERR_UNSUPPORTED otherwise), except for the link
 *     columns of qk_pattern_search;
 *     operators that can produce "no match" report it as index -1;
 *   - row counts fit int32 per call (a batch is < 2^31 rows); totals are int64.
 */
#ifndef QK_H
#define QK_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define QK_VERSION 100    /* qk_column.lanes took the place of the always-zero `reserved` word, and 0 keeps its meaning */
#define QK_API __attribute__((visibility("default")))

/* ---- error codes ---- */
#define QK_OK 0
#define QK_ERR_INVALID -1      /* bad argument */
#define QK_ERR_UNSUPPORTED -2  /* valid request outside the implemented subset */
#define QK_ERR_CUDA -3         /* a CUDA runtime call failed */
#define QK_ERR_CAPACITY -4     /* caller-provided buffer too small */

/* ---- column dtypes (Arrow fixed-width layouts) ---- */
#define QK_U8 1     /* uint8: dictionary codes, bool */
#define QK_I32 2    /* int32 (also date32 days) */
#define QK_I64 3    /* int64 */
#define QK_F32 4
#define QK_F64 5
#define QK_F16 6    /* IEEE half: vector columns only (lanes > 1) */

typedef struct qk_column {
    const void* data;        /* device */
    const uint8_t* validity; /* must be NULL */
    int64_t length;
    int32_t dtype;           /* QK_U8 .. QK_F16 */
    int32_t lanes;           /* 0 or 1: scalar column.  > 1: a fixed-width vector column of `length` rows, each `lanes`
                              * contiguous elements of `dtype` (row-major, row i at data + i * lanes * size(dtype)).
                              * Only qk_gather, qk_xchg_push, qk_xchg_recv and qk_knn_topk take lanes > 1; every other
                              * entry point returns QK_ERR_UNSUPPORTED for such a column, and for QK_F16. */
} qk_column;

/* ---- expression programs (postfix), the subset of pyquokka/sql_utils.py:86-223 `evaluate`
 *      that the judged queries use (SURVEY.md Appendix E) ---- */
#define QK_OP_COL 1          /* push (double) column[a0]                       */
#define QK_OP_CONST 2        /* push imm                                        */
#define QK_OP_ADD 3
#define QK_OP_SUB 4
#define QK_OP_MUL 5
#define QK_OP_DIV 6
#define QK_OP_NEG 7
#define QK_OP_LT 8           /* float compares: push 1.0 / 0.0                  */
#define QK_OP_LE 9
#define QK_OP_GT 10
#define QK_OP_GE 11
#define QK_OP_EQ 12
#define QK_OP_NE 13
#define QK_OP_AND 14
#define QK_OP_OR 15
#define QK_OP_NOT 16
#define QK_OP_CMP_COL_IMM 17 /* exact integer compare: column[a0] <a1=cmp> imm_i   (u8/i32/i64 columns) */
#define QK_OP_CMP_COL_COL 18 /* exact integer compare: column[a0] <a1&0xff> column[a1>>8] */
#define QK_OP_RINT 19        /* round to nearest even (CAST(x AS INT) of a double) */
#define QK_OP_IN_SET 20      /* set membership of an integer / dictionary-code column: push bit column[a0] of a bitmap of
                              * a1 bits (codes < 0 or >= a1 are not members).  a1 <= 64: the bitmap is imm_i itself;
                              * a1 > 64: imm_i is a DEVICE pointer to ceil(a1/32) uint32 words (caller-owned, alive
                              * until the call's work has run).  One node replaces the OR-chain a `col LIKE pat` /
                              * `col IN (...)` on a dictionary column would otherwise expand to
                              * (pyquokka/sql_utils.py:131-149 evaluates those through Polars string kernels). */
#define QK_OP_SELECT 21      /* pop else, then, cond; push cond != 0 ? then : else  (CASE WHEN; the condition is
                              * evaluated once and an unselected arm that is NaN / inf does not leak) */

#define QK_OP_EXTRACT 22     /* EXTRACT(part FROM date): replace the top of the stack (days since 1970-01-01) by its civil
                              * year (a1 = 0), month (1) or day of month (2) -- pyquokka/sql_utils.py:204-211 (`.dt.year()` ...) */

#define QK_OP_RANGE_COL_IMM 23 /* exact integer range test: imm_i <= column[a0] <= (int64) imm  (closed; a1 != 0 negates).  What
                              * `col >= a AND col < b` / BETWEEN on a date or key column compiles to: ONE node, so the scan keeps
                              * its fast compaction shape (and its semi-join filter) instead of the per-row interpreter.
                              * The upper bound travels in `imm` (exact for |bound| <= 2^53; larger bounds stay two compares). */

#define QK_CMP_LT 0
#define QK_CMP_LE 1
#define QK_CMP_GT 2
#define QK_CMP_GE 3
#define QK_CMP_EQ 4
#define QK_CMP_NE 5

typedef struct qk_expr_node {
    int32_t op;
    int32_t a0;
    int32_t a1;
    int32_t reserved;
    double imm;
    int64_t imm_i;
} qk_expr_node;

typedef struct qk_expr {
    const qk_expr_node* nodes; /* HOST memory, postfix order; n_nodes == 0 means "true" / absent */
    int32_t n_nodes;
    int32_t reserved;
} qk_expr;

#define QK_MAX_COLS 16
#define QK_MAX_EXPR_NODES 48
#define QK_MAX_STACK 8
#define QK_MAX_AGGS 8
#define QK_MAX_PROJ 16

/* aggregate ops */
#define QK_AGG_SUM 1
#define QK_AGG_MIN 2
#define QK_AGG_MAX 3

QK_API const char* qk_last_error(void);
QK_API int qk_version(void);
/* number of kernel launches issued by this library in this process (bench.py's gpu_launches) */
QK_API int64_t qk_launch_count(void);

/* ---- K1: scan -> filter -> project --------------------------------------------------------
 * Replaces: Arrow `dataset.to_table(filter, columns)` (pyquokka/dataset/unordered_readers.py:98-99),
 * the edge predicate `x.filter(predicate)` / DuckDB `select * ... where` (pyquokka/core.py:156-170),
 * folded `with_columns` batch_funcs (pyquokka/datastream.py:1288-1296) and the projection
 * `payload[sorted(projection)]` (core.py:190-193), in one pass.
 * proj[i]: a single QK_OP_COL node copies the column verbatim in its own dtype (keys stay bit-exact);
 * anything else is evaluated in fp64 and written as QK_F64.
 * pred and every proj[i]: at most QK_MAX_EXPR_NODES nodes and QK_MAX_STACK stack slots each, 112 nodes together
 * (QK_ERR_UNSUPPORTED beyond).
 * out[i].data must hold `nrows` elements; *out_rows (device int64) receives the surviving row count.
 * stable != 0 keeps input row order (two passes over the predicate columns, needs
 * qk_scan_workspace_bytes(nrows) bytes of device workspace); stable == 0 compacts in arrival order
 * (DataStreams are unordered, pyquokka/datastream.py:822). */
QK_API size_t qk_scan_workspace_bytes(int64_t nrows);
QK_API int qk_scan_filter_project(const qk_column* cols, int32_t ncols, int64_t nrows, const qk_expr* pred,
                           const qk_expr* proj, int32_t nproj, qk_column* out, int64_t* out_rows,
                           int32_t stable, void* workspace, size_t ws_bytes, void* stream);

/* ---- semi-join reduction of a probe-side scan (not in the reference; same results) -------------
 * Before a shuffled join's probe input is partitioned and sent, rows whose key cannot be on the build side
 * are dropped by a blocked Bloom filter built from the build keys (one 32-byte block per key, 3 bits).
 * `bits` = nparts filters of words_per_part uint32 words (multiple of 8), filter p covering the build keys with
 * key % nparts == p -- the layout an all-gather of per-rank filters produces.  False positives only cost work:
 * the hash join (BuildProbeJoinExecutor, sql_executors.py:371) still decides every match exactly. */
typedef struct qk_bloom {
    const uint32_t* bits;     /* device */
    int64_t words_per_part;
    int32_t nparts;
    int32_t key_proj;         /* index into proj[] of the (verbatim) join-key column */
} qk_bloom;
/* ORs the keys of `key` into bits[(key % nparts) * words_per_part ...]; bits must be zeroed by the caller */
QK_API int qk_bloom_build(const qk_column* key, uint32_t* bits, int64_t words_per_part, int32_t nparts, void* stream);
/* qk_scan_filter_project restricted to its TMA compaction shape (integer-range predicate or none, verbatim
 * columns), with the Bloom test fused into the predicate; stable output; QK_ERR_UNSUPPORTED otherwise */
QK_API int qk_scan_filter_project_sj(const qk_column* cols, int32_t ncols, int64_t nrows, const qk_expr* pred,
                                     const qk_expr* proj, int32_t nproj, qk_column* out, int64_t* out_rows,
                                     const qk_bloom* bloom, void* workspace, size_t ws_bytes, void* stream);

/* ---- K1+K2: scan -> filter -> project -> dense (dictionary-key) aggregate -----------------
 * Replaces the per-batch partial aggregate `select keys, SUM/MIN/MAX/COUNT(*) ... group by keys`
 * (pyquokka/datastream.py:795-801 via _grouped_aggregate_sql :1829) fused behind the predicate,
 * for group keys whose columns are small non-negative codes (dictionary / u8 / small ints):
 * group id = sum_k code_k * stride_k, stride from `group_card`.  Accumulates (+=, min, max) into
 * acc[n_groups][nagg] (device f64) and cnt[n_groups] (device int64, COUNT(*)), so repeated calls
 * over successive batches implement the partial + final phases of SQLAggExecutor
 * (pyquokka/executors/sql_executors.py:556-599).  Deterministic: per-CTA partials are reduced in a
 * fixed order.  Workspace: qk_scan_agg_workspace_bytes(n_groups, nagg). */
QK_API size_t qk_scan_agg_workspace_bytes(int32_t n_groups, int32_t nagg);
QK_API int qk_scan_filter_agg_dense(const qk_column* cols, int32_t ncols, int64_t nrows, const qk_expr* pred,
                             const int32_t* group_cols, const int32_t* group_card, int32_t ngroup_cols,
                             const qk_expr* agg_expr, const int32_t* agg_op, int32_t nagg,
                             double* acc, int64_t* cnt, void* workspace, size_t ws_bytes,
                             int32_t variant, void* stream);
/* variant: 0 = auto (3, else the interpreter), 1 = generic interpreter, 3 = a typed fused plan with
 * cp.async.bulk (TMA engine) staging of column tiles into shared memory, else the runtime-described
 * fused plan over the same tile ring, 7 = the runtime-described plan only.  Any other value is
 * QK_ERR_INVALID.  Returns QK_ERR_UNSUPPORTED if a forced fused variant has no plan for the request. */
/* name of the kernel variant the last qk_scan_filter_agg_dense call on this thread dispatched to */
QK_API const char* qk_last_variant(void);
/* launch shape of that kernel, e.g. "nt256v2s3" = 256 threads, 2 rows/thread/tile, 3 TMA stages */
QK_API const char* qk_last_variant_config(void);

/* ---- K2 (high cardinality): hash aggregate -------------------------------------------------
 * Replaces the DuckDB hash aggregate behind the partial / final SQL of _grouped_aggregate_sql
 * (pyquokka/datastream.py:1819-1856) and SQLAggExecutor.done (sql_executors.py:592-599) when keys are
 * not dense codes (Q3: ~1.16 M groups).  Keys: 1..4 integer columns (u8/i32/i64) totalling <= 128
 * bits, compared exactly.  Values: nagg fp64 columns (sum / min / max) + COUNT(*).
 * The state lives in caller memory of qk_hashagg_state_bytes(capacity, nagg) bytes; capacity is a
 * power of two and must stay > the number of distinct groups (QK_ERR_CAPACITY is reported through
 * *overflow, device int32, set non-zero when the table fills). */
typedef struct qk_hashagg_desc {   /* HOST memory, caller-owned, the same values on every call */
    int64_t capacity;              /* power of two */
    int32_t nkeys;                 /* 1..4 */
    int32_t key_dtype[4];
    int32_t nagg;                  /* 0..QK_MAX_AGGS */
    int32_t agg_op[QK_MAX_AGGS];
} qk_hashagg_desc;
QK_API size_t qk_hashagg_state_bytes(const qk_hashagg_desc* desc);
QK_API int qk_hashagg_init(const qk_hashagg_desc* desc, void* state, void* stream);
QK_API int qk_hashagg_update(const qk_hashagg_desc* desc, void* state, const qk_column* keys, const qk_column* vals,
                      int64_t nrows, int32_t* overflow, void* stream);
/* compacts occupied slots: out_keys[i] (dtype as in desc), out_vals[j] (f64), out_cnt (device int64);
 * each needs room for min(capacity, expected groups) rows -- `out_capacity` rows are never exceeded;
 * *out_groups (device int64) = total number of groups (> out_capacity means truncated output). */
QK_API int qk_hashagg_finalize(const qk_hashagg_desc* desc, const void* state, qk_column* out_keys, qk_column* out_vals,
                        int64_t* out_cnt, int64_t out_capacity, int64_t* out_groups, void* stream);

/* ---- K3: partition -------------------------------------------------------------------------
 * Replaces `partition_key_str` (pyquokka/quokka_runtime.py:217-231): integer keys -> channel
 * `key % nparts` (mode QK_PART_MOD, bit-identical placement to the reference for non-negative keys)
 * followed by Polars `partition_by`.  Also used with QK_PART_CODE (key is already a dense code
 * in [0, nparts), codes outside are clamped: segment-by-symbol for the as-of join and the windows).
 * Stable: rows keep their relative order inside a partition.  dest[i] (device int32) = output
 * position of row i; part_offsets (device int64[nparts+1]) = start of each partition in the output.
 * Then qk_scatter moves each column.  QK_PART_MOD takes nparts in [1, 16384]; QK_PART_CODE any
 * nparts >= 1 (above 16384 the partition runs one stable pass per 14-bit digit of the code), bounded
 * by qk_partition_workspace_bytes(nrows, nparts). */
#define QK_PART_MOD 0
#define QK_PART_CODE 1
QK_API size_t qk_partition_workspace_bytes(int64_t nrows, int32_t nparts);
QK_API int qk_partition_plan(const qk_column* key, int32_t nparts, int32_t mode, int32_t* dest,
                      int64_t* part_offsets, void* workspace, size_t ws_bytes, void* stream);
QK_API int qk_scatter(const qk_column* cols, int32_t ncols, const int32_t* dest, qk_column* out, void* stream);
/* ---- K6: the shuffle over peer-mapped memory ------------------------------------------------------
 * Replaces TaskManager.push -> Flight do_put / do_get (pyquokka/core.py:276-376, pyquokka/flight.py:44-264): one
 * process per GPU, every rank owns a CHANNEL = a control block (qk_xchg_ctrl_bytes(), zeroed once) + a mailbox, both
 * inside a symmetric allocation that every peer has mapped (ctrl[p] / mailbox[p] = rank p's copies as THIS process
 * addresses them).  One exchange = qk_xchg_meta -> [host reads the meta matrix] -> qk_xchg_push[_scatter] ->
 * qk_xchg_recv, all ranks with the same `epoch` (1, 2, 3, ... per channel).  No NCCL call, no host barrier: ranks
 * synchronise through release / acquire flags in the control blocks (waits are single-CTA kernels with a deadline;
 * a wait that times out sets the error word reported by the next qk_xchg_meta).
 *
 * qk_xchg_meta: stores this rank's meta row into every peer -- words[0 .. QK_XCHG_META_WORDS) from the host, except that
 *   with part_offsets != NULL (device int64[world+1], the partition plan's output) words[d] = rows for rank d are taken
 *   from the device, so the producer needs no host sync to learn its own counts -- waits for every peer's row and
 *   writes the matrix [world][QK_XCHG_META_WORDS] + one error word to out_dev (device) and / or out_host (pinned host
 *   memory, device-accessible).  It is also the "mailbox may be overwritten" barrier for this epoch.
 * qk_xchg_push: contiguous rows [send_lo[d], send_hi[d]) of every column go to rank d (broadcast, single owner,
 *   pre-grouped rows); dst_byte_off[d * ncols + c] = byte offset inside rank d's mailbox of the first element this
 *   rank writes for column c.
 * qk_xchg_push_scatter: the fused partition scatter + all-to-all: row i goes to the rank whose partition holds
 *   dest[i] (qk_partition_plan's output), at element (dest[i] - part_offsets[rank]) from dst_byte_off; a tile of rows
 *   is ordered by destination in shared memory and leaves as one coalesced run per destination.
 * qk_xchg_recv: waits until every peer's rows of this epoch have landed, then copies column c (out[c].length
 *   rows from byte offset src_byte_off[c] of the own mailbox, 16-byte aligned) into out[c].
 * A row of column c is size(dtype) * max(1, lanes) bytes: qk_xchg_push and qk_xchg_recv move vector columns (lanes > 1);
 * qk_xchg_push_scatter returns QK_ERR_UNSUPPORTED for them.  A link has at most QK_MAX_PEERS ranks.
 * One push / recv takes at most QK_XCHG_MAX_BUFS buffers (24 columns + a validity mask for each, as uint8 buffers), more
 * than QK_MAX_COLS: every buffer of an edge must go in ONE push, because the push releases the peers' "data landed" flag
 * after its last store and a receiver may copy out as soon as it sees that flag. */
#define QK_MAX_PEERS 16
#define QK_XCHG_MAX_BUFS 48
#define QK_XCHG_META_WORDS 48
#define QK_XCHG_CTRL_BYTES 16384
typedef struct qk_xchg {
    int32_t world, rank;
    uint64_t ctrl[QK_MAX_PEERS];
    uint64_t mailbox[QK_MAX_PEERS];
    int64_t mailbox_bytes;
    int64_t timeout_ms;        /* deadline of a wait; <= 0: 30 s */
} qk_xchg;
QK_API size_t qk_xchg_ctrl_bytes(void);
QK_API int qk_xchg_meta(const qk_xchg* x, uint64_t epoch, const int64_t* part_offsets, const int64_t* words,
                        int64_t* out_dev, int64_t* out_host, void* stream);
QK_API int qk_xchg_push(const qk_xchg* x, uint64_t epoch, const qk_column* cols, int32_t ncols, const int64_t* send_lo,
                        const int64_t* send_hi, const int64_t* dst_byte_off, void* stream);
QK_API int qk_xchg_push_scatter(const qk_xchg* x, uint64_t epoch, const qk_column* cols, int32_t ncols, const int32_t* dest,
                                const int64_t* part_offsets, const int64_t* dst_byte_off, void* stream);
QK_API int qk_xchg_recv(const qk_xchg* x, uint64_t epoch, const int64_t* src_byte_off, qk_column* out, int32_t ncols, void* stream);
/* out[c][i] = cols[c][idx[i]] for i < n_idx; idx == -1 writes 0 (left join / as-of "no match").  A vector column (lanes > 1)
 * moves whole rows; out[c] must have the same dtype and lanes. */
QK_API int qk_gather(const qk_column* cols, int32_t ncols, const int32_t* idx, int64_t n_idx, qk_column* out,
              void* stream);

/* ---- K4 / K5: hash join build + probe ------------------------------------------------------
 * Replaces BuildProbeJoinExecutor (pyquokka/executors/sql_executors.py:325-377): stream 1 batches
 * are inserted (state.vstack, :356-358) -- the table is PERSISTENT across probe batches, unlike
 * Polars `batch.join(state)` which rebuilds per call (:371) -- stream 0 batches probe it.
 * Open addressing, linear probing, int64 keys compared exactly, duplicate build keys kept (each
 * build row owns a slot).  Table memory: qk_join_table_bytes(capacity), capacity = power of two
 * >= 2 x build rows.  Build rows are numbered row_base + i so several build batches share one table. */
#define QK_JOIN_INNER 0
#define QK_JOIN_LEFT 1
#define QK_JOIN_SEMI 2
#define QK_JOIN_ANTI 3
QK_API size_t qk_join_table_bytes(int64_t capacity);
QK_API int qk_join_init(void* table, int64_t capacity, void* stream);
/* *flags (device int32, optional): bit 0 set when the table overflowed, bit 1 when a key equals the
 * reserved EMPTY sentinel INT64_MIN (such rows are skipped), bit 2 when duplicate build keys exist. */
QK_API int qk_join_build(void* table, int64_t capacity, const qk_column* key, int32_t row_base, int32_t* flags, void* stream);
/* Probe.  out_probe_idx / out_build_idx: device int32[out_capacity]; *out_count: device int64,
 * total pairs (may exceed out_capacity: then only the first out_capacity are written and the caller
 * retries with a larger buffer).  semi/anti write probe indices only.  Pair order is unspecified. */
QK_API int qk_join_probe(const void* table, int64_t capacity, const qk_column* key, int32_t how, int32_t* out_probe_idx,
                  int32_t* out_build_idx, int64_t out_capacity, int64_t* out_count, void* stream);
/* Ordered probe, behind DataStream.join(maintain_sort_order="left" | "right") (pyquokka/datastream.py:1453-1469, :1536-1553,
 * where the reference keeps the order by joining batch by batch in its executor).  The same table, arguments and pairs as
 * qk_join_probe, in a fixed order: by probe row, a row's matches in ascending build-row number; a left join's unmatched row
 * is one pair with build -1; semi / anti write probe indices only, ascending.  Deterministic for any number of matches per
 * row.  *out_count = total pairs (may exceed out_capacity: then nothing past out_capacity is written and the caller retries).
 * Workspace: qk_join_probe_ordered_workspace_bytes(key->length) (16 B per probe row; too small: QK_ERR_CAPACITY). */
QK_API size_t qk_join_probe_ordered_workspace_bytes(int64_t nrows);
QK_API int qk_join_probe_ordered(const void* table, int64_t capacity, const qk_column* key, int32_t how, int32_t* out_probe_idx,
                                 int32_t* out_build_idx, int64_t out_capacity, int64_t* out_count, void* workspace,
                                 size_t ws_bytes, void* stream);
/* Placement of an ordered join's rows that come back to the rank holding the left rows: pos (device int32[nrecv]) = the left
 * position of every received row, in [0, nleft); each sender's run is ascending and all rows of one position are contiguous.
 * Output row d, in left order (rows of one position in the order they arrived): out_src[d] = the received row,
 * out_left[d] (optional) = its position; nrecv rows in all.  Deterministic, no sort.
 * Workspace: qk_join_place_workspace_bytes(nleft) (16 B per left row; too small: QK_ERR_CAPACITY). */
QK_API size_t qk_join_place_workspace_bytes(int64_t nleft);
QK_API int qk_join_place(const int32_t* pos, int64_t nrecv, int64_t nleft, int32_t* out_src, int32_t* out_left, void* workspace,
                         size_t ws_bytes, void* stream);

/* ---- K7: backward as-of join by key ---------------------------------------------------------
 * Replaces Polars `join_asof(by=..., strategy="backward")` in SortedAsofExecutor
 * (pyquokka/executors/ts_executors.py:369,383).  Both sides time-sorted (int64 `time`), `by` = dense
 * int32 codes in [0, n_by).  out_ridx[i] (device int32) = index of the LAST right row with the same
 * code and r_time <= l_time[i], or -1. */
QK_API size_t qk_asof_workspace_bytes(int64_t n_right, int32_t n_by);
QK_API int qk_asof_backward(const qk_column* l_time, const qk_column* l_by, const qk_column* r_time,
                     const qk_column* r_by, int32_t n_by, int32_t* out_ridx, void* workspace,
                     size_t ws_bytes, void* stream);

/* The sorted-merge form of the same join (the default when the per-key table fits shared memory: n_by <= ~40 000):
 * ONE sweep over the merged timeline carrying last[key] = newest right row of every key, cut into windows of 1024 merged
 * rows (merge-path diagonals), a CTA per run of windows with its table in shared memory; no sort, no scatter.
 * n_left = 0 is allowed and computes carry_out only (the newest right row of every key).  carry_in rows must be numbered
 * below r_base (they are older than every row of this call).
 * Streaming: carry_in (device int32[n_by] or NULL = all -1) is what a left row receives when no right row of its key
 * precedes it in THIS call (the newest row of earlier batches); the rows of this call are numbered r_base + i in the
 * output; carry_out (device int32[n_by] or NULL) receives the table after the last right row.  So successive batches of
 * the two sorted streams cost O(batch) each (SortedAsofExecutor keeps its whole quote state and re-joins against it,
 * pyquokka/executors/ts_executors.py:359-383).  Same tie rule as qk_asof_backward: the LAST right row with r_time <= l_time. */
QK_API size_t qk_asof_merge_workspace_bytes(int64_t n_left, int64_t n_right, int32_t n_by);
QK_API int qk_asof_merge(const qk_column* l_time, const qk_column* l_by, const qk_column* r_time, const qk_column* r_by,
                         int32_t n_by, const int32_t* carry_in, int32_t r_base, int32_t* carry_out, int32_t* out_ridx,
                         void* workspace, size_t ws_bytes, void* stream);

/* As-of joins in the other directions, and with a match tolerance: OrderedStream.join_asof(strategy=..., tolerance=...)
 * (pyquokka/orderedstream.py:114-191 offers backward only; the reference's apps/rottnest/backtester.py:60 fills every
 * signal at the next trade tick with Polars' strategy="forward").  The target is pandas.merge_asof(direction=strategy,
 * tolerance=tolerance):
 *   QK_ASOF_BACKWARD  the LAST right row of the key with r_time <= l_time (the join above);
 *   QK_ASOF_FORWARD   the FIRST right row of the key with r_time >= l_time (the earliest in stream order among equal times);
 *   QK_ASOF_NEAREST   of the backward and the forward candidate the one with the smaller |r_time - l_time|; a distance tie goes
 *                     to the backward one (an exact match takes the LAST right row at that time).
 * tolerance >= 0 keeps the chosen row only if |r_time - l_time| <= tolerance (else -1); tolerance < 0 = none.  The nearest pick
 * and the tolerance are applied where the answer is written. */
#define QK_ASOF_BACKWARD 0
#define QK_ASOF_FORWARD 1
#define QK_ASOF_NEAREST 2
/* The sorted-merge form (n_by within the shared-memory table; 0 from the sizing function otherwise, or for an unknown strategy).
 * Forward is the mirror of qk_asof_merge's sweep: left rows first on merge-path ties, a table of the OLDEST right row at or after
 * the current point, walked from the end.  Nearest runs both sweeps.  Local right rows are numbered r_base + i.
 * carry_back (device int32[n_by] or NULL): the answer of a key with no local right row at or before l_time; its rows are below
 * r_base.  carry_fwd: the same for no local right row at or after l_time; its rows are at or past r_base + n_right (and below
 * 2^31 - 1).  carry_back_time / carry_fwd_time (device int64[n_by]) are the times of those rows, required with their table.
 * Backward takes carry_back only, forward carry_fwd only, nearest both.  carry_out (device int32[n_by] or NULL; not for nearest):
 * backward = the newest row of every key after this call's rows (as qk_asof_merge), forward = the OLDEST row of every key
 * (local or carry_fwd), -1 none; n_left = 0 computes it alone.  Workspace: qk_asof_join_workspace_bytes (QK_ERR_CAPACITY when
 * short, before any launch). */
QK_API size_t qk_asof_join_workspace_bytes(int64_t n_left, int64_t n_right, int32_t n_by, int32_t strategy);
QK_API int qk_asof_join(const qk_column* l_time, const qk_column* l_by, const qk_column* r_time, const qk_column* r_by,
                        int32_t n_by, int32_t strategy, int64_t tolerance, const int32_t* carry_back, const int64_t* carry_back_time,
                        const int32_t* carry_fwd, const int64_t* carry_fwd_time, int32_t r_base, int32_t* carry_out,
                        int32_t* out_ridx, void* workspace, size_t ws_bytes, void* stream);
/* The partition + search form for any n_by (the large symbol sets): lower bound for forward, both neighbours of the upper
 * bound for nearest, the tolerance at the write.  out_ridx[i] = right row, or -1.  Workspace: qk_asof_workspace_bytes. */
QK_API int qk_asof_search_join(const qk_column* l_time, const qk_column* l_by, const qk_column* r_time, const qk_column* r_by,
                               int32_t n_by, int32_t strategy, int64_t tolerance, int32_t* out_ridx, void* workspace,
                               size_t ws_bytes, void* stream);

/* ---- time-series windows over a key-segmented, time-sorted stream ------------------------------------------------
 * Replace Polars groupby_rolling / groupby_dynamic and the DuckDB window SQL of HoppingWindowExecutor,
 * SlidingWindowExecutor and SessionWindowExecutor (pyquokka/executors/ts_executors.py:12-288).  Inputs are in KEY-SEGMENTED
 * order (qk_partition_plan with QK_PART_CODE + qk_scatter: rows of one key contiguous, time-sorted inside): time int64,
 * by = dense int32 codes, seg = device int64[n_by + 1] segment starts.
 * qk_window_sliding: out[o][i] = aggregate ops[o] of vals[srcs[o]] over the rows of row i's key with time in
 *   (time[i] - size, time[i]] (ties at time[i] included), all fp64 (COUNT too).
 * qk_window_hop_expand: row i goes to every window [k * hop, k * hop + size) that contains it; `slots` >= ceil(size / hop)
 *   output slots per row: wstart / key / src (src = i, or -1 for an unused slot or a window that starts before the key's
 *   first truncated timestamp, which Polars' start_by = "window" does not produce).  The caller hash-aggregates on (key, wstart).
 * qk_window_session_ids: ids[i] (device int64, 1-based, increasing) = session of row i: a new one starts at a key's
 *   first row and after every gap > timeout. */
#define QK_WIN_SUM 1
#define QK_WIN_MIN 2
#define QK_WIN_MAX 3
#define QK_WIN_COUNT 4
#define QK_WIN_AVG 5
QK_API int qk_window_sliding(const qk_column* time, const qk_column* by, const int64_t* seg, int32_t n_by, int64_t size,
                             const qk_column* vals, int32_t nvals, const int32_t* ops, const int32_t* srcs, int32_t nout,
                             qk_column* out, void* stream);
QK_API int qk_window_hop_expand(const qk_column* time, const qk_column* by, const int64_t* seg, int32_t n_by, int64_t size, int64_t hop,
                                int32_t slots, int64_t* wstart, int32_t* key, int32_t* src, void* stream);
QK_API size_t qk_window_session_workspace_bytes(int64_t nrows);
QK_API int qk_window_session_ids(const qk_column* time, const qk_column* by, int64_t timeout, int64_t* ids, void* workspace,
                                 size_t ws_bytes, void* stream);

/* Per-event (OnEventTrigger) tumbling and session windows: the DuckDB window query of HoppingWindowExecutor /
 * SessionWindowExecutor (ts_executors.py:64-96, 109-136, 239-288), PARTITION BY key, window ORDER BY time
 * RANGE UNBOUNDED PRECEDING.  The rows of a key are cut into runs: QK_WIN_RUN_TUMBLING, param = size > 0: the rows with one
 * floor(time / size); QK_WIN_RUN_SESSION, param = timeout >= 0: a new run after every gap > timeout.  out[o][i] = aggregate
 * ops[o] of vals[srcs[o]] over the rows of row i's run with time <= time[i] (rows with equal times all get the value that
 * includes them), all fp64 (COUNT too), in the same arguments as qk_window_sliding.  Deterministic: the same bits on every
 * call.  Workspace: qk_window_running_workspace_bytes(rows). */
#define QK_WIN_RUN_TUMBLING 1
#define QK_WIN_RUN_SESSION 2
QK_API size_t qk_window_running_workspace_bytes(int64_t nrows);
QK_API int qk_window_running(const qk_column* time, const qk_column* by, const int64_t* seg, int32_t n_by, int32_t kind, int64_t param,
                             const qk_column* vals, int32_t nvals, const int32_t* ops, const int32_t* srcs, int32_t nout,
                             qk_column* out, void* workspace, size_t ws_bytes, void* stream);

/* ---- K8: top-k candidates -------------------------------------------------------------------
 * Replaces the `order by ... limit k` of DataStream.top_k / ConcatThenSQLExecutor
 * (pyquokka/datastream.py:1746-1767, sql_executors.py:45-67) for the primary sort column: radix
 * select on an order-preserving 64-bit image of `key` (descending != 0 flips it); writes the indices
 * of every row whose key is >= (<=) the k-th best (ties included) to out_idx (device int32[n]) and
 * their number to *out_n (device int64).  The host orders the few survivors on all sort columns. */
QK_API size_t qk_topk_workspace_bytes(int64_t nrows);
QK_API int qk_topk_candidates(const qk_column* key, int32_t k, int32_t descending, int32_t* out_idx,
                       int64_t* out_n, void* workspace, size_t ws_bytes, void* stream);

/* ---- K9: Gram matrix on the FP64 tensor cores ------------------------------------------------
 * Replaces the per-batch np.dot(x.T, x) of DataStream.gramian and the sums of DataStream.covariance
 * (pyquokka/datastream.py:1033-1147).  X = nrows x k, cols[i] one column (QK_F64 / QK_F32 / QK_I32 / QK_I64, all of length
 * nrows), widened to fp64 as it is staged; shift (device fp64[k] or NULL = 0) is subtracted in fp64 before the product, so a
 * shifted value rounds as `x.to_numpy() - demean` does.  Accumulates
 *     gram[i * k + j] += sum_rows (x_i - c_i)(x_j - c_j)   (device fp64[k * k], row-major, symmetric)
 *     sums[i]         += sum_rows (x_i - c_i)              (device fp64[k], or NULL = not computed)
 * so successive calls over the batches of a stream sum up.  Products run on mma.sync f64 (DMMA); only the tiles on and above
 * the diagonal are computed and mirrored.  Deterministic: per-CTA partial tiles are folded in a fixed order, so the same
 * inputs give bit-identical results on the same device.  Every row is read once when k + 1 <= 128 (one column block).
 * variant: 0 = auto (m16n8k16 where the tile shape allows it, k + 1 > 8; m8n8k4 below), 1 = m8n8k4, 2 = m16n8k16.
 * Workspace: qk_gram_workspace_bytes(nrows, k) bytes; the column table travels in it, so any k fits.  nrows == 0 is a no-op.
 * Errors: k < 1, null data with length > 0, a length != nrows or an unsupported dtype: QK_ERR_INVALID; a validity mask:
 * QK_ERR_UNSUPPORTED; workspace too small: QK_ERR_CAPACITY. */
QK_API size_t qk_gram_workspace_bytes(int64_t nrows, int32_t k);
QK_API int qk_gram(const qk_column* cols, int32_t k, int64_t nrows, const double* shift, double* gram, double* sums,
                   int32_t variant, void* workspace, size_t ws_bytes, void* stream);
/* tile shape, MMA shape and row-range split of the last qk_gram call on this thread, e.g. "T128 m8n8k4 s1" */
QK_API const char* qk_gram_last_plan(void);

/* ---- K10: quantile sketch -------------------------------------------------------------------------
 * Replaces the host t-digest plugin (ldbpy.NTDigest) of DataStream.approximate_quantile / approximate_median
 * (pyquokka/datastream.py:905-1031).  Every value is widened to fp64 and mapped to its order-preserving image
 * (sign bit set for positives, all bits flipped for negatives; NaN first made 0x7FF8000000000000, so it sorts last).  The
 * sketch is an open-addressed device table of `capacity` qk_qslot (a power of two): per key = column << 22 | bucket,
 * bucket = image >> QK_QSKETCH_SHIFT (sign, exponent and the top 10 mantissa bits), the row count and the smallest and
 * largest image.  An empty slot is {QK_QSKETCH_EMPTY, 0, ~0, 0}: the caller fills a new table with that pattern.  The state
 * depends only on the multiset of values, so sketches of any split of the rows merge into the same table.
 * ctrl: device uint64[4] owned by the caller, zero when the table is new.  ctrl[0] = occupied slots (reservations included
 * while a call runs; exact when it has finished), ctrl[1] = tiles deferred by the last update, ctrl[2] = 1 when a probe ran
 * through the whole table (a caller that broke the load limit; the entries concerned were dropped).
 *
 * qk_qsketch_update: folds k columns of nrows rows (QK_F64 / QK_F32 / QK_I64 / QK_I32 / QK_U8) into the table.  valid: NULL
 * or a HOST array of k device uint8 row masks (an entry may be NULL); a row counts where its mask is non-zero
 * (qk_column.validity stays NULL, per the convention above).  The work unit is a tile of QK_QSKETCH_TILE rows of one column,
 * tile t = column * ceil(nrows / QK_QSKETCH_TILE) + row tile.  tiles: NULL = all k * ceil(nrows / TILE) tiles (ntiles must
 * equal that), or a device int32 list of ntiles tile ids.  A tile whose new buckets would push the load past capacity / 2
 * is not counted at all: its id is appended to `deferred` (device int32, room for ntiles) and ctrl[1] counts it.  The
 * caller reads ctrl, grows the table (qk_qsketch_merge of the old entries into a larger one) and runs the deferred list
 * again; every row is counted exactly once.  ctrl[1] is cleared by the call.  Workspace: qk_qsketch_workspace_bytes(k).
 * qk_qsketch_merge: inserts n compacted entries (device uint64 key / count / min image / max image arrays; key
 * QK_QSKETCH_EMPTY is skipped), adding counts and taking min / max, and counts newly claimed slots in ctrl[0].  The caller
 * keeps ctrl[0] + n <= capacity / 2.
 * Errors: k < 1, a length != nrows, a bad dtype, a capacity that is not a power of two in [QK_QSKETCH_MIN_CAPACITY, 2^31],
 * null table / ctrl, an ntiles that does not match: QK_ERR_INVALID; a validity bitmap, more than 2^31 - 1 tiles:
 * QK_ERR_UNSUPPORTED; a small workspace, n > capacity / 2 in a merge: QK_ERR_CAPACITY. */
#define QK_QSKETCH_SHIFT 42
#define QK_QSKETCH_EMPTY 0xFFFFFFFFFFFFFFFFULL
#define QK_QSKETCH_MIN_CAPACITY 4096
#define QK_QSKETCH_TILE 2048
typedef struct qk_qslot {
    uint64_t key;
    uint64_t count;
    uint64_t min_image;
    uint64_t max_image;
} qk_qslot;
QK_API size_t qk_qsketch_workspace_bytes(int32_t k);
QK_API int qk_qsketch_update(const qk_column* cols, const uint8_t* const* valid, int32_t k, int64_t nrows, qk_qslot* table,
                             int64_t capacity, uint64_t* ctrl, const int32_t* tiles, int64_t ntiles, int32_t* deferred,
                             void* workspace, size_t ws_bytes, void* stream);
QK_API int qk_qsketch_merge(const uint64_t* keys, const uint64_t* counts, const uint64_t* mins, const uint64_t* maxs, int64_t n,
                            qk_qslot* table, int64_t capacity, uint64_t* ctrl, void* stream);

/* ---- K11: nearest neighbours by cosine similarity -------------------------------------------------
 * Replaces the per-batch np.dot + argsort of DFProbeDataStreamNNExecutor1 (pyquokka/executors/vector_executors.py:8-52) behind
 * DataStream.vector_nn_join.  x = one vector column (QK_F32 or QK_F16, lanes = d in [1, QK_KNN_MAX_DIM], length n rows);
 * probes = device fp32 [q][d], already normalised (the host normalises in fp64 and rounds to fp32).  For every probe p the
 * score of row i is s = (x_i . p) / ||x_i||; rows whose squared norm (fp64) is 0 or not finite -- zero rows, rows holding a NaN
 * or an inf -- and non-finite scores never match.  Writes the k best rows of the call per probe,
 * out_score[p * k + j] (f32) / out_row[p * k + j] (int64 row of x), in descending score, ties by smaller row; fewer than k
 * valid rows leave row -1 and score -inf in the remaining slots.  1 <= k <= QK_KNN_MAX_K, q >= 1.
 * One fused pass: rows are staged into shared memory by cp.async (16-byte copies when the column is 16-byte aligned and a row
 * is a whole number of 16-byte units), dot products run on the tensor cores (mma.sync TF32, 3xTF32: x_lo p_hi + x_hi p_lo +
 * x_hi p_hi with f32 accumulation; an f16 row is exact in TF32, so f16 rows take the two probe terms), the row's squared norm
 * accumulates in fp64 from the same staged chunk, and each CTA keeps a per-probe top-k in shared memory (only scores above its
 * current k-th enter); the per-CTA lists are folded in CTA order.  The n x q score matrix is never written.
 * Error: |s - s64| <= (d + 8) * 2^-21, s64 the exact cosine of the stored values and the fp32 probe, for rows whose non-zero
 * elements have magnitudes in [2^-80, 2^80] (the fp32 products and sums of the dot product stay normal and finite there);
 * outside that range a score may be less accurate, and a row whose dot product overflows never matches.
 * Determinism: a score is computed by the same sequence of operations (8-element MMA steps in element order with the three
 * terms in a fixed order; the squared norm in fixed blocks of 16) whatever the row's position, the batch size, q, k or the grid,
 * so it is bit-identical across batchings and ranks, and the output, a total order on (score, row), is bit-identical across
 * calls.
 * Workspace: qk_knn_workspace_bytes(n, d, q, k); the caller chunks large q to bound it.
 * qk_knn_merge: per probe, the best k of two candidate lists a (q x ka) and b (q x kb), each sorted by the same rule with
 * 64-bit keys (arrival order) in place of rows and key -1 after its last entry: descending score, ties by smaller key, ties
 * of both by a.  out_src[p * k + j] = p * ka + i for a's entry i, q * ka + p * kb + i for b's, -1 for padding (key -1,
 * score -inf).  Used across the batches of a rank and across ranks. */
#define QK_KNN_MAX_DIM 4096
#define QK_KNN_MAX_K 256
QK_API size_t qk_knn_workspace_bytes(int64_t n, int32_t d, int32_t q, int32_t k);
QK_API int qk_knn_topk(const qk_column* x, const float* probes, int32_t q, int32_t k, float* out_score, int64_t* out_row,
                       void* workspace, size_t ws_bytes, void* stream);
QK_API int qk_knn_merge(int32_t q, const float* a_score, const int64_t* a_key, int32_t ka, const float* b_score,
                        const int64_t* b_key, int32_t kb, int32_t k, float* out_score, int64_t* out_key, int32_t* out_src,
                        void* stream);

/* ---- K12: complex event recognition over a key-segmented, time-sorted stream ---------------------------------------
 * Replaces the per-batch DuckDB range join and Python DFS of CEPExecutor (pyquokka/executors/cep_executors.py:86-178) behind
 * OrderedStream.pattern_recognize (pyquokka/orderedstream.py:37-53).  Inputs are in KEY-SEGMENTED order (as for the windows):
 * time int64, by = dense int32 codes in [0, n_by), seg = device int64[n_by + 1] segment starts.  cand = device uint8[n]: bit e set
 * when row r satisfies the row-local conjuncts of event e (evaluated before by qk_scan_filter_project).  starts = device int32
 * rows (each with cand bit 0 set and inside its key's segment, seg[by[s]] <= s < seg[by[s] + 1] <= n; others give no match).  m = 2 .. QK_PATTERN_MAX_EVENTS events.
 * A match of start r0 is rows r0 < r1 < ... < r(m-1) of r0's segment with time strictly increasing from one event to the next,
 * t(r(m-1)) <= t(r0) + maxspan, cand bit e of r_e set and links[e] true over the bound rows.  The reported match is the one with
 * the lexicographically smallest (t1 .. t(m-1)); out_bound[s * m + e] (device int32) = its row for event e, or -1 for every e when
 * start s has none.
 * links = HOST array of m programs: links[0] is empty, links[e] (empty = true) is postfix over the link columns with
 * QK_OP_COL a0 = link column, a1 = the event whose bound row is read (a1 = e: the row being tested); ops: COL, CONST, ADD, SUB,
 * MUL, DIV, NEG, the six float compares, AND, OR, NOT, SELECT; fp64; at most QK_MAX_EXPR_NODES nodes each, 128 together.
 * link_cols: nlink <= QK_MAX_COLS scalar columns of n rows.  THIS IS THE ONE ENTRY POINT THAT ACCEPTS qk_column.validity: a
 * device uint8 per row (0 = NULL); a link program that reads a NULL is false.
 * budget: the rows one start may test; a start that exceeds it gives -1 and is counted in status.  status = device
 * uint64[QK_PATTERN_STATUS_WORDS], zeroed by the call: [0] starts over budget, [1] n_starts - (smallest index into starts of such a
 * start), 0 when none; the other words are the call's own.  rows_tested (device uint64 or NULL) accumulates the rows tested.
 * Errors: bad arguments or programs: QK_ERR_INVALID; an op outside the subset, more stack or nodes than allowed, a vector link
 * column: QK_ERR_UNSUPPORTED. */
#define QK_PATTERN_MAX_EVENTS 8
#define QK_PATTERN_STATUS_WORDS 4
QK_API int qk_pattern_search(const qk_column* time, const qk_column* by, const int64_t* seg, int32_t n_by, const uint8_t* cand,
                             const int32_t* starts, int64_t n_starts, int32_t m, int64_t maxspan, const qk_column* link_cols,
                             int32_t nlink, const qk_expr* links, int64_t budget, int32_t* out_bound, uint64_t* status,
                             uint64_t* rows_tested, void* stream);

/* ---- K13: stable radix sort to a permutation ---------------------------------------------------------------------
 * Replaces the per-batch polars sort, the spill files and the final merge of SuperFastSortExecutor
 * (pyquokka/executors/sql_executors.py:128,153,185) behind DataStream.sort.  key = one scalar column (QK_U8 / QK_I32 / QK_I64 /
 * QK_F32 / QK_F64) of nrows rows.  perm_out (device int32[nrows]) receives the row numbers of `key` in ascending order of the
 * 64-bit order image: integers exact over their whole range, -0.0 = +0.0, every NaN after +inf; descending != 0 sorts by the
 * complemented image (NaN first).  valid (device uint8 per row of `key`, or NULL): rows with valid == 0 come after every valid
 * row in both directions and tie with each other (NULLS LAST).
 * STABLE: rows with equal images keep the order they have in perm_in (device int32[nrows], a permutation of the row numbers;
 * NULL = identity), so a multi-column sort is a chain of calls, last column first, each reading key[perm_in[i]].
 * image_out (device uint64[nrows] or NULL) receives the sorted images as the sort compared them (already complemented when
 * descending; the image of a NULL row is 0, ~0 when descending).
 * An LSD radix sort of (image, row number) pairs by 8-bit digits; a digit in which all valid rows agree costs no pass, which the
 * device decides from the histograms of the first pass (no host round trip).  Deterministic: positions are sums of counts.
 * Workspace: qk_sort_workspace_bytes(nrows) (two pair buffers: 24 B/row, plus 3 MB).  nrows == 0 is a no-op.
 * Errors: nrows > 2^31 - 1: QK_ERR_UNSUPPORTED; key->length != nrows, a bad dtype, null perm_out: QK_ERR_INVALID; a vector
 * column: QK_ERR_UNSUPPORTED; workspace too small: QK_ERR_CAPACITY.
 * qk_sort_last_plan: the passes the last qk_sort_perm of this thread ran, e.g. "d8 passes=2/8 nulls=0" (8-bit digits, live
 * image passes of 8, whether the NULL pass ran).  It waits for the device and reads the plan back: for tests and benchmarks. */
QK_API size_t qk_sort_workspace_bytes(int64_t nrows);
QK_API int qk_sort_perm(const qk_column* key, const uint8_t* valid, int32_t descending, const int32_t* perm_in, int32_t* perm_out,
                        uint64_t* image_out, int64_t nrows, void* workspace, size_t workspace_bytes, void* stream);
QK_API const char* qk_sort_last_plan(void);

/* ---- K14: lag / lead per key over a stream in order -----------------------------------------------------------------
 * Stands in for OrderedStream.shift(n, by, fill_value) (pyquokka/orderedstream.py:13-35), whose ShiftOperator the reference
 * imports and never defines; the semantics are Polars' pl.all().shift(n, fill_value).over(by).
 * qk_shift_plan: rows 0 .. nrows-1 in stream order.  by = device int32 codes in [0, n_by), with dest / seg the output of
 * qk_partition_plan(by, n_by, QK_PART_CODE) (stable); or all three NULL: one key.  For each row i in [lo, hi), src[i - lo]
 * (device int32) receives the row n places EARLIER in i's key (n > 0, a lag) or |n| places LATER (n < 0, a lead), or -1 when
 * there is none; n == 0 gives the row itself, |n| >= 2^31 no row.  Source rows are numbered from lo: row r is reported as
 * r - lo for r >= lo and r - lo + nrows below lo, so a caller that puts other ranks' rows in front of its own ([B | A], lo =
 * rows of B) gets A's rows as [0, n_a) and B's after them -- the numbering qk_shift_gather reads.
 * edge (device uint8[nrows] or NULL): 1 for the rows among the last n (lag) / first |n| (lead) rows of their key: the rows a
 * later (earlier) rank needs.  time (device int64[nrows] or NULL): *status (device uint64, zeroed by the call) receives the
 * number of rows whose time is below that of the previous row of their key -- the order check, in the same pass.
 * Workspace: qk_shift_workspace_bytes(nrows) (the inverse permutation; unused without by).  Two launches with by, one without.
 * Errors: nrows > 2^31 - 1: QK_ERR_UNSUPPORTED; by / dest / seg not all given or all NULL, [lo, hi) outside the rows, null src
 * with hi > lo, time without status: QK_ERR_INVALID; workspace too small: QK_ERR_CAPACITY.
 * qk_shift_gather: out[c][i] for i < nrows, all shifted columns in one launch: src[i] in [0, n_a) reads a_cols[c] (n_a =
 * a_cols[0].length, the rank's own rows), src[i] in [n_a, n_a + n_b) reads b_cols[c] (the boundary rows of other ranks), -1
 * writes the fill value: the low dtype_size bytes of fill[c] (HOST uint64 array).  Validity: a_valid / b_valid are NULL or HOST
 * arrays of ncols device uint8 masks (an entry may be NULL = all valid); out_valid is NULL or a HOST array of ncols device
 * uint8[nrows] outputs (an entry may be NULL: not written), receiving fill_valid[c] (HOST uint8 array) for -1 and the source
 * row's validity otherwise.  Scalar QK_U8 / QK_I32 / QK_I64 / QK_F32 / QK_F64 columns, b_cols[c] of a_cols[c]'s dtype, at most
 * QK_MAX_COLS columns.  Errors: a vector column: QK_ERR_UNSUPPORTED; mismatched dtypes or lengths: QK_ERR_INVALID; a short
 * output: QK_ERR_CAPACITY. */
QK_API size_t qk_shift_workspace_bytes(int64_t nrows);
QK_API int qk_shift_plan(const int32_t* by, int32_t n_by, const int32_t* dest, const int64_t* seg, int64_t nrows, int64_t n,
                         int64_t lo, int64_t hi, int32_t* src, uint8_t* edge, const int64_t* time, uint64_t* status,
                         void* workspace, size_t ws_bytes, void* stream);
QK_API int qk_shift_gather(const qk_column* a_cols, const qk_column* b_cols, int32_t ncols, const uint8_t* const* a_valid,
                           const uint8_t* const* b_valid, const uint64_t* fill, const uint8_t* fill_valid, const int32_t* src,
                           int64_t nrows, int64_t n_b, qk_column* out, uint8_t* const* out_valid, void* stream);

/* ---- synthetic TPC-H-shaped / SIP-shaped columns, generated in HBM --------------------------
 * Bit-identical to oracle/tpch_gen.py (counter-based hash of (table, column, row)); lets bench.py hold
 * SF-100 (600 037 902 lineitem rows) resident without a 23 GB host copy.  `column` ids: see
 * quokka_b200/synth.py.  sizes[] = {n_orders, n_customer, n_supplier, n_part, n_symbols, gap}. */
QK_API int qk_synth_column(int32_t table, int32_t column, const int64_t* sizes, int64_t row_lo, int64_t nrows,
                    void* out, int32_t out_dtype, void* stream);

/* ---- Parquet column chunks decoded in HBM (SURVEY.md section 8(f).1) ----------------------------
 * Replaces the Arrow C++ Parquet reader behind `pq.ParquetFile(...).read_row_groups` /
 * `dataset.to_table` (pyquokka/dataset/unordered_readers.py:51,98-99): the raw bytes of the selected
 * column chunks are copied to the device as they lie in the file and decoded there.
 *
 * Step 1 (HOST, no device work): qk_parquet_walk_chunk parses the page headers of ONE column chunk
 * (Thrift compact protocol) and appends one qk_pq_run per PLAIN page / per RLE or bit-packed group of a
 * dictionary-coded page to `runs`.  Definition levels of OPTIONAL columns are checked to hold no null
 * (nulls are outside the hot path: QK_ERR_UNSUPPORTED) and skipped.  Supported: data pages V1 and V2,
 * PLAIN and RLE_DICTIONARY / PLAIN_DICTIONARY encodings, BOOLEAN / INT32 / INT64 / FLOAT / DOUBLE
 * values and BYTE_ARRAY dictionaries (strings stay dictionary codes), flat schemas, uncompressed
 * pages; anything else returns QK_ERR_UNSUPPORTED with the reason in qk_last_error().
 *   bytes[chunk_offset .. chunk_offset+chunk_bytes) = the column chunk (dictionary page first);
 *   payload offsets written to the runs are relative to `bytes`;  *dense (in/out) is the running count of
 *   values described so far (the output row of the next value);  *n_runs (in/out) the runs used so far;
 *   QK_ERR_CAPACITY leaves both untouched (grow `runs` and call again).
 * Step 2 (DEVICE): qk_parquet_decode writes value t of the run table to out[t]:
 *   PLAIN runs copy elem_bytes-wide elements (unaligned in the file) ; BOOL runs expand bits to uint8;
 *   RLE / PACKED runs look their index up in `dictionary` (elem_bytes-wide entries, entry dict_base+index;
 *   for string columns the "dictionary" is the int32 table mapping chunk-local to global codes; RLE-coded BOOLEAN
 *   pages (the V2 default) come out as RLE / PACKED runs over the two-entry uint8 dictionary {0, 1}).
 *   `runs` holds n_runs entries plus a sentinel with dense_start = n_values.  `bytes` must be 8-byte
 *   aligned and readable 16 bytes past n_bytes.  status (device int32, may be NULL) gets bit 0 set when an
 *   index falls outside the dictionary (corrupt input; that value decodes as entry 0). */
#define QK_PQ_RUN_PLAIN 0   /* payload = byte offset of fixed-width little-endian elements              */
#define QK_PQ_RUN_RLE 1     /* payload = the repeated dictionary index                                    */
#define QK_PQ_RUN_PACKED 2  /* payload = byte offset of LSB-first bit-packed indices, bit_width bits each */
#define QK_PQ_RUN_BOOL 3    /* payload = byte offset of PLAIN booleans, one bit per value                 */

#define QK_PQ_BOOLEAN 0     /* parquet.thrift Type */
#define QK_PQ_INT32 1
#define QK_PQ_INT64 2
#define QK_PQ_INT96 3
#define QK_PQ_FLOAT 4
#define QK_PQ_DOUBLE 5
#define QK_PQ_BYTE_ARRAY 6
#define QK_PQ_FIXED_LEN_BYTE_ARRAY 7

typedef struct qk_pq_run {
    int64_t dense_start;    /* index of the run's first value among all values of the table */
    int64_t payload;
    int32_t dict_base;      /* RLE / PACKED: offset of this chunk's entries in the dictionary array */
    uint8_t kind;           /* QK_PQ_RUN_* */
    uint8_t bit_width;      /* PACKED */
    uint16_t reserved;
} qk_pq_run;

typedef struct qk_pq_chunk_info {
    int64_t dict_offset;     /* byte offset (relative to `bytes`) of the dictionary page's PLAIN values, -1 = none */
    int64_t dict_bytes;
    int64_t n_values;        /* values of all data pages of the chunk */
    int32_t dict_num_values;
    int32_t n_data_pages;
} qk_pq_chunk_info;

QK_API int qk_parquet_walk_chunk(const uint8_t* bytes, int64_t chunk_offset, int64_t chunk_bytes, int64_t num_values,
                          int32_t physical_type, int32_t max_def_level, int32_t compression, int32_t dict_base,
                          qk_pq_run* runs, int64_t runs_cap, int64_t* n_runs, int64_t* dense, qk_pq_chunk_info* info);
QK_API int qk_parquet_decode(const uint8_t* bytes, int64_t n_bytes, const qk_pq_run* runs, int64_t n_runs,
                      int64_t n_values, const void* dictionary, int64_t dict_len, int32_t elem_bytes, void* out,
                      int32_t* status, void* stream);

/* ---- compressed chunks: pages inflated and walked on the device ------------------------------------
 * With a page codec the host cannot look inside the pages, so the work splits differently:
 *   qk_parquet_walk_pages (HOST) parses only the page headers into a page table and lays the uncompressed
 *     images of the pages out in a scratch buffer (8-byte aligned, *scratch_bytes in/out = bytes used so far);
 *   qk_parquet_inflate (DEVICE) writes each page's uncompressed image: a Snappy decoder, one warp per page (lane 0
 *     parses the element tags, all lanes move the literal / copy bytes), or a plain copy for stored pages.  V2 pages
 *     keep their level bytes uncompressed in front of the values; only the values are inflated;
 *   qk_parquet_page_runs (DEVICE) is the run-header walk of qk_parquet_walk_chunk, one thread per page over the
 *     inflated images: with run_offsets == NULL it only counts (pages[i].n_runs), else it writes page i's runs
 *     at runs[run_offsets[i] ...]; V1 definition levels are checked here (pages[i].status bit 1 = nulls);
 *   qk_parquet_decode then reads the scratch buffer as its `bytes`.
 *   ZSTD pages (the default of the Polars writer, apps/convert.py:5-19) are decoded by one thread per page (a
 *     sequential RFC 8878 frame decoder, csrc/zstd_core.h) and need a workspace of slots (decoding tables + a 128 KB
 *     literals buffer each), one per page in flight; the rest follow round-robin.  qk_parquet_inflate_workspace_bytes(n)
 *     sizes it for n such pages: min(n, 8 per SM) slots in whole CTAs of the inflate kernel, 0 for n <= 0.  A smaller
 *     `work` (at least one CTA's slots) puts fewer pages in flight.  GZIP pages use the same slots (their state is ~1.5 KB).
 * compression: QK_PQ_CODEC_* ; other codecs: QK_ERR_UNSUPPORTED. */
#define QK_PQ_CODEC_NONE 0
#define QK_PQ_CODEC_SNAPPY 1
#define QK_PQ_CODEC_ZSTD 2
#define QK_PQ_CODEC_GZIP 3     /* gzip members or a zlib stream around DEFLATE (csrc/deflate_core.h), one thread per page */
#define QK_PQ_PAGE_DATA_V1 0
#define QK_PQ_PAGE_DATA_V2 1
#define QK_PQ_PAGE_DICT 2

typedef struct qk_pq_page {
    int64_t src_offset;     /* first byte to inflate (V2: past the level bytes), relative to `bytes`        */
    int64_t dst_offset;     /* where the page's uncompressed image starts in the scratch buffer               */
    int64_t dense_start;    /* data page: row of its first value; dictionary page: its first entry's index   */
    int32_t src_bytes;      /* bytes to inflate from                                                          */
    int32_t dst_bytes;      /* size of the uncompressed image                                                 */
    int32_t num_values;
    int32_t dict_base;
    int32_t n_runs;         /* written by qk_parquet_page_runs                                                */
    uint8_t kind;           /* QK_PQ_PAGE_*                                                                   */
    uint8_t encoding;       /* parquet.thrift Encoding of the values                                          */
    uint8_t compressed;     /* QK_PQ_CODEC_* of the bytes to inflate (NONE = stored)                          */
    uint8_t max_def;        /* V1: definition levels precede the values when > 0                              */
    int32_t status;         /* written by the device: 1 malformed, 2 holds nulls, 4 unsupported encoding, 8 corrupt compressed stream, 16 no workspace */
    int32_t reserved;
} qk_pq_page;

QK_API int qk_parquet_walk_pages(const uint8_t* bytes, int64_t chunk_offset, int64_t chunk_bytes, int64_t num_values,
                          int32_t physical_type, int32_t max_def_level, int32_t compression, int32_t dict_base,
                          qk_pq_page* pages, int64_t pages_cap, int64_t* n_pages, int64_t* dense,
                          int64_t* scratch_bytes, qk_pq_chunk_info* info);
QK_API size_t qk_parquet_inflate_workspace_bytes(int64_t n_zstd_pages);
QK_API int qk_parquet_inflate(const uint8_t* bytes, int64_t n_bytes, qk_pq_page* pages, int64_t n_pages, uint8_t* scratch,
                       int64_t scratch_bytes, void* work, int64_t work_bytes, void* stream);
QK_API int qk_parquet_page_runs(const uint8_t* scratch, int64_t scratch_bytes, qk_pq_page* pages, int64_t n_pages,
                         int32_t physical_type, const int64_t* run_offsets, qk_pq_run* runs, int64_t runs_cap, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* QK_H */
