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
 *   - no nulls on the hot path: qk_column.validity must be NULL (QK_ERR_UNSUPPORTED otherwise);
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

#define QK_VERSION 100
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

typedef struct qk_column {
    const void* data;        /* device */
    const uint8_t* validity; /* must be NULL */
    int64_t length;
    int32_t dtype;           /* QK_U8 .. QK_F64 */
    int32_t reserved;
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
/* SM count of the current device (grids are sized in multiples of it) */
QK_API int qk_sm_count(void);

/* ---- K1: scan -> filter -> project --------------------------------------------------------
 * Replaces: Arrow `dataset.to_table(filter, columns)` (pyquokka/dataset/unordered_readers.py:98-99),
 * the edge predicate `x.filter(predicate)` / DuckDB `select * ... where` (pyquokka/core.py:156-170),
 * folded `with_columns` batch_funcs (pyquokka/datastream.py:1288-1296) and the projection
 * `payload[sorted(projection)]` (core.py:190-193), in one pass.
 * proj[i]: a single QK_OP_COL node copies the column verbatim in its own dtype (keys stay bit-exact);
 * anything else is evaluated in fp64 and written as QK_F64.
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
/* variant: 0 = auto, 1 = generic interpreter, 2 = fused template (vector LDG), 3 = fused template
 * with cp.async.bulk (TMA engine) staging of column tiles into shared memory. Returns
 * QK_ERR_UNSUPPORTED if a forced fused variant has no instantiation for the plan. */
/* name of the kernel variant the last qk_scan_filter_agg_dense call on this thread dispatched to */
QK_API const char* qk_last_variant(void);
/* launch shape of that kernel, e.g. "nt512v2s2" = 512 threads, 2 rows/thread/tile, 2 TMA stages */
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
/* Fused partition-scatter + shuffle over peer memory (replaces qk_scatter + the all-to-all of
 * TaskManager.push, pyquokka/core.py:276-376, when the ranks' mailboxes are mapped into each other's address
 * space): row i is stored directly into peer p's receive column at row peer_row_off[p] + (dest[i] -
 * part_offsets[p]), p being the partition dest[i] falls in.  peer_col_ptrs = HOST array [nparts][ncols] of device
 * pointers (peer-mapped, e.g. symmetric memory); peer_row_off = HOST array [nparts].  The caller separates
 * successive uses of a mailbox with a cross-rank barrier. */
#define QK_MAX_PEERS 16
QK_API int qk_scatter_peer(const qk_column* cols, int32_t ncols, const int32_t* dest, const int64_t* part_offsets, int32_t nparts,
                           const uint64_t* peer_col_ptrs, const int64_t* peer_row_off, void* stream);
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
 *   elements from byte offset src_byte_off[c] of the own mailbox, 16-byte aligned) into out[c]. */
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
/* out[c][i] = cols[c][idx[i]] for i < n_idx; idx == -1 writes 0 (left join / as-of "no match") */
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
 *     sequential RFC 8878 frame decoder, csrc/zstd_core.h) and need a workspace: `work` holds `work_bytes /
 *     qk_parquet_inflate_slot_bytes()` slots (decoding tables + a 128 KB literals buffer each); that many pages are in
 *     flight at once, the rest follow round-robin.  GZIP pages use the same slots (their state is ~1.5 KB).
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
QK_API size_t qk_parquet_inflate_slot_bytes(void);
QK_API int qk_parquet_inflate(const uint8_t* bytes, int64_t n_bytes, qk_pq_page* pages, int64_t n_pages, uint8_t* scratch,
                       int64_t scratch_bytes, void* work, int64_t work_bytes, void* stream);
QK_API int qk_parquet_page_runs(const uint8_t* scratch, int64_t scratch_bytes, qk_pq_page* pages, int64_t n_pages,
                         int32_t physical_type, const int64_t* run_offsets, qk_pq_run* runs, int64_t runs_cap, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* QK_H */
