"""ctypes binding of libqk.so (include/qk.h).  There is NO fallback: if the CUDA library is missing
or fails to load, every operator raises -- a silent CPU path would void the parity claims."""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libqk.so")

QK_U8, QK_I32, QK_I64, QK_F32, QK_F64, QK_F16 = 1, 2, 3, 4, 5, 6
KNN_MAX_DIM, KNN_MAX_K = 4096, 256
PATTERN_MAX_EVENTS, PATTERN_STATUS_WORDS, PATTERN_MAX_LINK_NODES = 8, 4, 128   # csrc/pattern.cu PT_MAX_NODES
(OP_COL, OP_CONST, OP_ADD, OP_SUB, OP_MUL, OP_DIV, OP_NEG, OP_LT, OP_LE, OP_GT, OP_GE, OP_EQ, OP_NE,
 OP_AND, OP_OR, OP_NOT, OP_CMP_COL_IMM, OP_CMP_COL_COL, OP_RINT, OP_IN_SET, OP_SELECT, OP_EXTRACT, OP_RANGE_COL_IMM) = range(1, 24)
CMP_LT, CMP_LE, CMP_GT, CMP_GE, CMP_EQ, CMP_NE = range(6)
AGG_SUM, AGG_MIN, AGG_MAX = 1, 2, 3
WIN_SUM, WIN_MIN, WIN_MAX, WIN_COUNT, WIN_AVG = 1, 2, 3, 4, 5
WIN_RUN_TUMBLING, WIN_RUN_SESSION = 1, 2
PART_MOD, PART_CODE = 0, 1
JOIN_INNER, JOIN_LEFT, JOIN_SEMI, JOIN_ANTI = 0, 1, 2, 3
ASOF_BACKWARD, ASOF_FORWARD, ASOF_NEAREST = 0, 1, 2
MAX_COLS, MAX_AGGS, MAX_PROJ = 16, 8, 16
MAX_EXPR_NODES, MAX_TOTAL_NODES, MAX_STACK = 48, 112, 8      # include/qk.h QK_MAX_EXPR_NODES / csrc/scan.cu MAX_NODES / QK_MAX_STACK
PQ_RUN_PLAIN, PQ_RUN_RLE, PQ_RUN_PACKED, PQ_RUN_BOOL = 0, 1, 2, 3
PQ_PAGE_DATA_V1, PQ_PAGE_DATA_V2, PQ_PAGE_DICT = 0, 1, 2
PQ_CODEC_NONE, PQ_CODEC_SNAPPY, PQ_CODEC_ZSTD, PQ_CODEC_GZIP = 0, 1, 2, 3
(PQ_BOOLEAN, PQ_INT32, PQ_INT64, PQ_INT96, PQ_FLOAT, PQ_DOUBLE, PQ_BYTE_ARRAY, PQ_FIXED_LEN_BYTE_ARRAY) = range(8)
ERR_INVALID, ERR_UNSUPPORTED, ERR_CUDA, ERR_CAPACITY = -1, -2, -3, -4


class QkError(RuntimeError):
    pass


class qk_column(C.Structure):
    _fields_ = [("data", C.c_void_p), ("validity", C.c_void_p), ("length", C.c_int64),
                ("dtype", C.c_int32), ("lanes", C.c_int32)]


class qk_expr_node(C.Structure):
    _fields_ = [("op", C.c_int32), ("a0", C.c_int32), ("a1", C.c_int32), ("reserved", C.c_int32),
                ("imm", C.c_double), ("imm_i", C.c_int64)]


class qk_expr(C.Structure):
    _fields_ = [("nodes", C.POINTER(qk_expr_node)), ("n_nodes", C.c_int32), ("reserved", C.c_int32)]


class qk_bloom(C.Structure):
    _fields_ = [("bits", C.c_void_p), ("words_per_part", C.c_int64), ("nparts", C.c_int32), ("key_proj", C.c_int32)]


MAX_PEERS, XCHG_MAX_BUFS, XCHG_META_WORDS, XCHG_CTRL_BYTES = 16, 48, 48, 16384


class qk_xchg(C.Structure):
    _fields_ = [("world", C.c_int32), ("rank", C.c_int32), ("ctrl", C.c_uint64 * MAX_PEERS), ("mailbox", C.c_uint64 * MAX_PEERS),
                ("mailbox_bytes", C.c_int64), ("timeout_ms", C.c_int64)]


class qk_hashagg_desc(C.Structure):
    _fields_ = [("capacity", C.c_int64), ("nkeys", C.c_int32), ("key_dtype", C.c_int32 * 4),
                ("nagg", C.c_int32), ("agg_op", C.c_int32 * MAX_AGGS)]


class qk_pq_run(C.Structure):
    _fields_ = [("dense_start", C.c_int64), ("payload", C.c_int64), ("dict_base", C.c_int32), ("kind", C.c_uint8),
                ("bit_width", C.c_uint8), ("reserved", C.c_uint16)]


class qk_pq_page(C.Structure):
    _fields_ = [("src_offset", C.c_int64), ("dst_offset", C.c_int64), ("dense_start", C.c_int64), ("src_bytes", C.c_int32),
                ("dst_bytes", C.c_int32), ("num_values", C.c_int32), ("dict_base", C.c_int32), ("n_runs", C.c_int32),
                ("kind", C.c_uint8), ("encoding", C.c_uint8), ("compressed", C.c_uint8), ("max_def", C.c_uint8),
                ("status", C.c_int32), ("reserved", C.c_int32)]


class qk_pq_chunk_info(C.Structure):
    _fields_ = [("dict_offset", C.c_int64), ("dict_bytes", C.c_int64), ("n_values", C.c_int64),
                ("dict_num_values", C.c_int32), ("n_data_pages", C.c_int32)]


_P = C.POINTER
_SIGNATURES = {
    "qk_last_error": (C.c_char_p, []),
    "qk_last_variant": (C.c_char_p, []),
    "qk_last_variant_config": (C.c_char_p, []),
    "qk_version": (C.c_int, []),
    "qk_launch_count": (C.c_int64, []),
    "qk_scan_workspace_bytes": (C.c_size_t, [C.c_int64]),
    "qk_scan_filter_project": (C.c_int, [_P(qk_column), C.c_int32, C.c_int64, _P(qk_expr), _P(qk_expr), C.c_int32,
                                         _P(qk_column), C.c_void_p, C.c_int32, C.c_void_p, C.c_size_t, C.c_void_p]),
    "qk_bloom_build": (C.c_int, [_P(qk_column), C.c_void_p, C.c_int64, C.c_int32, C.c_void_p]),
    "qk_scan_filter_project_sj": (C.c_int, [_P(qk_column), C.c_int32, C.c_int64, _P(qk_expr), _P(qk_expr), C.c_int32,
                                            _P(qk_column), C.c_void_p, _P(qk_bloom), C.c_void_p, C.c_size_t, C.c_void_p]),
    "qk_scan_agg_workspace_bytes": (C.c_size_t, [C.c_int32, C.c_int32]),
    "qk_scan_filter_agg_dense": (C.c_int, [_P(qk_column), C.c_int32, C.c_int64, _P(qk_expr), _P(C.c_int32), _P(C.c_int32),
                                           C.c_int32, _P(qk_expr), _P(C.c_int32), C.c_int32, C.c_void_p, C.c_void_p,
                                           C.c_void_p, C.c_size_t, C.c_int32, C.c_void_p]),
    "qk_hashagg_state_bytes": (C.c_size_t, [_P(qk_hashagg_desc)]),
    "qk_hashagg_init": (C.c_int, [_P(qk_hashagg_desc), C.c_void_p, C.c_void_p]),
    "qk_hashagg_update": (C.c_int, [_P(qk_hashagg_desc), C.c_void_p, _P(qk_column), _P(qk_column), C.c_int64,
                                    C.c_void_p, C.c_void_p]),
    "qk_hashagg_finalize": (C.c_int, [_P(qk_hashagg_desc), C.c_void_p, _P(qk_column), _P(qk_column), C.c_void_p,
                                      C.c_int64, C.c_void_p, C.c_void_p]),
    "qk_partition_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int32]),
    "qk_partition_plan": (C.c_int, [_P(qk_column), C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                    C.c_size_t, C.c_void_p]),
    "qk_scatter": (C.c_int, [_P(qk_column), C.c_int32, C.c_void_p, _P(qk_column), C.c_void_p]),
    "qk_xchg_ctrl_bytes": (C.c_size_t, []),
    "qk_xchg_meta": (C.c_int, [_P(qk_xchg), C.c_uint64, C.c_void_p, _P(C.c_int64), C.c_void_p, C.c_void_p, C.c_void_p]),
    "qk_xchg_push": (C.c_int, [_P(qk_xchg), C.c_uint64, _P(qk_column), C.c_int32, _P(C.c_int64), _P(C.c_int64), _P(C.c_int64), C.c_void_p]),
    "qk_xchg_push_scatter": (C.c_int, [_P(qk_xchg), C.c_uint64, _P(qk_column), C.c_int32, C.c_void_p, C.c_void_p, _P(C.c_int64), C.c_void_p]),
    "qk_xchg_recv": (C.c_int, [_P(qk_xchg), C.c_uint64, _P(C.c_int64), _P(qk_column), C.c_int32, C.c_void_p]),
    "qk_gather": (C.c_int, [_P(qk_column), C.c_int32, C.c_void_p, C.c_int64, _P(qk_column), C.c_void_p]),
    "qk_join_table_bytes": (C.c_size_t, [C.c_int64]),
    "qk_join_init": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p]),
    "qk_join_build": (C.c_int, [C.c_void_p, C.c_int64, _P(qk_column), C.c_int32, C.c_void_p, C.c_void_p]),
    "qk_join_probe": (C.c_int, [C.c_void_p, C.c_int64, _P(qk_column), C.c_int32, C.c_void_p, C.c_void_p,
                                C.c_int64, C.c_void_p, C.c_void_p]),
    "qk_join_probe_ordered_workspace_bytes": (C.c_size_t, [C.c_int64]),
    "qk_join_probe_ordered": (C.c_int, [C.c_void_p, C.c_int64, _P(qk_column), C.c_int32, C.c_void_p, C.c_void_p,
                                        C.c_int64, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "qk_join_place_workspace_bytes": (C.c_size_t, [C.c_int64]),
    "qk_join_place": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "qk_asof_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int32]),
    "qk_asof_backward": (C.c_int, [_P(qk_column), _P(qk_column), _P(qk_column), _P(qk_column), C.c_int32,
                                   C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "qk_asof_merge_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int64, C.c_int32]),
    "qk_asof_merge": (C.c_int, [_P(qk_column), _P(qk_column), _P(qk_column), _P(qk_column), C.c_int32, C.c_void_p, C.c_int32,
                                C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "qk_asof_join_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int64, C.c_int32, C.c_int32]),
    "qk_asof_join": (C.c_int, [_P(qk_column), _P(qk_column), _P(qk_column), _P(qk_column), C.c_int32, C.c_int32, C.c_int64,
                               C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                               C.c_size_t, C.c_void_p]),
    "qk_asof_search_join": (C.c_int, [_P(qk_column), _P(qk_column), _P(qk_column), _P(qk_column), C.c_int32, C.c_int32, C.c_int64,
                                      C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "qk_window_sliding": (C.c_int, [_P(qk_column), _P(qk_column), C.c_void_p, C.c_int32, C.c_int64, _P(qk_column), C.c_int32, _P(C.c_int32),
                                    _P(C.c_int32), C.c_int32, _P(qk_column), C.c_void_p]),
    "qk_window_hop_expand": (C.c_int, [_P(qk_column), _P(qk_column), C.c_void_p, C.c_int32, C.c_int64, C.c_int64, C.c_int32, C.c_void_p,
                                       C.c_void_p, C.c_void_p, C.c_void_p]),
    "qk_window_session_workspace_bytes": (C.c_size_t, [C.c_int64]),
    "qk_window_session_ids": (C.c_int, [_P(qk_column), _P(qk_column), C.c_int64, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "qk_window_running_workspace_bytes": (C.c_size_t, [C.c_int64]),
    "qk_window_running": (C.c_int, [_P(qk_column), _P(qk_column), C.c_void_p, C.c_int32, C.c_int32, C.c_int64, _P(qk_column), C.c_int32,
                                    _P(C.c_int32), _P(C.c_int32), C.c_int32, _P(qk_column), C.c_void_p, C.c_size_t, C.c_void_p]),
    "qk_topk_workspace_bytes": (C.c_size_t, [C.c_int64]),
    "qk_topk_candidates": (C.c_int, [_P(qk_column), C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_size_t, C.c_void_p]),
    "qk_gram_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int32]),
    "qk_gram": (C.c_int, [_P(qk_column), C.c_int32, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p,
                          C.c_size_t, C.c_void_p]),
    "qk_gram_last_plan": (C.c_char_p, []),
    "qk_qsketch_workspace_bytes": (C.c_size_t, [C.c_int32]),
    "qk_qsketch_update": (C.c_int, [_P(qk_column), C.c_void_p, C.c_int32, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p,
                                    C.c_int64, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "qk_qsketch_merge": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p,
                                   C.c_void_p]),
    "qk_knn_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int32, C.c_int32, C.c_int32]),
    "qk_knn_topk": (C.c_int, [_P(qk_column), C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                              C.c_void_p]),
    "qk_knn_merge": (C.c_int, [C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                               C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "qk_pattern_search": (C.c_int, [_P(qk_column), _P(qk_column), C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32,
                                    C.c_int64, _P(qk_column), C.c_int32, _P(qk_expr), C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p,
                                    C.c_void_p]),
    "qk_sort_workspace_bytes": (C.c_size_t, [C.c_int64]),
    "qk_sort_perm": (C.c_int, [_P(qk_column), C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p,
                               C.c_size_t, C.c_void_p]),
    "qk_sort_last_plan": (C.c_char_p, []),
    "qk_shift_workspace_bytes": (C.c_size_t, [C.c_int64]),
    "qk_shift_plan": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_int64,
                                C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "qk_shift_gather": (C.c_int, [_P(qk_column), _P(qk_column), C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                  C.c_void_p, C.c_int64, C.c_int64, _P(qk_column), C.c_void_p, C.c_void_p]),
    "qk_synth_column": (C.c_int, [C.c_int32, C.c_int32, _P(C.c_int64), C.c_int64, C.c_int64, C.c_void_p,
                                  C.c_int32, C.c_void_p]),
    "qk_parquet_walk_chunk": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                        C.c_void_p, C.c_int64, _P(C.c_int64), _P(C.c_int64), _P(qk_pq_chunk_info)]),
    "qk_parquet_walk_pages": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                        C.c_void_p, C.c_int64, _P(C.c_int64), _P(C.c_int64), _P(C.c_int64), _P(qk_pq_chunk_info)]),
    "qk_parquet_inflate_workspace_bytes": (C.c_size_t, [C.c_int64]),
    "qk_parquet_inflate": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64,
                                     C.c_void_p]),
    "qk_parquet_page_runs": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p, C.c_int64,
                                       C.c_void_p]),
    "qk_parquet_decode": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_int64, C.c_int32,
                                    C.c_void_p, C.c_void_p, C.c_void_p]),
}
EXPORTS = sorted(_SIGNATURES)

_lib = None


def lib():
    """The loaded library; raises QkError (never falls back) when it is absent."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise QkError(f"{LIB_PATH} is missing: build it with `python -m quokka_b200.build` "
                          "(quokka_b200 has no CPU fallback)")
        try:
            l = C.CDLL(LIB_PATH)
        except OSError as e:
            raise QkError(f"cannot load {LIB_PATH}: {e}") from e
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(l, name)
            fn.restype = res
            fn.argtypes = args
        _lib = l
    return _lib


def check(rc: int, what: str = ""):
    if rc != 0:
        msg = lib().qk_last_error().decode(errors="replace")
        raise QkError(f"{what or 'libqk'} failed ({rc}): {msg}")
