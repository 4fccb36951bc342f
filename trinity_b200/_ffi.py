"""ctypes binding of include/trinity_b200.h.  Loading fails loudly when the native library is missing:
there is no Python/CPU fallback for any engine entry point."""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import numpy as np

_LIB_PATH = Path(__file__).resolve().parent / "libtrinity_b200.so"

# every symbol include/trinity_b200.h declares (tests check the library exports all of them)
EXPORTS = [
    "trn_builder_create", "trn_builder_destroy", "trn_builder_begin_term", "trn_builder_begin_document",
    "trn_builder_new_hit", "trn_builder_end_document", "trn_builder_end_term", "trn_builder_add_term",
    "trn_builder_set_google_skiplist_countdown", "trn_builder_index", "trn_builder_hits", "trn_builder_last_error",
    "trn_synth_build", "trn_synth_build_shard", "trn_synth_build_ex", "trn_builder_set_google_block", "trn_synth_destroy", "trn_synth_index", "trn_synth_hits", "trn_synth_terms", "trn_synth_sum_hits",
    "trn_synth_postings", "trn_synth_positions",
    "trn_directory_probe", "trn_directory_stats", "trn_directory_lookup", "trn_dict_create", "trn_dict_destroy", "trn_parse_query_dict", "trn_segment_open", "trn_segment_close", "trn_segment_info", "trn_segment_index", "trn_segment_terms",
    "trn_segment_masked", "trn_parse_query", "trn_query_truth_table", "trn_debug_compile", "trn_bm25_idf", "trn_bm25_score",
    "trn_create", "trn_destroy", "trn_last_error", "trn_set_stream", "trn_upload_index", "trn_set_masked_documents", "trn_index_info_get",
    "trn_exec_batch", "trn_exec_batch_device", "trn_last_topk_device", "trn_merge_topk", "trn_fetch_results", "trn_last_timings",
    "trn_decode_terms", "trn_result_for_each", "trn_result_decode", "trn_upload_hits", "trn_debug_positions", "trn_encode_google", "trn_debug_chunk_plan",
    "trn_debug_last_routes", "trn_debug_plan",
]

TERM_DTYPE = np.dtype([("documents", "<u4"), ("chunk_off", "<u4"), ("chunk_len", "<u4")])
QNODE_DTYPE = np.dtype([("kind", "u1"), ("nchildren", "u1"), ("first_child", "<u2"), ("term", "<u4"), ("weight", "<f8")])
STEP_DTYPE = np.dtype([("op", "u1"), ("mode", "u1"), ("dst", "u1"), ("src", "u1"), ("flags", "u1"), ("pad", "u1", (3,)), ("term", "<u4"), ("pad2", "<u4"), ("idf", "<f8")])
assert TERM_DTYPE.itemsize == 12 and QNODE_DTYPE.itemsize == 16 and STEP_DTYPE.itemsize == 24


class TrnTerm(C.Structure):
    _fields_ = [("documents", C.c_uint32), ("chunk_off", C.c_uint32), ("chunk_len", C.c_uint32)]


class TrnQuery(C.Structure):
    _fields_ = [("nodes", C.c_void_p), ("nnodes", C.c_uint32), ("root", C.c_uint32)]


class TrnIndexInfo(C.Structure):
    _fields_ = [("codec", C.c_int), ("nterms", C.c_uint32), ("max_docid", C.c_uint32), ("tile_docs", C.c_uint32),
                ("ntiles", C.c_uint32), ("block_docs", C.c_uint32), ("index_bytes", C.c_uint64), ("directory_bytes", C.c_uint64),
                ("total_blocks", C.c_uint64), ("total_postings", C.c_uint64)]


class TrnResult(C.Structure):
    _fields_ = [("nq", C.c_uint32), ("total", C.c_uint64), ("offsets", C.POINTER(C.c_uint64)),
                ("docids", C.POINTER(C.c_uint32)), ("scores", C.POINTER(C.c_float)),
                ("match_counts", C.POINTER(C.c_uint64)), ("postings_scanned", C.c_uint64),
                ("index_bytes_touched", C.c_uint64), ("kernel_launches", C.c_uint32), ("device_ms", C.c_float), ("exec_kernel_ms", C.c_float),
                ("words", C.POINTER(C.c_uint32)), ("total_words", C.c_uint64), ("item_desc", C.POINTER(C.c_uint32)), ("qitems", C.c_void_p)]


CONSIDER_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_uint32)  # trn_consider_fn


class TrnTimings(C.Structure):
    _fields_ = [(n, C.c_float) for n in ("host_compile_ms", "enqueue_ms", "chunk_wait_ms", "final_wait_ms", "kernel_ms", "total_ms", "chunks")]


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not _LIB_PATH.exists():
        raise ImportError(
            f"{_LIB_PATH} is missing: build it with `python -m trinity_b200.build` (needs nvcc). "
            "trinity_b200 has no CPU fallback; the CUDA extension is mandatory.")
    L = C.CDLL(str(_LIB_PATH))
    vp, u32, u64, i32 = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int
    P = C.POINTER

    def sig(name, res, *args):
        f = getattr(L, name)
        f.restype = res
        f.argtypes = list(args)

    sig("trn_builder_create", i32, i32, P(vp))
    sig("trn_builder_destroy", None, vp)
    sig("trn_builder_begin_term", i32, vp)
    sig("trn_builder_begin_document", i32, vp, u32)
    sig("trn_builder_new_hit", i32, vp, u32, vp, C.c_uint8)
    sig("trn_builder_end_document", i32, vp)
    sig("trn_builder_end_term", i32, vp, P(TrnTerm))
    sig("trn_builder_add_term", i32, vp, vp, vp, u32, vp, P(TrnTerm))
    sig("trn_builder_set_google_skiplist_countdown", i32, vp, u32)
    sig("trn_builder_index", i32, vp, P(vp), P(u64))
    sig("trn_builder_hits", i32, vp, P(vp), P(u64))
    sig("trn_builder_last_error", C.c_char_p, vp)
    sig("trn_synth_build", i32, i32, u32, u32, u32, u64, i32, i32, P(vp))
    sig("trn_synth_build_shard", i32, i32, u32, u32, u32, u64, i32, i32, u32, u32, P(vp))
    sig("trn_synth_build_ex", i32, i32, u32, u32, u32, u64, i32, i32, u32, u32, u32, u32, P(vp))
    sig("trn_builder_set_google_block", i32, vp, u32, u32)
    sig("trn_synth_destroy", None, vp)
    sig("trn_synth_index", i32, vp, P(vp), P(u64))
    sig("trn_synth_hits", i32, vp, P(vp), P(u64))
    sig("trn_synth_terms", i32, vp, P(vp), P(u32))
    sig("trn_synth_sum_hits", u64, vp)
    sig("trn_synth_postings", i32, u32, u32, u32, u64, vp, vp, u32, P(u32))
    sig("trn_synth_positions", i32, u32, u32, u32, u64, vp, u64, P(u64))
    sig("trn_directory_probe", i32, i32, vp, u64, P(TrnTerm), vp, vp, u32, P(u32), P(u32), C.c_char_p, C.c_size_t)
    sig("trn_directory_stats", i32, i32, vp, u64, vp, u32, i32, P(u64), P(u64), P(u64), C.c_char_p, C.c_size_t)
    sig("trn_directory_lookup", i32, i32, vp, u64, P(TrnTerm), vp, u32, vp, P(u32), P(u32), C.c_char_p, C.c_size_t)
    sig("trn_dict_create", i32, vp, u32, P(vp))
    sig("trn_dict_destroy", None, vp)
    sig("trn_parse_query_dict", i32, C.c_char_p, vp, vp, u32, P(u32), P(u32), C.c_char_p, C.c_size_t)
    sig("trn_segment_open", i32, C.c_char_p, P(vp), C.c_char_p, C.c_size_t)
    sig("trn_segment_close", None, vp)
    sig("trn_segment_info", i32, vp, P(i32), P(u32), P(u64), P(u64), P(u32), P(u64), P(u32), P(u64))
    sig("trn_segment_index", i32, vp, P(vp), P(u64))
    sig("trn_segment_terms", i32, vp, P(vp), P(vp), P(u32))
    sig("trn_segment_masked", i32, vp, P(vp), P(u64))
    sig("trn_debug_compile", i32, i32, vp, u64, vp, u32, vp, u32, u32, i32, vp, u32, P(u32), P(u32), P(u32), C.c_char_p, C.c_size_t)
    sig("trn_query_truth_table", i32, vp, u32, u32, P(u32), P(u32), P(u32), P(u32))
    sig("trn_parse_query", i32, C.c_char_p, vp, u32, vp, u32, P(u32), P(u32), C.c_char_p, C.c_size_t)
    sig("trn_bm25_idf", C.c_double, u32, u64)
    sig("trn_bm25_score", C.c_float, C.c_double, C.c_uint16)
    sig("trn_create", i32, i32, P(vp))
    sig("trn_destroy", None, vp)
    sig("trn_last_error", C.c_char_p, vp)
    sig("trn_set_stream", i32, vp, vp)
    sig("trn_upload_index", i32, vp, i32, vp, u64, vp, u32, u32)
    sig("trn_set_masked_documents", i32, vp, vp, u64)
    sig("trn_index_info_get", i32, vp, P(TrnIndexInfo))
    sig("trn_exec_batch", i32, vp, vp, u32, i32, u32, P(TrnResult))
    sig("trn_exec_batch_device", i32, vp, vp, u32, i32, u32, P(TrnResult))
    sig("trn_last_topk_device", i32, vp, P(vp), P(vp), P(vp))
    sig("trn_merge_topk", i32, vp, vp, vp, u32, u32, u32, vp, vp)
    sig("trn_fetch_results", i32, vp, P(TrnResult))
    sig("trn_upload_hits", i32, vp, vp, C.c_uint64, vp, C.c_uint64)
    sig("trn_debug_positions", i32, i32, vp, C.c_uint64, vp, C.c_uint64, vp, vp, u32, vp, vp, C.c_uint64, P(C.c_uint64), C.c_char_p, C.c_size_t)
    sig("trn_result_decode", i32, P(TrnResult), u32, vp, C.c_uint64, P(C.c_uint64))
    sig("trn_result_for_each", i32, P(TrnResult), u32, CONSIDER_FN, vp)
    sig("trn_last_timings", i32, vp, P(TrnTimings))
    sig("trn_decode_terms", i32, vp, vp, u32, i32, vp, vp, vp, P(C.c_float))
    sig("trn_debug_chunk_plan", i32, u32, i32, C.c_uint64, C.c_uint64, u32, C.c_uint64, i32, i32, C.c_double, C.c_double, C.c_uint64, C.c_uint64, i32, vp, u32,
        P(u32), P(i32))
    sig("trn_encode_google", i32, vp, vp, u32, vp, vp, vp, u32, u32, P(u32), vp, C.c_uint64, P(C.c_uint64), vp, P(C.c_float))
    sig("trn_debug_last_routes", i32, vp, vp, u32, P(u32))
    sig("trn_debug_plan", i32, i32, vp, u64, vp, u32, u32, vp, u32, i32, u32, vp, P(u32), C.c_char_p, C.c_size_t)
    _lib = L
    return L
