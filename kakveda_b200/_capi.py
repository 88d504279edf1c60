"""ctypes binding of libkakveda_b200.so (the C ABI declared in include/kakveda_b200.h).

There is no CPU implementation behind this module: if the shared object is missing the
import of any compute entry point raises, and every device call on a box without a GPU
returns KV_ERR_CUDA (raised as RuntimeError).
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

KV_OK, KV_ERR_INVALID, KV_ERR_CUDA, KV_ERR_EMPTY_VOCAB, KV_ERR_NOMEM, KV_ERR_NONASCII, KV_ERR_STATE = range(7)
KV_TEXT_RAW_ASCII, KV_TEXT_TOKENS, KV_TEXT_MIXED = 0, 1, 2

_LIB_PATH = Path(__file__).resolve().parent / "lib" / "libkakveda_b200.so"
_lib = None

c_i64p = C.POINTER(C.c_int64)
c_u32p = C.POINTER(C.c_uint32)
c_f64p = C.POINTER(C.c_double)
c_f32p = C.POINTER(C.c_float)

# name -> (restype, argtypes); every symbol include/kakveda_b200.h declares
SIGNATURES = {
    "kv_last_error": (C.c_char_p, []),
    "kv_version": (C.c_char_p, []),
    "kv_device_count": (C.c_int, []),
    "kv_vocab_create": (C.c_int, [C.POINTER(C.c_void_p)]),
    "kv_vocab_destroy": (None, [C.c_void_p]),
    "kv_vocab_size": (C.c_int64, [C.c_void_p]),
    "kv_vocab_export": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint64), C.c_int64]),
    "kv_vocab_import": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint64), C.c_int64]),
    "kv_featurize": (C.c_int, [C.c_void_p, C.c_char_p, c_i64p, C.c_int64, C.c_int, C.c_int, C.c_int,
                               C.POINTER(C.c_void_p), c_i64p]),
    "kv_csr_view": (C.c_int, [C.c_void_p, c_i64p, C.POINTER(c_i64p), C.POINTER(c_u32p), C.POINTER(c_u32p),
                              C.POINTER(c_f64p)]),
    "kv_csr_destroy": (None, [C.c_void_p]),
    "kv_vocab_mirror_create": (C.c_int, [C.c_int, C.POINTER(C.c_void_p)]),
    "kv_vocab_mirror_destroy": (None, [C.c_void_p]),
    "kv_vocab_mirror_sync": (C.c_int, [C.c_void_p, C.c_void_p, c_i64p]),
    "kv_featurize_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_char_p, c_i64p, C.c_int64, C.c_int, C.POINTER(C.c_void_p),
                                      c_i64p]),
    "kv_text_order": (C.c_int, [c_i64p, c_u32p, C.c_int64, C.POINTER(C.c_int32), C.c_int]),
    "kv_csr_gather_rows": (C.c_int, [c_i64p, c_u32p, c_u32p, C.c_int64, c_i64p, C.c_int64, c_i64p, c_u32p, c_u32p, C.c_int]),
    "kv_index_create": (C.c_int, [C.c_int, C.c_int64, C.POINTER(C.c_void_p)]),
    "kv_index_destroy": (None, [C.c_void_p]),
    "kv_index_append": (C.c_int, [C.c_void_p, c_i64p, c_u32p, c_u32p, C.c_int64]),
    "kv_index_set_mode": (C.c_int, [C.c_void_p, C.c_int]),
    "kv_jaccard_counts": (C.c_int, [C.c_void_p, c_i64p, c_u32p, c_f64p, C.c_int64, C.c_int, c_i64p,
                                    C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    "kv_index_set_global_df": (C.c_int, [C.c_void_p, c_u32p, C.c_int64, C.c_int64]),
    "kv_index_local_df": (C.c_int, [C.c_void_p, c_u32p, C.c_int64]),
    "kv_index_finalize": (C.c_int, [C.c_void_p, C.c_int64]),
    "kv_index_last_finalize_kind": (C.c_int, [C.c_void_p]),
    "kv_index_rows": (C.c_int64, [C.c_void_p]),
    "kv_score": (C.c_int, [C.c_void_p, c_u32p, c_u32p, C.c_int64, C.c_double, c_f64p]),
    "kv_topk": (C.c_int, [C.c_void_p, c_i64p, c_u32p, c_u32p, c_f64p, C.c_int64, C.c_int, c_f32p, c_i64p]),
    "kv_topk_device": (C.c_int, [C.c_void_p, c_i64p, c_u32p, c_u32p, c_f64p, C.c_int64, C.c_int, C.c_void_p,
                                 C.c_void_p]),
    "kv_query_upload": (C.c_int, [C.c_void_p, c_i64p, c_u32p, c_u32p, c_f64p, C.c_int64]),
    "kv_query_prepare_slice": (C.c_int, [C.c_void_p, c_i64p, c_u32p, c_u32p, c_f64p, C.c_int64, c_i64p, c_u32p, c_u32p,
                                         c_f64p, C.POINTER(C.c_int32), C.POINTER(C.c_uint8)]),
    "kv_query_upload_runs": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p),
                                       C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.POINTER(C.c_void_p),
                                       C.POINTER(C.c_void_p), c_i64p]),
    "kv_query_upload_text": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_char_p, c_i64p, C.c_int64, C.c_int, c_i64p]),
    "kv_index_last_prepare_ms": (C.c_int, [C.c_void_p, c_f32p]),
    "kv_debug_query_order": (C.c_int, [C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_uint8), C.c_int64]),
    "kv_topk_resident": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "kv_topk_resident_host": (C.c_int, [C.c_void_p, C.c_int, c_f32p, c_i64p]),
    "kv_topk_resident_seed": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "kv_index_raise_thresholds": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64]),
    "kv_topk_resident_finish": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "kv_query_set_exclusions": (C.c_int, [C.c_void_p, c_i64p, C.c_int64]),
    "kv_selfjoin_upload": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64]),
    "kv_index_set_row_labels": (C.c_int, [C.c_void_p, C.POINTER(C.c_int32), C.c_int64]),
    "kv_query_set_filter": (C.c_int, [C.c_void_p, C.POINTER(C.c_int32), C.c_int64]),
    "kv_index_set_row_groups": (C.c_int, [C.c_void_p, C.POINTER(C.c_int32), C.c_int64]),
    "kv_query_set_distinct": (C.c_int, [C.c_void_p, C.c_int]),
    "kv_index_delete_rows": (C.c_int, [C.c_void_p, c_i64p, C.c_int64]),
    "kv_index_live_rows": (C.c_int64, [C.c_void_p]),
    "kv_index_deleted_rows": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint8), C.c_int64]),
    "kv_rescore_pairs": (C.c_int, [C.c_void_p, c_i64p, c_u32p, c_u32p, c_f64p, C.c_int64, C.c_int, c_i64p, c_f64p]),
    "kv_range_resident": (C.c_int, [C.c_void_p, C.c_float, c_i64p]),
    "kv_range_fetch": (C.c_int, [C.c_void_p, c_i64p, c_i64p, c_f32p]),
    "kv_jaccard_range_resident": (C.c_int, [C.c_void_p, C.c_float, c_i64p]),
    "kv_jaccard_range_fetch": (C.c_int, [C.c_void_p, c_i64p, c_i64p, c_f32p, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    "kv_range_fetch_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "kv_jaccard_range_fetch_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "kv_cluster_topk": (C.c_int, [C.c_int64, C.c_int, c_i64p, c_f32p, C.c_float, c_i64p, c_i64p]),
    "kv_cluster_csr": (C.c_int, [C.c_int64, c_i64p, c_i64p, c_i64p, c_i64p]),
    "kv_cluster_csr_device": (C.c_int, [C.c_int, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, c_i64p]),
    "kv_debug_range_order": (C.c_int, [C.c_int, C.c_int, C.c_void_p, C.c_int64, C.c_int64, C.c_int64, c_i64p, c_i64p, c_f32p,
                                       C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    "kv_index_thresholds_export": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p]),
    "kv_index_thresholds_peers": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int64]),
    "kv_merge_topk_device": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int64, C.c_int, C.c_void_p,
                                       C.c_void_p]),
    "kv_merge_topk_device_on": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int64, C.c_int, C.c_int64, C.c_int64,
                                          C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]),
    "kv_index_last_timing": (C.c_int, [C.c_void_p, c_f32p]),
    "kv_index_last_kernel_ms": (C.c_int, [C.c_void_p, c_f32p]),
    "kv_index_last_score_ms": (C.c_int, [C.c_void_p, c_f32p]),
    "kv_debug_bound_numerators": (C.c_int, [C.c_void_p, C.c_int, c_f32p, C.POINTER(C.c_int32)]),
    "kv_debug_bound_codes": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_uint8), C.POINTER(C.c_int32),
                                       C.POINTER(C.c_int32), c_f32p, c_f32p, C.POINTER(C.c_int32)]),
    "kv_index_layout": (C.c_int, [C.c_void_p, c_i64p, c_i64p]),
    "kv_index_layout_save": (C.c_int, [C.c_void_p, C.c_char_p]),
    "kv_index_layout_load": (C.c_int, [C.c_void_p, C.c_char_p]),
    "kv_dense_create": (C.c_int, [C.c_int, C.c_int, C.c_int64, C.POINTER(C.c_void_p)]),
    "kv_dense_destroy": (None, [C.c_void_p]),
    "kv_dense_append": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint16), C.c_int64]),
    "kv_dense_finalize": (C.c_int, [C.c_void_p]),
    "kv_dense_rows": (C.c_int64, [C.c_void_p]),
    "kv_dense_topk": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint16), C.c_int64, C.c_int, c_f32p, c_i64p]),
    "kv_dense_append_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64]),
    "kv_dense_topk_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_void_p, C.c_void_p]),
    "kv_dense_selfjoin_device": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int, C.c_void_p, C.c_void_p]),
    "kv_dense_range": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint16), C.c_int64, C.c_float, c_i64p]),
    "kv_dense_range_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_float, C.c_int64, c_i64p]),
    "kv_dense_selfjoin_range": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_float, c_i64p]),
    "kv_dense_range_fetch": (C.c_int, [C.c_void_p, c_i64p, c_i64p, c_f32p]),
    "kv_dense_range_fetch_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "kv_dense_last_timing": (C.c_int, [C.c_void_p, c_f32p, c_i64p]),
    "kv_dense_delete_rows": (C.c_int, [C.c_void_p, c_i64p, C.c_int64]),
    "kv_dense_live_rows": (C.c_int64, [C.c_void_p]),
    "kv_dense_deleted_rows": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint8), C.c_int64]),
    "kv_dense_set_row_labels": (C.c_int, [C.c_void_p, C.POINTER(C.c_int32), C.c_int64]),
    "kv_dense_set_query_filter": (C.c_int, [C.c_void_p, C.POINTER(C.c_int32), C.c_int64]),
    "kv_dense_last_skipped": (C.c_int, [C.c_void_p, c_i64p, c_i64p]),
    "kv_hash_create": (C.c_int, [C.c_int, C.c_int64, C.POINTER(C.c_void_p)]),
    "kv_hash_destroy": (None, [C.c_void_p]),
    "kv_hash_append": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint64), C.c_int64]),
    "kv_hash_rows": (C.c_int64, [C.c_void_p]),
    "kv_hash_match": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint64), C.c_int64, C.c_int, c_i64p, c_i64p]),
    "kv_hash_last_timing": (C.c_int, [C.c_void_p, c_f32p, C.POINTER(C.c_int)]),
    "kv_synth_signatures": (C.c_int, [C.c_uint64, C.c_int64, C.c_int64, C.c_uint64, C.c_int64, C.c_char_p,
                                      C.c_int64, c_i64p]),
}


def lib_path() -> Path:
    return Path(os.environ.get("KAKVEDA_B200_LIB", _LIB_PATH))


def load():
    """Load the shared object once; raise (never fall back) when it is absent."""
    global _lib
    if _lib is not None:
        return _lib
    p = lib_path()
    if not p.exists():
        raise ImportError(
            f"{p} not found: build it with `python -m kakveda_b200.build` (nvcc, sm_90a). "
            "kakveda_b200 has no CPU fallback."
        )
    lib = C.CDLL(str(p))
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the .so does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def last_error() -> str:
    return load().kv_last_error().decode("utf-8", "replace")


def no_distinct(distinct: bool, what: str) -> None:
    """Distinct top-k (one row per group) is built for the TF-IDF ``GfkbIndex`` only."""
    if distinct:
        raise NotImplementedError(f"{what}: distinct top-k (kv_query_set_distinct) is only built for a single GfkbIndex")


def check(rc: int) -> None:
    if rc == KV_OK:
        return
    msg = last_error()
    if rc in (KV_ERR_INVALID, KV_ERR_EMPTY_VOCAB, KV_ERR_NONASCII):
        raise ValueError(msg)
    if rc == KV_ERR_NOMEM:
        raise MemoryError(msg)
    raise RuntimeError(msg)
