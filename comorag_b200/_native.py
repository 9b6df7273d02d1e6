"""ctypes binding of libcomorag_b200.so (the C ABI declared in include/comorag_b200.h).

There is no CPU fallback: if the library is missing or a call fails the error
is raised, never papered over.
"""
from __future__ import annotations

import ctypes as C
import threading
from pathlib import Path

LIB_PATH = Path(__file__).resolve().parent / "lib" / "libcomorag_b200.so"

CRAG_OK = 0


class NativeError(RuntimeError):
    """A libcomorag_b200 entry point returned a non-zero status."""


_c_i64p = C.POINTER(C.c_int64)
_c_f32p = C.POINTER(C.c_float)

# name -> (restype, argtypes); mirrors include/comorag_b200.h one to one.
SIGNATURES = {
    "crag_version": (C.c_int, []),
    "crag_last_error": (C.c_char_p, []),
    "crag_sm_count": (C.c_int, []),
    "crag_vmem_reserve": (C.c_int, [C.c_size_t, C.POINTER(C.c_uint64), C.POINTER(C.c_size_t)]),
    "crag_vmem_grow": (C.c_int, [C.c_uint64, C.c_size_t, C.c_size_t]),
    "crag_vmem_release": (C.c_int, [C.c_uint64, C.c_size_t, C.c_size_t]),
    "crag_search_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "crag_search_topk": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_int64, C.c_void_p, C.c_int,
                                   C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                                   C.c_void_p]),
    "crag_gemm_bf16": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64,
                                 C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "crag_pool_normalize": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                      C.c_int64, C.c_void_p]),
    # struct-taking entry points get their argtypes in comorag_b200/encoder.py
    "crag_encoder_workspace_bytes": (C.c_size_t, None),
    "crag_encoder_forward": (C.c_int, None),
    "crag_encoder_classify": (C.c_int, None),
    "crag_attention_varlen": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                        C.c_void_p]),
    "crag_attention_varlen_tc": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                           C.c_void_p, C.c_void_p]),
    "crag_layernorm": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_float, C.c_void_p,
                                 C.c_void_p]),
    "crag_search_topk_after": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_int64, C.c_void_p, C.c_int,
                                         C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.c_size_t, C.c_void_p]),
    "crag_search_scan": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_void_p, C.c_int, C.c_int, C.c_void_p,
                                   C.c_size_t, C.c_void_p]),
    "crag_search_finalize": (C.c_int, [C.c_void_p, C.c_size_t, C.c_int64, C.c_int, C.c_int, C.c_int64, C.c_void_p,
                                       C.c_void_p, C.c_void_p, C.c_void_p]),
    "crag_merge_topk_packed": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.c_void_p]),
    "crag_ivf_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int64, C.c_int]),
    "crag_ivf_search": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_void_p, C.c_void_p, C.c_int, C.c_int64,
                                  C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p,
                                  C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "crag_exchange_buffer_bytes": (C.c_size_t, [C.c_int]),
    "crag_search_finalize_exchange": (C.c_int, [C.c_void_p, C.c_size_t, C.c_int64, C.c_int, C.c_int, C.c_int64, C.c_void_p,
                                                C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                C.c_void_p, C.c_void_p]),
    "crag_ivf_assign": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                  C.c_void_p, C.c_size_t, C.c_void_p]),
    "crag_search_scores": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_void_p, C.c_int, C.c_void_p, C.c_int64,
                                     C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "crag_rank_workspace_bytes": (C.c_size_t, [C.c_int64]),
    "crag_rank_scores": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "crag_knn_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int]),
    "crag_knn_topk": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_int64, C.c_void_p, C.c_int, C.c_int,
                                C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "crag_knn_threshold": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_void_p, C.c_int, C.c_float, C.c_int,
                                     C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_size_t, C.c_void_p]),
    "crag_ppr_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int64]),
    "crag_ppr": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_float, C.c_int,
                           C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "crag_ppr_batch_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int64, C.c_int]),
    "crag_ppr_batch": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_int,
                                 C.c_float, C.c_int, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_size_t,
                                 C.c_void_p]),
    "crag_merge_topk": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                  C.c_void_p, C.c_void_p, C.c_void_p]),
    "crag_quantize_rows_i8": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p,
                                        C.c_void_p]),
    "crag_search_topk_i8": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_int64, C.c_void_p,
                                      C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_size_t, C.c_void_p]),
    "crag_rescore_topk": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_int64, C.c_void_p, C.c_int,
                                    C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "crag_binarize_rows": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p,
                                     C.c_void_p]),
    "crag_search_topk_b1": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_int64, C.c_void_p,
                                      C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_size_t, C.c_void_p]),
    "crag_knn_code_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int]),
    "crag_knn_topk_i8": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_int64, C.c_void_p,
                                   C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.c_size_t, C.c_void_p]),
    "crag_knn_topk_b1": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_int64, C.c_void_p,
                                   C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.c_size_t, C.c_void_p]),
    "crag_ivf_i8_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int64, C.c_int]),
    "crag_ivf_search_i8": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int64, C.c_void_p, C.c_int, C.c_int64,
                                     C.c_int64, C.c_void_p, C.c_void_p, C.c_int, C.c_int64, C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                     C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "crag_ivf_pq_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int64, C.c_int, C.c_int]),
    "crag_ivf_search_pq": (C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_void_p, C.c_void_p, C.c_int, C.c_int64,
                                     C.c_int64, C.c_void_p, C.c_void_p, C.c_int, C.c_int64, C.c_void_p, C.c_void_p,
                                     C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "crag_ivf_i8_wide_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int64, C.c_int, C.c_int64]),
    "crag_ivf_search_i8_wide": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int64, C.c_void_p, C.c_int, C.c_int64,
                                          C.c_int64, C.c_void_p, C.c_void_p, C.c_int, C.c_int64, C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                          C.c_int, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                                          C.c_void_p]),
    "crag_ivf_pq_wide_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int64, C.c_int, C.c_int64, C.c_int]),
    "crag_ivf_search_pq_wide": (C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_void_p, C.c_void_p, C.c_int, C.c_int64,
                                          C.c_int64, C.c_void_p, C.c_void_p, C.c_int, C.c_int64, C.c_void_p, C.c_void_p,
                                          C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int64,
                                          C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "crag_pq_encode": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_void_p, C.c_int, C.c_void_p, C.c_int64,
                                 C.c_void_p]),
    "crag_gmm_sweep_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int, C.c_int]),
    "crag_gmm_sweep": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                 C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                 C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "crag_umap_fuzzy_graph_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int]),
    "crag_umap_fuzzy_graph": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "crag_umap_spectral_init_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int]),
    "crag_umap_spectral_init": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_uint64,
                                          C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "crag_umap_optimize_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int]),
    "crag_umap_optimize": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int, C.c_float,
                                     C.c_float, C.c_int, C.c_int, C.c_int, C.c_uint64, C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
}

_lib = None
_lock = threading.Lock()


def load() -> C.CDLL:
    """Load (once) and return the shared library with typed entry points."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not LIB_PATH.exists():
            raise NativeError(
                f"{LIB_PATH} is missing: build it with `python -m comorag_b200.build` "
                "(or __graft_entry__.build()); this engine has no CPU fallback")
        lib = C.CDLL(str(LIB_PATH))
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)  # AttributeError if the .so is stale
            fn.restype = res
            if args is not None:
                fn.argtypes = args
        _lib = lib
        return lib


def check(rc: int, what: str) -> None:
    if rc != CRAG_OK:
        msg = load().crag_last_error().decode("utf-8", "replace")
        raise NativeError(f"{what} failed (rc={rc}): {msg}")


def ptr(t) -> int:
    """Device/host address of a torch tensor (0 for None)."""
    return 0 if t is None else t.data_ptr()
