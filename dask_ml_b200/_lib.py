"""ctypes binding of the C-ABI shared library ``libbkm_b200.so`` (include/bkm_b200.h).

The library is built in-tree by ``__graft_entry__.build()`` / ``make -C dask_ml_b200/csrc``.
There is no CPU fallback: if the library is missing, or a call returns a non-zero status,
a ``RuntimeError`` is raised.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libbkm_b200.so")

BKM_F32 = 0
BKM_F64 = 1
BKM_BF16 = 2

# further operand types of bkm_metric_chunk
BKM_M_F16 = 3
BKM_M_I32 = 4
BKM_M_I64 = 5
BKM_M_U8 = 6
METRIC_EQ = 0
METRIC_ERR = 1
METRIC_LOGLOSS = 2
ENCODE_CODES = 0
ENCODE_DENSE = 1
ENCODE_CSR = 2
ENCODE_KEEP = 8
TEXT_NORM = {None: 0, "l1": 1, "l2": 2}

NB_JLL = 0
NB_LOG_PROBA = 1
NB_PROBA = 2

FLAG_FORCE_SIMT = 1
FLAG_FORCE_TC = 2
FLAG_NO_RECHECK = 4
FLAG_FIRST_CHUNK = 8
FLAG_COUNTS_F64 = 16
FLAG_FULL_PROBE = 32

_c_void_p = ctypes.c_void_p
_i64 = ctypes.c_int64
_u64 = ctypes.c_uint64
_int = ctypes.c_int
_dbl = ctypes.c_double
_szp = ctypes.POINTER(ctypes.c_size_t)


class SgdParams(ctypes.Structure):
    """``bkm_sgd_params`` of include/bkm_b200.h."""

    _fields_ = [("loss", ctypes.c_int), ("penalty", ctypes.c_int), ("learning_rate", ctypes.c_int),
                ("fit_intercept", ctypes.c_int), ("epsilon", ctypes.c_double), ("alpha", ctypes.c_double),
                ("l1_ratio", ctypes.c_double), ("eta0", ctypes.c_double), ("optimal_init", ctypes.c_double),
                ("t0", ctypes.c_double), ("intercept_decay", ctypes.c_double), ("average", ctypes.c_double)]


_sgdp = ctypes.POINTER(SgdParams)

# name -> (restype, argtypes); mirrors include/bkm_b200.h one to one
SIGNATURES = {
    "bkm_version": (_int, []),
    "bkm_error_string": (ctypes.c_char_p, [_int]),
    "bkm_device_info": (_int, [_int, ctypes.POINTER(_int), ctypes.POINTER(_int), ctypes.POINTER(_int)]),
    "bkm_kernel_family": (_int, [_int, _int, _int, _int]),
    "bkm_centers_pack_bytes": (_int, [_int, _int, _int, _szp]),
    "bkm_pack_centers": (_int, [_c_void_p, _int, _int, _int, _c_void_p, ctypes.c_size_t, _c_void_p]),
    "bkm_workspace_bytes": (_int, [_i64, _int, _int, _int, _szp]),
    "bkm_lloyd_chunk": (_int, [_c_void_p, _i64, _int, _i64, _int, _c_void_p, _int, _c_void_p, _c_void_p,
                               _c_void_p, _c_void_p, _c_void_p, _c_void_p, ctypes.c_size_t, _int, _c_void_p, _c_void_p]),
    "bkm_min_fold_chunk": (_int, [_c_void_p, _c_void_p, _i64, _int, _c_void_p, _c_void_p]),
    "bkm_make_blobs_chunk": (_int, [_c_void_p, _c_void_p, _i64, _int, _i64, _int, _c_void_p, _c_void_p, _int, _u64,
                                    _c_void_p]),
    "bkm_make_glm_chunk": (_int, [_c_void_p, _c_void_p, _i64, _int, _i64, _int, _i64, _int, _c_void_p, _int, _int,
                                  _dbl, _dbl, _u64, _c_void_p, _c_void_p]),
    "bkm_loop_state_bytes": (_int, [_szp]),
    "bkm_loop_reset": (_int, [_c_void_p, _dbl, _c_void_p, _int, _c_void_p]),
    "bkm_finalize_step": (_int, [_c_void_p, _c_void_p, _c_void_p, _c_void_p, _int, _int, _int, _c_void_p,
                                 ctypes.c_size_t, _c_void_p]),
    "bkm_minibatch_step": (_int, [_c_void_p, _c_void_p, _c_void_p, _c_void_p, _c_void_p, _int, _int, _int, _c_void_p,
                                  ctypes.c_size_t, _c_void_p]),
    "bkm_assign_chunk": (_int, [_c_void_p, _i64, _int, _i64, _int, _c_void_p, _int, _c_void_p, _c_void_p,
                                _int, _c_void_p, _c_void_p, ctypes.c_size_t, _int, _c_void_p]),
    "bkm_sample_chunk": (_int, [_c_void_p, _i64, _int, _dbl, _u64, _u64, _c_void_p, _i64, _c_void_p, _c_void_p]),
    "bkm_transform_chunk": (_int, [_c_void_p, _i64, _int, _i64, _int, _c_void_p, _int, _c_void_p, _i64, _int, _dbl, _int,
                                   _c_void_p]),
    "bkm_kernel_colsum_chunk": (_int, [_c_void_p, _i64, _int, _i64, _int, _c_void_p, _int, _dbl, _c_void_p, _c_void_p,
                                       ctypes.c_size_t, _int, _c_void_p]),
    "bkm_nystrom_embed_chunk": (_int, [_c_void_p, _i64, _int, _i64, _int, _c_void_p, _int, _dbl, _c_void_p, _int,
                                       _c_void_p, _i64, _int, _c_void_p]),
    "bkm_gram_workspace_bytes": (_int, [_i64, _int, _szp]),
    "bkm_gram_chunk": (_int, [_c_void_p, _i64, _int, _i64, _int, _c_void_p, _c_void_p, _c_void_p, _c_void_p,
                              ctypes.c_size_t, _int, _c_void_p]),
    "bkm_project_chunk": (_int, [_c_void_p, _i64, _int, _i64, _int, _c_void_p, _c_void_p, _int, _c_void_p, _i64, _int,
                                 _c_void_p, _i64, _int, _c_void_p]),
    "bkm_nb_workspace_bytes": (_int, [_i64, _int, _int, _szp]),
    "bkm_class_moments_chunk": (_int, [_c_void_p, _i64, _int, _i64, _int, _c_void_p, _int, _int, _c_void_p, _c_void_p,
                                       _c_void_p, _c_void_p, ctypes.c_size_t, _int, _c_void_p]),
    "bkm_nb_jll_chunk": (_int, [_c_void_p, _i64, _int, _i64, _int, _c_void_p, _c_void_p, _c_void_p, _int, _c_void_p,
                                _c_void_p, _i64, _int, _c_void_p, _int, _c_void_p]),
    "bkm_class_counts_chunk": (_int, [_c_void_p, _i64, _int, _i64, _int, _c_void_p, _int, _c_void_p, _int, _dbl,
                                      _c_void_p, _c_void_p, _c_void_p, ctypes.c_size_t, _int, _c_void_p]),
    "bkm_csc_class_counts_chunk": (_int, [_c_void_p, _c_void_p, _c_void_p, _int, _int, _i64, _c_void_p, _c_void_p, _int,
                                          _c_void_p, _int, _dbl, _c_void_p, _c_void_p, ctypes.c_size_t, _int,
                                          _c_void_p]),
    "bkm_nb_linear_jll_chunk": (_int, [_c_void_p, _i64, _int, _i64, _int, _int, _dbl, _c_void_p, _c_void_p, _int,
                                       _c_void_p, _c_void_p, _i64, _int, _int, _c_void_p]),
    "bkm_nb_csr_jll_chunk": (_int, [_c_void_p, _c_void_p, _c_void_p, _int, _i64, _int, _i64, _int, _dbl, _c_void_p,
                                    _c_void_p, _int, _c_void_p, _c_void_p, _i64, _int, _int, _c_void_p]),
    "bkm_glm_workspace_bytes": (_int, [_i64, _int, _szp]),
    "bkm_glm_pass_chunk": (_int, [_c_void_p, _i64, _int, _i64, _int, _c_void_p, _c_void_p, _int, _int, _c_void_p,
                                  _c_void_p, _c_void_p, _c_void_p, _c_void_p, ctypes.c_size_t, _int, _c_void_p]),
    "bkm_gram_weighted_chunk": (_int, [_c_void_p, _i64, _int, _i64, _int, _c_void_p, _c_void_p, _c_void_p,
                                       ctypes.c_size_t, _int, _c_void_p]),
    "bkm_glm_csr_workspace_bytes": (_int, [_i64, _szp]),
    "bkm_glm_csr_pass_chunk": (_int, [_c_void_p, _c_void_p, _c_void_p, _int, _i64, _int, _i64, _c_void_p, _c_void_p,
                                      _int, _int, _c_void_p, _c_void_p, _c_void_p, _c_void_p, _c_void_p, _c_void_p,
                                      ctypes.c_size_t, _int, _c_void_p]),
    "bkm_csr_transpose_workspace_bytes": (_int, [_i64, _int, _i64, _szp, _szp]),
    "bkm_csr_transpose_chunk": (_int, [_c_void_p, _c_void_p, _c_void_p, _int, _i64, _int, _i64, _c_void_p, _c_void_p,
                                       _c_void_p, _c_void_p, ctypes.c_size_t, _c_void_p, ctypes.c_size_t, _c_void_p]),
    "bkm_csc_matvec_workspace_bytes": (_int, [_int, _i64, _szp]),
    "bkm_csc_matvec_chunk": (_int, [_c_void_p, _c_void_p, _c_void_p, _int, _int, _i64, _c_void_p, _c_void_p,
                                    _c_void_p, _c_void_p, _c_void_p, _c_void_p, ctypes.c_size_t, _int, _c_void_p]),
    "bkm_gram_weighted_csr_workspace_bytes": (_int, [_int, _i64, _szp]),
    "bkm_gram_weighted_csr_chunk": (_int, [_c_void_p, _c_void_p, _c_void_p, _int, _i64, _int, _i64, _c_void_p,
                                           _c_void_p, _c_void_p, _c_void_p, _i64, _c_void_p, _c_void_p, _c_void_p,
                                           ctypes.c_size_t, _int, _c_void_p]),
    "bkm_csr_panel_chunk": (_int, [_c_void_p, _c_void_p, _c_void_p, _int, _i64, _int, _i64, _c_void_p, _int, _c_void_p,
                                   _i64, _int, _c_void_p, _i64, _c_void_p]),
    "bkm_csc_panel_workspace_bytes": (_int, [_int, _i64, _int, _szp]),
    "bkm_csc_panel_chunk": (_int, [_c_void_p, _c_void_p, _c_void_p, _int, _int, _i64, _c_void_p, _c_void_p, _int,
                                   _c_void_p, _c_void_p, ctypes.c_size_t, _int, _c_void_p]),
    "bkm_sparse_pack_workspace_bytes": (_int, [_int, _int, _szp]),
    "bkm_sparse_pack_centers": (_int, [_c_void_p, _int, _int, _c_void_p, _c_void_p, ctypes.c_size_t, _c_void_p]),
    "bkm_csr_assign_workspace_bytes": (_int, [_i64, _int, _szp]),
    "bkm_csr_assign_chunk": (_int, [_c_void_p, _c_void_p, _c_void_p, _int, _i64, _int, _i64, _c_void_p, _int, _int,
                                    _c_void_p, _c_void_p, _int, _c_void_p, _c_void_p, _c_void_p, _i64, _int, _c_void_p,
                                    ctypes.c_size_t, _int, _c_void_p, _c_void_p]),
    "bkm_csc_label_sums_workspace_bytes": (_int, [_int, _i64, _int, _szp]),
    "bkm_csc_label_sums_chunk": (_int, [_c_void_p, _c_void_p, _c_void_p, _int, _int, _i64, _c_void_p, _c_void_p, _int,
                                        _c_void_p, _c_void_p, ctypes.c_size_t, _int, _c_void_p, _c_void_p]),
    "bkm_sparse_finalize_step": (_int, [_c_void_p, _c_void_p, _c_void_p, _c_void_p, _int, _int, _c_void_p,
                                        ctypes.c_size_t, _c_void_p]),
    "bkm_csr_kernel_colsum_workspace_bytes": (_int, [_i64, _int, _szp]),
    "bkm_csr_kernel_colsum_chunk": (_int, [_c_void_p, _c_void_p, _c_void_p, _int, _i64, _int, _i64, _c_void_p, _int,
                                           _dbl, _c_void_p, _c_void_p, ctypes.c_size_t, _int, _c_void_p]),
    "bkm_csr_nystrom_embed_chunk": (_int, [_c_void_p, _c_void_p, _c_void_p, _int, _i64, _int, _i64, _c_void_p, _int,
                                           _dbl, _c_void_p, _int, _c_void_p, _i64, _int, _int, _c_void_p]),
    "bkm_sparse_minibatch_step": (_int, [_c_void_p, _c_void_p, _c_void_p, _c_void_p, _c_void_p, _int, _int, _c_void_p,
                                         ctypes.c_size_t, _c_void_p]),
    "bkm_sgd_order": (_int, [_i64, ctypes.c_uint32, _c_void_p]),
    "bkm_sgd_block": (_int, [_c_void_p, _i64, _int, _i64, _int, _c_void_p, _c_void_p, _c_void_p, _c_void_p, _c_void_p,
                             _int, _sgdp, _c_void_p, _c_void_p, _c_void_p, _c_void_p, _c_void_p]),
    "bkm_sgd_csr_block": (_int, [_c_void_p, _c_void_p, _c_void_p, _int, _i64, _int, _i64, _c_void_p, _c_void_p,
                                 _c_void_p, _c_void_p, _c_void_p, _int, _sgdp, _c_void_p, _c_void_p, _c_void_p,
                                 _c_void_p, _c_void_p]),
    "bkm_colstats_workspace_bytes": (_int, [_i64, _int, _szp]),
    "bkm_colstats_chunk": (_int, [_c_void_p, _i64, _int, _i64, _int, _c_void_p, _c_void_p, _c_void_p, _c_void_p,
                                  ctypes.c_size_t, _int, _c_void_p]),
    "bkm_radix_state_bytes": (_int, [_int, _int, _szp]),
    "bkm_radix_hist_chunk": (_int, [_c_void_p, _i64, _int, _i64, _int, _c_void_p, _int, _int, _c_void_p, _int,
                                    _c_void_p]),
    "bkm_radix_select_step": (_int, [_c_void_p, _c_void_p, _int, _int, _int, _int, _c_void_p, _c_void_p]),
    "bkm_affine_chunk": (_int, [_c_void_p, _i64, _int, _i64, _int, _c_void_p, _c_void_p, _int, _int, _c_void_p, _i64,
                                _int, _c_void_p]),
    "bkm_quantile_state_bytes": (_int, [_int, _int, _szp]),
    "bkm_quantile_hist_chunk": (_int, [_c_void_p, _i64, _int, _i64, _int, _c_void_p, _int, _int, _c_void_p, _int,
                                       _c_void_p]),
    "bkm_quantile_select_step": (_int, [_c_void_p, _c_void_p, _int, _int, _int, _int, _c_void_p, _c_void_p]),
    "bkm_quantile_transform_chunk": (_int, [_c_void_p, _i64, _int, _i64, _int, _c_void_p, _c_void_p, _int, _int, _int,
                                            _dbl, _dbl, _c_void_p, _i64, _c_void_p]),
    "bkm_impute_stats_workspace_bytes": (_int, [_i64, _int, _szp]),
    "bkm_impute_stats_chunk": (_int, [_c_void_p, _i64, _int, _i64, _int, _int, _dbl, _c_void_p, _c_void_p, _c_void_p,
                                      ctypes.c_size_t, _int, _c_void_p]),
    "bkm_quantile_hist_masked_chunk": (_int, [_c_void_p, _i64, _int, _i64, _int, _dbl, _c_void_p, _int, _int,
                                              _c_void_p, _int, _c_void_p]),
    "bkm_mode_count_chunk": (_int, [_c_void_p, _i64, _int, _i64, _int, _int, _dbl, _c_void_p, _c_void_p, _c_void_p,
                                    _i64, _int, _c_void_p]),
    "bkm_mode_best_workspace_bytes": (_int, [_int, _i64, _szp]),
    "bkm_mode_best": (_int, [_c_void_p, _c_void_p, _c_void_p, _int, _i64, _c_void_p, _c_void_p, _c_void_p, _c_void_p,
                             ctypes.c_size_t, _c_void_p]),
    "bkm_mode_compact": (_int, [_c_void_p, _c_void_p, _c_void_p, _int, _c_void_p, _c_void_p, _c_void_p]),
    "bkm_mode_merge": (_int, [_c_void_p, _i64, _c_void_p, _c_void_p, _c_void_p, _int, _i64, _c_void_p]),
    "bkm_impute_chunk": (_int, [_c_void_p, _i64, _int, _i64, _int, _int, _dbl, _c_void_p, _c_void_p, _int, _int, _int,
                                _int, _c_void_p, _i64, _int, _c_void_p, _c_void_p]),
    "bkm_distinct_chunk": (_int, [_c_void_p, _i64, _int, _i64, _int, _c_void_p, _c_void_p, _c_void_p, _i64, _c_void_p,
                                  _int, _c_void_p]),
    "bkm_encode_chunk": (_int, [_c_void_p, _i64, _int, _i64, _int, _c_void_p, _c_void_p, _i64, _int, _c_void_p, _i64,
                                _int, _c_void_p, _c_void_p, _c_void_p]),
    "bkm_decode_chunk": (_int, [_c_void_p, _i64, _int, _i64, _int, _c_void_p, _c_void_p, _int, _c_void_p, _i64,
                                _c_void_p, _c_void_p]),
    "bkm_text_workspace_bytes": (_int, [_i64, _i64, _i64, _szp]),
    "bkm_text_tokens_chunk": (_int, [_c_void_p, _i64, _c_void_p, _i64, _int, _int, _c_void_p, _i64, _c_void_p,
                                     _c_void_p, _c_void_p, _c_void_p, ctypes.c_size_t, _c_void_p]),
    "bkm_text_hash_chunk": (_int, [_c_void_p, _i64, _c_void_p, _c_void_p, _c_void_p, _i64, _i64, _i64, _int, _int,
                                   _int, _i64, _int, _int, _int, _int, _c_void_p, _c_void_p, _c_void_p, _c_void_p,
                                   _c_void_p, ctypes.c_size_t, _c_void_p]),
    "bkm_text_write_chunk": (_int, [_c_void_p, _c_void_p, _c_void_p, _c_void_p, _i64, _int, _c_void_p, _c_void_p,
                                    _int, _c_void_p]),
    "bkm_split_indices_chunk": (_int, [_u64, _i64, _i64, _i64, _i64, _c_void_p, _c_void_p]),
    "bkm_gather_rows_chunk": (_int, [_c_void_p, _i64, _i64, _i64, _c_void_p, _i64, _i64, _c_void_p, _i64, _c_void_p]),
    "bkm_metric_workspace_bytes": (_int, [_i64, _int, _int, _szp]),
    "bkm_metric_chunk": (_int, [_c_void_p, _int, _c_void_p, _int, _c_void_p, _i64, _int, _int, _c_void_p, _dbl,
                                _c_void_p, _c_void_p, ctypes.c_size_t, _int, _c_void_p]),
    "bkm_finalize": (_int, [_c_void_p, _c_void_p, _c_void_p, _c_void_p, _c_void_p, _int, _int, _c_void_p]),
    "bkm_check_finite": (_int, [_c_void_p, _i64, _int, _i64, _int, _c_void_p, _c_void_p]),
    "bkm_p2p_mailbox_bytes": (_int, [_int, _i64, ctypes.POINTER(ctypes.c_size_t)]),
    "bkm_p2p_alloc": (_int, [ctypes.c_size_t, ctypes.POINTER(_c_void_p)]),
    "bkm_p2p_free": (_int, [_c_void_p]),
    "bkm_p2p_export": (_int, [_c_void_p, _c_void_p]),
    "bkm_p2p_import": (_int, [_c_void_p, ctypes.POINTER(_c_void_p)]),
    "bkm_p2p_close": (_int, [_c_void_p]),
    "bkm_allreduce_p2p": (_int, [_c_void_p, _i64, _c_void_p, _int, _int, _i64, ctypes.c_uint, _c_void_p]),
    "bkm_launch_count": (_i64, []),
    "bkm_debug_fallback_count": (_i64, []),
    "bkm_debug_abort_code": (ctypes.c_uint, []),
    "bkm_debug_abort_detail": (None, [_c_void_p]),
    "bkm_debug_trace": (_int, [_c_void_p, _int]),
    "bkm_debug_reset": (None, []),
    "bkm_debug_deferred_rows": (_int, [_c_void_p, _i64, _int, _int, _int, ctypes.POINTER(_int)]),
    "bkm_debug_tc_layout": (_int, [_int, _int, _int, _int, _int, ctypes.POINTER(_int)]),
    "bkm_debug_tc2_layout": (_int, [_int, _int, _i64, _int, ctypes.POINTER(_int)]),
    "bkm_debug_core_layout": (_int, [_int, _int, _i64, _int, _int, _int, _int, ctypes.POINTER(_int)]),
}

_lib = None


def load():
    """Load libbkm_b200.so (once) and declare every prototype.  Raises if it is absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            "libbkm_b200.so not found at %s — build it with `python -c 'import __graft_entry__ as g; "
            "g.build()'` or `make -C dask_ml_b200/csrc`.  There is no CPU fallback." % LIB_PATH
        )
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)       # AttributeError if a declared symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc, what):
    if rc != 0:
        msg = load().bkm_error_string(rc)
        raise RuntimeError("%s failed: %s (code %d)" % (what, msg.decode() if msg else "?", rc))


def call(name, *args):
    """Call the entry point ``name``; raise with its name and the library's message on a non-zero status."""
    rc = getattr(_lib or load(), name)(*args)
    if rc:
        check(rc, name)
