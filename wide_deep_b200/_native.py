"""ctypes binding of libwd_b200.so (the C-ABI declared in include/wd_b200.h).

The library is the product: there is no Python/PyTorch fallback for any compute entry point.  Importing
this module only needs the shared object (it loads without a GPU so host-side code and CPU tests can use
the loader and the hash functions); creating a model without a CUDA device raises ``NativeError``.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.path.join(_HERE, "libwd_b200.so")
_lib = None

OK, EINVAL, ENODEVICE, ECUDA, ENOMEM, EUNSUPPORTED, ESTATE = 0, -1, -2, -3, -4, -5, -6


class NativeError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("libwd_b200 error %d: %s" % (code, msg))
        self.code = code


class BatchC(ctypes.Structure):
    _fields_ = [("batch_size", ctypes.c_int32), ("cat_offsets", ctypes.c_void_p), ("cat_keys", ctypes.c_void_p),
                ("nnz", ctypes.c_int64), ("dense", ctypes.c_void_p), ("label", ctypes.c_void_p), ("weight", ctypes.c_void_p)]


class TsvSpecC(ctypes.Structure):
    _fields_ = [("n_columns", ctypes.c_int32), ("col_role", ctypes.c_void_p), ("col_target", ctypes.c_void_p),
                ("n_cat_fields", ctypes.c_int32), ("n_dense_fields", ctypes.c_int32), ("multivalue", ctypes.c_int32),
                ("tf_compat_pad", ctypes.c_int32), ("pos_weight", ctypes.c_float), ("neg_weight", ctypes.c_float),
                ("use_weight", ctypes.c_int32), ("has_label", ctypes.c_int32)]


# every symbol include/wd_b200.h declares: name -> (restype, argtypes)
_vp, _i32, _i64, _u64 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64, ctypes.c_uint64
SYMBOLS = {
    "wd_last_error": (ctypes.c_char_p, []),
    "wd_version": (ctypes.c_int, []),
    "wd_device_count": (ctypes.c_int, []),
    "wd_model_create": (ctypes.c_int, [_vp, ctypes.c_int, ctypes.POINTER(_vp)]),
    "wd_model_destroy": (ctypes.c_int, [_vp]),
    "wd_model_init": (ctypes.c_int, [_vp, _u64]),
    "wd_set_opt_step": (ctypes.c_int, [_vp, _i64]),
    "wd_tensor_io": (ctypes.c_int, [_vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, _vp, _i64, ctypes.c_int]),
    "wd_tensor_io_rows": (ctypes.c_int, [_vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, _i64, _i64, _vp, ctypes.c_int]),
    "wd_tensor_size": (_i64, [_vp, ctypes.c_int, ctypes.c_int, ctypes.c_int]),
    "wd_memory_usage": (ctypes.c_int, [_vp, ctypes.POINTER(_i64), ctypes.POINTER(_i64)]),
    "wd_host_cache_enable": (ctypes.c_int, [_vp, _i64]),
    "wd_shard_cache_enable": (ctypes.c_int, [_vp, _i64]),
    "wd_host_cache_stats": (ctypes.c_int, [_vp, ctypes.POINTER(_i64), _i32, _i32]),
    "wd_deferred_adam_stats": (ctypes.c_int, [_vp, ctypes.POINTER(_i64), _i32, _i32]),
    "wd_train_step": (ctypes.c_int, [_vp, _vp, ctypes.POINTER(ctypes.c_float)]),
    "wd_forward": (ctypes.c_int, [_vp, _vp, _vp, ctypes.POINTER(ctypes.c_float)]),
    "wd_batch_upload": (ctypes.c_int, [_vp, _vp]),
    "wd_train_step_resident": (ctypes.c_int, [_vp, ctypes.POINTER(ctypes.c_float)]),
    "wd_forward_resident": (ctypes.c_int, [_vp, _vp, ctypes.POINTER(ctypes.c_float)]),
    "wd_step_backward": (ctypes.c_int, [_vp, _vp, ctypes.POINTER(ctypes.c_float)]),
    "wd_step_backward_slot": (ctypes.c_int, [_vp, ctypes.c_int, ctypes.POINTER(ctypes.c_float)]),
    "wd_step_apply": (ctypes.c_int, [_vp]),
    "wd_dense_grad_count": (_i64, [_vp]),
    "wd_dense_grad_ptr": (_vp, [_vp]),
    "wd_sparse_grads": (ctypes.c_int, [_vp, ctypes.c_int, ctypes.POINTER(_vp), ctypes.POINTER(_vp), ctypes.POINTER(_i64),
                                       ctypes.POINTER(_i32), ctypes.POINTER(_i64)]),
    "wd_sparse_set": (ctypes.c_int, [_vp, ctypes.c_int, _vp, _vp, _i64]),
    "wd_sparse_set_sorted": (ctypes.c_int, [_vp, ctypes.c_int, _vp, _vp, ctypes.c_int32, _i64]),
    "wd_shard_info": (ctypes.c_int, [_vp, ctypes.POINTER(_i32), ctypes.POINTER(_i32), ctypes.POINTER(_i64)]),
    "wd_shard_ipc_handle": (ctypes.c_int, [_vp, _vp]),
    "wd_shard_connect_ipc": (ctypes.c_int, [_vp, _vp, _i32]),
    "wd_shard_connect_local": (ctypes.c_int, [_vp, _i32]),
    "wd_shard_local_sync": (ctypes.c_int, [_vp, _i32]),
    "wd_shard_phase": (ctypes.c_int, [_vp, ctypes.c_int, ctypes.c_int, ctypes.c_int]),
    "wd_shard_finish": (ctypes.c_int, [_vp, ctypes.POINTER(ctypes.c_float), _vp]),
    "wd_shard_train_step_slot": (ctypes.c_int, [_vp, ctypes.c_int, ctypes.POINTER(ctypes.c_float)]),
    "wd_shard_forward_slot": (ctypes.c_int, [_vp, ctypes.c_int, _vp, ctypes.POINTER(ctypes.c_float)]),
    "wd_shard_eval_accumulate_slot": (ctypes.c_int, [_vp, ctypes.c_int, _i32]),
    "wd_shard_eval_accumulate_phase": (ctypes.c_int, [_vp, _i32]),
    "wd_shard_eval_finish": (ctypes.c_int, [_vp, _vp]),
    "wd_eval_reset": (ctypes.c_int, [_vp]),
    "wd_eval_accumulate": (ctypes.c_int, [_vp, _vp]),
    "wd_eval_finish": (ctypes.c_int, [_vp, _vp]),
    "wd_eval_accumulate_slot": (ctypes.c_int, [_vp, ctypes.c_int]),
    "wd_fingerprint64_device": (ctypes.c_int, [_vp, _vp, _i64, _vp]),
    "wd_fingerprint64": (_u64, [ctypes.c_char_p, ctypes.c_size_t]),
    "wd_fingerprint_cat64": (_u64, [_u64, _u64]),
    "wd_debug_column_ids": (ctypes.c_int, [_vp, _vp, _i64, _vp, _i64, ctypes.POINTER(_i64)]),
    "wd_debug_slot": (ctypes.c_int, [_vp, ctypes.c_int, ctypes.POINTER(_i32), ctypes.POINTER(_i64), ctypes.POINTER(_i32), _vp, _vp, _vp,
                                     _vp, _vp]),
    "wd_debug_deep_input": (ctypes.c_int, [_vp, _vp, _i64]),
    "wd_debug_hidden": (ctypes.c_int, [_vp, ctypes.c_int, ctypes.c_int, _vp, _i64]),
    "wd_launch_count": (_i64, [_vp]),
    "wd_gemm_fallback_count": (_i64, [_vp]),
    "wd_graph_stats": (ctypes.c_int, [_vp, ctypes.POINTER(_i64), _i32]),
    "wd_last_timings": (ctypes.c_int, [_vp, _vp, ctypes.c_int]),
    "wd_timing_name": (ctypes.c_char_p, [_vp, ctypes.c_int]),
    "wd_batch_upload_slot": (ctypes.c_int, [_vp, ctypes.c_int, _vp]),
    "wd_batch_prefetch_slot": (ctypes.c_int, [_vp, ctypes.c_int, _vp]),
    "wd_last_loss": (ctypes.c_int, [_vp, _vp]),
    "wd_debug_gemm_probe": (ctypes.c_int, [_vp]),
    "wd_train_step_slot": (ctypes.c_int, [_vp, ctypes.c_int, ctypes.POINTER(ctypes.c_float)]),
    "wd_set_profile": (ctypes.c_int, [_vp, ctypes.c_int]),
    "wd_stream": (_vp, [_vp]),
    "wd_stream_sparse": (_vp, [_vp, ctypes.c_int]),
    "wd_sync": (ctypes.c_int, [_vp]),
    "wd_host_alloc": (ctypes.c_int, [ctypes.c_size_t, ctypes.POINTER(_vp)]),
    "wd_host_free": (ctypes.c_int, [_vp]),
    "wd_tsv_parse": (_i64, [_vp, ctypes.c_char_p, _i64, _i32, _vp, _vp, _i64, _vp, _vp, _vp, _i32]),
    "wd_tsv_index_lines": (_i64, [_vp, _i64, _vp, _vp, _i64]),
    "wd_tsv_parse_lines": (_i64, [_vp, _vp, _vp, _vp, _vp, _i32, _vp, _vp, _i64, _vp, _vp, _vp, _i32]),
    "wd_tsv_gather_lines": (_i64, [_vp, _vp, _vp, _vp, _i32, _vp, _i64, _vp, _i32]),
    "wd_tsv_parse_slot": (ctypes.c_int, [_vp, ctypes.c_int, _vp, _vp, _i64, _vp, _i32]),
    "wd_tsv_parse_stats": (ctypes.c_int, [_vp, ctypes.POINTER(_i64), _i32, _i32]),
    "wd_summary_limits": (ctypes.c_int, [_vp, _i32]),
    "wd_summary_segments": (ctypes.c_int, [_vp, _vp, _vp, _vp, _i32]),
    "wd_summary_arm": (ctypes.c_int, [_vp]),
    "wd_summary_read": (ctypes.c_int, [_vp, _vp, _vp, _vp, _i32]),
}


def lib():
    """Load libwd_b200.so (built in-tree by build_native.py).  Raises if it has not been built: the
    product never silently runs without its CUDA library."""
    global _lib
    if _lib is None:
        if not os.path.exists(SO_PATH):
            raise NativeError(ESTATE, "%s not found: run `python build_native.py` (nvcc, sm_90a)" % SO_PATH)
        L = ctypes.CDLL(SO_PATH)
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(L, name)
            fn.restype, fn.argtypes = res, args
        _lib = L
    return _lib


def check(rc):
    if rc != 0:
        raise NativeError(rc, lib().wd_last_error().decode("utf-8", "replace"))
    return rc
