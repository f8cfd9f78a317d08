"""ctypes binding of libmmrec_b200.so (the C ABI in include/mmrec_b200.h).

There is NO CPU fallback: if the shared library is missing or a call fails, this raises.
Build it with `python -c "import __graft_entry__ as g; g.build()"` or `make -C mmrec_b200/csrc`.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libmmrec_b200.so")

_i64, _i32, _f32, _f64, _sz, _p = C.c_int64, C.c_int, C.c_float, C.c_double, C.c_size_t, C.c_void_p

# name -> (restype, argtypes); pointers are passed as raw addresses (tensor.data_ptr())
PROTOTYPES = {
    "mmrec_abi_version": (_i32, []),
    "mmrec_last_error": (C.c_char_p, []),
    "mmrec_device_check": (_i32, []),
    "mmrec_launch_count": (_i64, []),
    "mmrec_csr_from_coo_workspace_bytes": (_sz, [_i64, _i64]),
    "mmrec_csr_from_coo": (_i32, [_i64, _p, _p, _p, _i64, _i64, _i32, _p, _p, _p, _p, _p, _sz, _p]),
    "mmrec_spmm_plan_workspace_bytes": (_sz, [_i64, _i64]),
    "mmrec_spmm_plan": (_i32, [_i64, _p, _i32, _i32, _i64, _p, _p, _p, _p, _sz, _p]),
    "mmrec_bipartite_norm_workspace_bytes": (_sz, [_i64, _i64]),
    "mmrec_bipartite_norm_f32": (_i32, [_i64, _p, _p, _i64, _i64, _f32, _p, _p, _sz, _p]),
    "mmrec_spmm_set_lanes": (_i32, [_i32]),
    "mmrec_spmm_run_f32": (_i32, [_i32, _i32, _p, _i32, _p]),
    "mmrec_edge_keep_bits": (_i32, [_i64, _p, _f32, _p, _p, _p, _p, _p]),
    "mmrec_project_set_path": (_i32, [_i32]),
    "mmrec_project_workspace_bytes": (_sz, [_i64, _i64, _i32]),
    "mmrec_project_f32": (_i32, [_i64, _p, _p, _i64, _i64, _p, _p, _i32, _i32, _p, _i64, _p, _sz, _p]),
    "mmrec_debug_mma_rate": (_i32, [_i32, _i32, _i32, _i32, _p, _p]),
    "mmrec_debug_stream_probe": (_i32, [_p, _i64, _i64, _i32, _i32, _i32, _p, _p]),
    "mmrec_score_set_path": (_i32, [_i32]),
    "mmrec_score_workspace_bytes": (_sz, [_i64, _i64, _i32]),
    "mmrec_score_f32": (_i32, [_i64, _p, _p, _i64, _i64, _p, _i64, _i32, _p, _i64, _p, _sz, _p]),
    "mmrec_mask_f32": (_i32, [_i64, _p, _p, _i64, _i64, _i64, _p, _i64, _p]),
    "mmrec_topk_rows_f32": (_i32, [_i64, _i64, _p, _i64, _i32, _i64, _p, _p, _p]),
    "mmrec_score_topk_workspace_bytes": (_sz, [_i64, _i64, _i32, _i32]),
    "mmrec_score_topk_f32": (_i32, [_i64, _p, _p, _i64, _i64, _p, _i64, _i32, _i64, _p, _p, _i32, _i64, _p, _p, _p,
                                    _sz, _p]),
    "mmrec_catalog_bytes": (_sz, [_i64, _i32]),
    "mmrec_catalog_pack_f32": (_i32, [_i64, _p, _i64, _i32, _p, _sz, _p]),
    "mmrec_score_topk_cat_f32": (_i32, [_i64, _p, _p, _i64, _i64, _p, _i64, _i32, _p, _i64, _p, _p, _i32, _i64, _p, _p, _p,
                                        _sz, _p]),
    "mmrec_debug_cf_timing": (_i32, [_p, _i32]),
    "mmrec_debug_fused_fallback_rows": (_i64, [_p, _i64, _i64, _i32, _i32, _i64, _i32]),
    "mmrec_debug_cf_scratch": (_i32, [_i64, _i64, _i32, _i32, _i64, _i32, _p, _i32]),
    "mmrec_knn_topk_workspace_bytes": (_sz, [_i64, _i32, _i64, _i32]),
    "mmrec_knn_topk_f32": (_i32, [_i64, _p, _i64, _i32, _i64, _p, _i32, _p, _p, _p, _sz, _p]),
    "mmrec_debug_knn_fallback_rows": (_i64, []),
    "mmrec_debug_knn_scratch": (_i32, [_i64, _i32, _i64, _i32, _p, _i32]),
    "mmrec_knn_topk_shrink_f32": (_i32, [_i64, _p, _i64, _i32, _i64, _p, _i32, _p, _f32, _p, _p, _p, _sz, _p]),
    "mmrec_sparse_scores_f32": (_i32, [_i64, _p, _i64, _p, _p, _p, _p, _p, _p, _p, _i64, _p]),
    "mmrec_sparse_score_topk_workspace_bytes": (_sz, [_i64, _i64, _i64, _i32]),
    "mmrec_sparse_score_topk_f32": (_i32, [_i64, _p, _i64, _p, _p, _p, _p, _p, _p, _i64, _p, _p, _i32, _p, _p, _p, _sz, _p]),
    "mmrec_debug_sparse_topk_fallback_rows": (_i64, []),
    "mmrec_expsum_rows_workspace_bytes": (_sz, [_i64, _i64, _i32]),
    "mmrec_expsum_rows_f32": (_i32, [_i64, _p, _i64, _i64, _p, _i64, _i32, _f32, _p, _p, _sz, _p]),
    "mmrec_expsum_rows_bwd_f32": (_i32, [_i64, _p, _i64, _i64, _p, _i64, _i32, _f32, _p, _p, _i64, _p, _i64, _p, _sz, _p]),
    "mmrec_topk_merge": (_i32, [_i32, _i64, _i32, _p, _p, _p, _p, _p]),
    "mmrec_topk_merge_peers": (_i32, [_i32, _i64, _i32, _p, _p, _i64, _i64, _i64, _i64, _p, _p, _p, _p, _i32, _p]),
    "mmrec_peer_exchange_f32": (_i32, [_i64, _i32, _i32, _p, _p, _p, _p, _p, _p, _f32, _i32, _p]),
    "mmrec_peer_barrier": (_i32, [_i32, _i32, _p, _p, _p]),
    "mmrec_peer_reduce_push_f32": (_i32, [_i64, _i32, _i32, _p, _p, _p, _p, _f32, _i32, _p]),
    "mmrec_peer_gather_f32": (_i32, [_i64, _i32, _p, _p, _p]),
    "mmrec_topk_metrics_f64": (_i32, [_i64, _i32, _p, _p, _p, _p, _p, _p, _p]),
    "mmrec_peer_sum_f32": (_i32, [_i64, _i32, _p, _p, _p, _f32, _p, _p]),
    "mmrec_index_sum_rows_f32": (_i32, [_i64, _p, _p, _i64, _i32, _i64, _p, _i64, _p]),
    "mmrec_linear_wgrad_workspace_bytes": (_sz, [_i64, _i64, _i32]),
    "mmrec_linear_wgrad_f32": (_i32, [_i64, _p, _p, _i64, _i32, _p, _i64, _i64, _p, _p, _p, _sz, _p]),
    "mmrec_linear_dgrad_f32": (_i32, [_i64, _p, _i64, _i32, _p, _i64, _p, _p]),
    "mmrec_linear_dgrad_adam_f32": (_i32, [_i64, _p, _i64, _i32, _p, _i64, _p, _p, _p, _f64, _f64, _f64, _f64, _f64, _f64, _p]),
    "mmrec_adam_f32": (_i32, [_i32, _p, _f64, _f64, _f64, _f64, _p]),
    "mmrec_gate_rows_f32": (_i32, [_i64, _i32, _p, _p, _p, _p, _p, _p]),
    "mmrec_mgcn_fuse_f32": (_i32, [_i64, _i32, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p]),
}

class SpmmOp(C.Structure):
    """`mmrec_spmm_op` of include/mmrec_b200.h."""
    _fields_ = [("n_rows", _i64), ("n_cols", _i64), ("rowptr", _p), ("colidx", _p), ("vals", _p),
                ("tasks", _p), ("n_tasks", _i64), ("n_cta_tasks", _i64), ("split_rows", _p), ("counters", _p), ("partial", _p),
                ("X", _p), ("ldx", _i64), ("X_hi", _p), ("ldx_hi", _i64), ("x_split", _i64),
                ("Y", _p), ("ldy", _i64), ("y_accumulate", _i32),
                ("acc_in", _p), ("acc_out", _p), ("ldacc", _i64), ("acc_div", _f32),
                ("acc_in_hi", _p), ("ldacc_in_hi", _i64), ("acc_in_split", _i64),
                ("gate_ref", _p), ("ldgate", _i64), ("post", _p), ("ldpost", _i64), ("post_row0", _i64),
                ("keep_bits", _p), ("keep_scale", _f32), ("sync_before", _i32)]


class AdamTensor(C.Structure):
    """`mmrec_adam_tensor` of include/mmrec_b200.h."""
    _fields_ = [("param", _p), ("grad", _p), ("exp_avg", _p), ("exp_avg_sq", _p), ("n", _i64), ("step_size", _f64), ("bc2_sqrt", _f64)]


_lib = None
ABI_VERSION = 4


class MMRecError(RuntimeError):
    pass


def load():
    """Load the library and bind every symbol of the header; raises if anything is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.isfile(LIB_PATH):
        raise MMRecError(f"{LIB_PATH} not found: the CUDA library is not built and there is no CPU fallback "
                         "(run `make -C mmrec_b200/csrc` or `__graft_entry__.build()`)")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in PROTOTYPES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype, fn.argtypes = res, args
    if lib.mmrec_abi_version() != ABI_VERSION:
        raise MMRecError("libmmrec_b200.so ABI version mismatch")
    _lib = lib
    return lib


def check(rc: int, what: str):
    if rc != 0:
        msg = load().mmrec_last_error().decode(errors="replace")
        raise MMRecError(f"{what} failed (code {rc}): {msg}")


def require_device():
    """Fail loudly unless an H100-class (sm_90) device is current."""
    import torch
    if not torch.cuda.is_available():
        raise MMRecError("mmrec_b200 needs a CUDA device (sm_90a); there is no CPU path")
    check(load().mmrec_device_check(), "mmrec_device_check")
