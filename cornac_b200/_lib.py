"""ctypes binding of libb200cornac.so (C ABI declared in include/b200cornac.h).

There is no CPU fallback: if the shared library is missing or a call fails, a
B200Error is raised.  Device pointers are taken from torch CUDA tensors, which this
package uses purely as device-memory containers (no torch.nn / autograd anywhere).
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libb200cornac.so")


class B200Error(RuntimeError):
    pass


_c = ctypes
_vp, _i64, _i32, _u64, _u32, _f32, _int = (_c.c_void_p, _c.c_int64, _c.c_int32, _c.c_uint64, _c.c_uint32,
                                           _c.c_float, _c.c_int)

# B200_SPARSE of include/b200cornac.h: ptr, idx, row, val, nnz, cptr, crow, cpos, cval
_SPARSE = [_vp] * 4 + [_i64] + [_vp] * 4
# B200_C2PF_PARAMS: variant, sizes, k, the ratings, the graph, (at, bt), the state
_C2PF = [_int, _i64, _i64, _int] + _SPARSE + [_i64] + [_vp] * 5 + [_c.c_double] * 2 + [_vp] * 9
# B200_EFM_DATA: the matrices A, X, Y; the two orders; the three sizes
_EFM = _SPARSE * 3 + [_vp] * 2 + [_i64] * 3

# name -> (restype, argtypes); mirrors include/b200cornac.h one to one
SIGNATURES = {
    "b200_last_error": (_c.c_char_p, []),
    "b200_abi_version": (_int, []),
    "b200_kernel_launches": (_i64, []),
    "b200_device_info": (_int, [_vp, _vp, _vp]),
    "b200_bpr_table_slots": (_i64, [_i64]),
    "b200_bpr_prepare": (_int, [_vp, _vp, _i64, _i64, _vp, _vp, _i64, _vp]),
    "b200_bpr_epoch": (_int, [_vp, _vp, _i64, _i64, _i64, _i64, _i64, _vp, _vp, _vp, _int, _f32, _f32, _int,
                              _u64, _u64, _u64, _c.c_uint, _vp, _vp]),
    "b200_bpr_draw_host": (_int, [_u64, _u64, _u64, _i64, _i64, _i64, _vp, _vp]),
    "b200_bpr_draw_host2": (_int, [_u64, _u64, _u64, _i64, _i64, _i64, _u32, _u32, _vp, _vp]),
    "b200_bpr_block_plan": (_int, [_i64, _i64, _int, _vp, _vp]),
    "b200_bpr_epoch_replay": (_int, [_vp, _vp, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _int, _f32, _f32, _int,
                                     _c.c_uint, _vp, _vp]),
    "b200_bpr_epoch_replay2": (_int, [_vp, _vp, _i64, _vp, _vp, _vp, _i64, _i64, _vp, _vp, _vp, _int, _f32, _f32, _int,
                                      _c.c_uint, _vp, _vp]),
    "b200_mt_sampler_create": (_vp, [_u32]),
    "b200_mt_sampler_destroy": (None, [_vp]),
    "b200_mt_sampler_fill_i64": (_int, [_vp, _i64, _i64, _vp]),
    "b200_mt_sampler_fill_i32": (_int, [_vp, _i64, _i64, _vp]),
    "b200_vebpr_epoch": (_int, [_vp, _vp, _vp, _i64, _i64, _i64, _vp, _vp, _vp, _vp, _int, _f32, _f32, _f32, _u64, _u64, _i64,
                                _vp, _vp]),
    "b200_vebpr_epoch_replay": (_int, [_vp, _vp, _vp, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _int, _f32, _f32, _f32, _vp, _vp]),
    "b200_vebpr_draw_host": (_int, [_vp, _vp, _vp, _i64, _i64, _vp, _vp, _vp, _i64, _vp, _vp, _vp]),
    "b200_sbpr_epoch": (_int, [_vp, _vp, _vp, _i64, _i64, _i64, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _int, _f32, _f32, _f32, _f32,
                               _int, _u64, _u64, _i64, _vp, _vp]),
    "b200_sbpr_epoch_replay": (_int, [_vp, _vp, _vp, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _int,
                                      _f32, _f32, _f32, _f32, _int, _vp, _vp]),
    "b200_sbpr_draw_host": (_int, [_vp, _vp, _i64, _i64, _vp, _vp, _i64, _vp, _vp, _vp]),
    "b200_mf_epoch": (_int, [_vp, _vp, _vp, _i64, _int, _i64, _i64, _vp, _vp, _vp, _vp, _int, _f32, _f32, _f32, _int, _int,
                             _c.c_uint, _vp, _vp]),
    "b200_wmf_step": (_int, [_vp, _vp, _vp, _vp, _int, _i64, _i64, _int, _vp, _vp, _vp, _vp, _vp, _vp,
                             _f32, _f32, _f32, _f32, _f32, _f32, _f32, _f32, _vp, _vp, _vp, _vp]),
    "b200_knn_similarity_workspace_bytes": (_i64, [_i64]),
    "b200_knn_similarity": (_int, [_i64, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _vp, _c.c_double, _vp, _vp, _vp]),
    "b200_knn_row_nnz": (_int, [_i64, _vp, _vp, _vp]),
    "b200_knn_compact": (_int, [_i64, _vp, _vp, _vp, _vp, _vp]),
    "b200_knn_score_workspace_bytes": (_i64, [_i64, _i64, _int]),
    "b200_knn_score_items": (_int, [_vp, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _int, _vp, _vp, _vp]),
    "b200_knn_score_users": (_int, [_vp, _i64, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _int, _vp, _vp, _vp]),
    "b200_pmf_schedule": (_int, [_vp, _vp, _i64, _i64, _i64, _vp, _vp, _vp]),
    "b200_pmf_fit": (_int, [_int, _vp, _vp, _vp, _vp, _i32, _i64, _int, _vp, _vp, _vp, _vp, _int, _f32, _f32, _f32, _vp,
                            _vp, _vp]),
    "b200_pmf_sigmoid": (_int, [_vp, _i64, _vp, _vp]),
    "b200_cofactor_schedule": (_int, [_int, _vp, _vp, _i64, _vp, _vp, _i64, _i64, _i64, _vp, _vp, _vp]),
    "b200_cofactor_fit": (_int, [_int, _vp, _vp, _vp, _vp, _vp, _i32, _i64, _i64, _int, _vp, _vp, _vp, _vp, _vp, _vp, _int,
                                 _f32, _f32, _f32, _f32, _vp, _vp, _vp]),
    "b200_csc_map": (_int, [_vp, _vp, _i64, _i64, _i64, _vp, _vp]),
    "b200_nmf_fit": (_int, [_i64, _i64] + _SPARSE + [_vp] * 6 + [_i32, _int] + [_vp] * 6 + [_int] + [_f32] * 6 +
                     [_int, _vp, _vp]),
    "b200_ease_gram_workspace_bytes": (_i64, [_i64]),
    "b200_ease_gram": (_int, [_i64, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _vp, _c.c_double, _vp, _vp, _vp]),
    "b200_spd_inverse_workspace_bytes": (_i64, [_i64]),
    "b200_spd_inverse": (_int, [_i64, _vp, _vp, _vp, _int, _vp]),
    "b200_ease_weights": (_int, [_i64, _vp, _vp, _int, _vp]),
    "b200_ease_score": (_int, [_vp, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp]),
    "b200_hpf_workspace_bytes": (_i64, [_i64, _i64, _i64, _int]),
    "b200_hpf_expect": (_int, [_vp, _vp, _i64, _vp, _vp]),
    "b200_hpf_update": (_int, [_int, _i64, _i64, _int] + _SPARSE + [_vp] * 10),
    "b200_hpf_fit": (_int, [_int, _i64, _i64, _int] + _SPARSE + [_vp] * 6 + [_int, _vp, _vp]),
    "b200_c2pf_workspace_bytes": (_i64, [_i64, _i64, _i64, _i64, _int]),
    "b200_c2pf_update": (_int, _C2PF + [_vp] * 11),
    "b200_c2pf_fit": (_int, _C2PF + [_int, _vp, _vp]),
    "b200_efm_fit": (_int, _EFM + [_int, _int] + [_vp] * 7 + [_int] + [_f32] * 5 + [_vp, _vp]),
    "b200_efm_queries": (_int, [_vp, _i64, _vp, _vp, _vp, _i64, _int, _int, _int, _c.c_double, _c.c_double, _vp, _vp]),
    "b200_mter_workspace_bytes": (_i64, [_i64] * 4 + [_int] * 6),
    "b200_mter_fit": (_int, [_i64] * 4 + [_int] * 4 + ([_vp] * 4 + [_i64]) * 3 + [_vp] * 4 + [_i64] + [_int] * 3 +
                      [_vp] * 4 + [_f32] * 3 + [_int, _u64, _u64] + [_vp] * 4),
    "b200_mter_queries": (_int, [_vp, _i64, _vp, _vp, _int, _int, _int, _vp, _vp]),
    "b200_score": (_int, [_vp, _i64, _vp, _i64, _int, _vp, _f32, _vp, _vp]),
    "b200_score_batch": (_int, [_vp, _vp, _i64, _vp, _i64, _int, _vp, _vp, _vp, _vp]),
    "b200_topk_rows": (_int, [_vp, _i64, _i64, _vp, _vp, _int, _vp, _vp, _vp]),
    "b200_score_batch_f64": (_int, [_vp, _vp, _i64, _vp, _i64, _int, _vp, _vp]),
    "b200_topk_rows_f64": (_int, [_vp, _i64, _i64, _vp, _vp, _int, _vp, _vp, _vp]),
    "b200_rank_topk_workspace_bytes": (_i64, [_i64, _i64, _int, _int]),
    "b200_rank_topk": (_int, [_vp, _vp, _i64, _vp, _i64, _int, _vp, _vp, _vp, _vp, _int, _vp, _vp,
                              _vp, _i64, _vp]),
    "b200_rank_items_bytes": (_i64, [_i64, _int]),
    "b200_rank_pack_items": (_int, [_vp, _i64, _int, _vp, _vp, _i64, _vp]),
    "b200_rank_topk_packed": (_int, [_vp, _vp, _i64, _vp, _i64, _int, _vp, _vp, _vp, _vp, _int, _vp, _vp,
                                     _vp, _vp, _i64, _vp]),
    "b200_rank_tc_debug_scores": (_int, [_vp, _i64, _vp, _i64, _int, _vp, _vp, _i64, _vp, _i64, _vp]),
    "b200_topk_metrics": (_int, [_vp, _i64, _int, _i64, _vp, _vp, _vp, _vp, _vp, _int, _vp, _vp]),
    "b200_rank_counts": (_int, [_vp, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "b200_delta_make": (_int, [_vp, _vp, _vp, _i64, _vp]),
    "b200_delta_apply": (_int, [_vp, _vp, _vp, _i64, _vp]),
    "b200_ipc_export": (_int, [_vp, _vp, _vp]),
    "b200_ipc_open": (_int, [_vp, _i64, _vp]),
    "b200_ipc_close": (_int, [_vp, _i64]),
    "b200_item_exchange_slice": (_int, [_int, _int, _i64, _vp, _vp]),
    "b200_item_exchange": (_int, [_int, _int, _vp, _vp, _vp, _i64, _u32, _int, _vp]),
}

SGD_ATOMIC = 1
SGD_EXACT_EXP = 2
SGD_UNBOUNDED = 4
BPR_NEG_WEIGHTED = 8
BPR_LOSS_HINGE = 16
BPR_BLOCKED = 32
BPR_DETERMINISTIC = 64
PMF_LINEAR, PMF_NON_LINEAR = 0, 1
COFACTOR_SOREC, COFACTOR_MCF = 0, 1
MTER_UNORDERED, MTER_PHILOX = 1, 2
SPD_POTRF, SPD_TRTRI, SPD_LAUUM, SPD_ALL = 1, 2, 4, 7
METRIC_NDCG, METRIC_PRECISION, METRIC_RECALL, METRIC_FMEASURE, METRIC_HIT, METRIC_NCRR = range(6)

_lib = None


def load():
    """Load the shared library (once).  Raises B200Error when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise B200Error(
            "libb200cornac.so not found at %s -- build it with `python -m cornac_b200.build` "
            "(nvcc, sm_90a).  There is no CPU fallback." % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)   # AttributeError if the header and the library disagree
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc, what):
    if rc != 0:
        msg = load().b200_last_error()
        raise B200Error("%s failed (status %d): %s" % (what, rc, msg.decode() if msg else "?"))


def ptr(t):
    """Device (or host) address of a torch tensor / numpy array / None."""
    if t is None:
        return None
    if hasattr(t, "data_ptr"):
        return t.data_ptr()
    return t.ctypes.data


def current_stream():
    import torch
    return torch.cuda.current_stream().cuda_stream
