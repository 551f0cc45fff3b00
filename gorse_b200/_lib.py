"""Loads libgorse_b200.so (the C-ABI product library) and declares every prototype of include/gorse_b200.h.

There is NO fallback: if the library is missing or a symbol is absent, importing fails loudly.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libgorse_b200.so")

NCCL_ID_BYTES = 128

OK = 0
ERR_ARG, ERR_CUDA, ERR_NCCL, ERR_OOM, ERR_RANGE, ERR_STATE, ERR_UNSUPPORTED, ERR_IO = -1, -2, -3, -4, -5, -6, -7, -8

SCATTER_STORE, SCATTER_ATOMIC = 0, 1
ORDER_HOGWILD, ORDER_SEQUENTIAL = 0, 1
METRIC_EUCLIDEAN, METRIC_NEG_DOT, METRIC_COSINE = 0, 1, 2
DISTANCE_COSINE, DISTANCE_EUCLIDEAN, DISTANCE_DOT = 0, 1, 2   # vectors.Distance


def _nd(dt):
    return np.ctypeslib.ndpointer(dtype=dt, flags="C_CONTIGUOUS")


F32, I32, I64 = _nd(np.float32), _nd(np.int32), _nd(np.int64)
VP = C.c_void_p
PVP = C.POINTER(C.c_void_p)

# name -> (restype, argtypes); mirrors include/gorse_b200.h one to one
PROTOTYPES = {
    "gorse_b200_version": (C.c_int32, []),
    "gorse_b200_last_error": (C.c_char_p, []),
    "gorse_b200_device_count": (C.c_int32, [C.POINTER(C.c_int32)]),
    "gorse_b200_ctx_create": (C.c_int32, [C.c_int32, PVP]),
    "gorse_b200_nccl_unique_id": (C.c_int32, [VP]),
    "gorse_b200_ctx_create_dist": (C.c_int32, [C.c_int32, C.c_int32, C.c_int32, VP, PVP]),
    "gorse_b200_ctx_destroy": (C.c_int32, [VP]),
    "gorse_b200_ctx_sync": (C.c_int32, [VP]),
    "gorse_b200_ctx_rank": (C.c_int32, [VP, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    "gorse_b200_ctx_timer_begin": (C.c_int32, [VP]),
    "gorse_b200_ctx_timer_end": (C.c_int32, [VP, C.POINTER(C.c_float)]),
    "gorse_b200_ctx_launch_count": (C.c_int32, [VP, C.POINTER(C.c_int64)]),
    "gorse_b200_device_bytes": (C.c_int32, [C.POINTER(C.c_int64)]),
    "gorse_b200_ctx_flush_l2": (C.c_int32, [VP]),
    "gorse_b200_ctx_barrier": (C.c_int32, [VP]),
    "gorse_b200_host_alloc": (C.c_int32, [C.c_size_t, PVP]),
    "gorse_b200_host_free": (C.c_int32, [VP]),
    "gorse_b200_cf_create": (C.c_int32, [VP, C.c_int32, C.c_int32, C.c_int32, VP, VP, VP, VP, PVP]),
    "gorse_b200_cf_destroy": (C.c_int32, [VP]),
    "gorse_b200_cf_set_factors": (C.c_int32, [VP, VP, VP]),
    "gorse_b200_cf_init_normal": (C.c_int32, [VP, C.c_float, C.c_float, C.c_uint64]),
    "gorse_b200_cf_get_factors": (C.c_int32, [VP, VP, VP]),
    "gorse_b200_cf_predict": (C.c_int32, [VP, VP, VP, C.c_int64, VP]),
    "gorse_b200_bpr_apply_triples": (C.c_int32, [VP, VP, C.c_int64, C.c_float, C.c_float, C.c_int32, C.c_int32]),
    "gorse_b200_bpr_sample_triples": (C.c_int32, [VP, C.c_uint64, C.c_int64, C.c_int64, VP]),
    "gorse_b200_bpr_epoch": (C.c_int32, [VP, C.c_float, C.c_float, C.c_int64, C.c_uint64, C.c_int32]),
    "gorse_b200_als_epoch": (C.c_int32, [VP, C.c_float, C.c_float]),
    "gorse_b200_cf_evaluate": (C.c_int32, [VP, VP, VP, VP, VP, C.c_int32, VP]),
    "gorse_b200_eval_create": (C.c_int32, [VP, VP, VP, VP, VP, C.c_int32, C.c_uint64, C.c_int32, PVP]),
    "gorse_b200_eval_run": (C.c_int32, [VP, VP]),
    "gorse_b200_eval_negatives": (C.c_int32, [VP, VP, VP]),
    "gorse_b200_eval_destroy": (C.c_int32, [VP]),
    "gorse_b200_fit_params_default": (C.c_int32, [C.c_int32, VP]),
    "gorse_b200_bpr_fit": (C.c_int32, [VP, VP, VP, VP, VP, VP, VP, VP, VP]),
    "gorse_b200_als_fit": (C.c_int32, [VP, VP, VP, VP, VP, VP, VP, VP, VP]),
    "gorse_b200_cf_fit_trials": (C.c_int32, [VP, C.c_int32, VP, VP, VP, VP, VP, VP, VP, VP, VP, VP, VP]),
    "gorse_b200_index_create": (C.c_int32, [VP, C.c_int32, C.c_int32, PVP]),
    "gorse_b200_index_destroy": (C.c_int32, [VP]),
    "gorse_b200_index_add": (C.c_int32, [VP, VP, C.c_int64, C.POINTER(C.c_int64)]),
    "gorse_b200_index_len": (C.c_int32, [VP, C.POINTER(C.c_int64)]),
    "gorse_b200_index_search_vectors": (C.c_int32, [VP, VP, C.c_int64, C.c_int32, C.c_int32, VP, VP, VP]),
    "gorse_b200_index_search_indices": (C.c_int32, [VP, VP, C.c_int64, C.c_int32, C.c_int32, VP, VP, VP]),
    "gorse_b200_index_search_range": (C.c_int32, [VP, C.c_int64, C.c_int64, C.c_int32, C.c_int32, VP, VP, VP]),
    "gorse_b200_index_stats": (C.c_int32, [VP, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_int64)]),
    "gorse_b200_index_stage1_scores": (C.c_int32, [VP, C.c_int64, C.c_int64, VP, VP]),
    "gorse_b200_bf16_truncate": (C.c_int32, [VP, C.c_int64, VP]),
    "gorse_b200_sparse_vector": (C.c_int32, [VP, C.c_int32, VP, C.c_int32, C.c_uint32, VP, VP, C.POINTER(C.c_int32)]),
    "gorse_b200_similar_scores": (C.c_int32, [C.c_int32, C.c_double, C.c_int32, C.c_int32, VP, VP, C.c_int32, VP, VP,
                                              C.POINTER(C.c_int32)]),
    "gorse_b200_index_query_similar": (C.c_int32, [VP, C.c_int64, C.c_int64, C.c_int32, C.c_double, VP, VP, VP]),
    "gorse_b200_sparse_index_create": (C.c_int32, [VP, PVP]),
    "gorse_b200_sparse_index_destroy": (C.c_int32, [VP]),
    "gorse_b200_sparse_index_add": (C.c_int32, [VP, VP, VP, VP, C.c_int64, C.POINTER(C.c_int64)]),
    "gorse_b200_sparse_index_len": (C.c_int32, [VP, C.POINTER(C.c_int64)]),
    "gorse_b200_sparse_index_search_range": (C.c_int32, [VP, C.c_int64, C.c_int64, C.c_int32, VP, VP, VP]),
    "gorse_b200_sparse_index_stats": (C.c_int32, [VP, C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_int64),
                                                  C.POINTER(C.c_double)]),
    "gorse_b200_vecdb_create": (C.c_int32, [VP, C.c_int32, C.c_int32, PVP]),
    "gorse_b200_vecdb_destroy": (C.c_int32, [VP]),
    "gorse_b200_vecdb_count": (C.c_int32, [VP, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "gorse_b200_vecdb_add": (C.c_int32, [VP, C.c_int64, VP, VP, VP, VP, VP, VP, VP, VP, C.POINTER(C.c_int64)]),
    "gorse_b200_vecdb_add_idf_vectors": (C.c_int32, [VP, C.c_int64, VP, VP, VP, C.c_int32, C.c_uint32, VP, VP, VP, C.c_int32, C.c_uint32, VP,
                                                     C.c_int64, VP, VP, VP, VP]),
    "gorse_b200_vecdb_get": (C.c_int32, [VP, VP, C.c_int64, VP, VP, VP, VP]),
    "gorse_b200_vecdb_get_sparse": (C.c_int32, [VP, C.c_int64, VP, VP, C.c_int32, C.POINTER(C.c_int32)]),
    "gorse_b200_vecdb_delete_before": (C.c_int32, [VP, C.c_int64, VP, C.c_int64, C.POINTER(C.c_int64)]),
    "gorse_b200_vecdb_compact": (C.c_int32, [VP, VP, VP]),
    "gorse_b200_vecdb_storage": (C.c_int32, [VP, C.POINTER(C.c_int32), C.POINTER(C.c_int64)]),
    "gorse_b200_vecdb_neighbour_cache": (C.c_int32, [VP, C.c_int32, C.c_int64]),
    "gorse_b200_vecdb_neighbour_cache_stats": (C.c_int32, [VP, VP]),
    "gorse_b200_vecdb_neighbour_cache_fill": (C.c_int32, [VP, VP]),
    "gorse_b200_vecdb_neighbour_cache_save": (C.c_int32, [VP, VP, VP, C.POINTER(C.c_int64)]),
    "gorse_b200_vecdb_neighbour_cache_load": (C.c_int32, [VP, VP, VP, VP]),
    "gorse_b200_vecdb_save": (C.c_int32, [VP, VP, VP, VP, C.POINTER(C.c_int64)]),
    "gorse_b200_vecdb_load": (C.c_int32, [VP, VP, VP, PVP, C.POINTER(C.c_int64)]),
    "gorse_b200_vecdb_add_item_factors": (C.c_int32, [VP, VP, VP, C.c_int64, VP, VP, VP]),
    "gorse_b200_marshal_latent_factors": (C.c_int32, [VP, C.c_int32, C.c_int32, VP, VP, VP, C.c_size_t, C.POINTER(C.c_size_t)]),
    "gorse_b200_vecdb_query": (C.c_int32, [VP, C.c_int64, VP, VP, VP, VP, C.c_int32, C.c_int32, VP, VP, VP]),
    "gorse_b200_vecdb_query_excluding": (C.c_int32, [VP, C.c_int64, VP, VP, C.c_int32, C.c_int32, VP, VP, VP, VP, VP,
                                                     C.POINTER(C.c_int64)]),
    "gorse_b200_vecdb_item_to_item": (C.c_int32, [VP, C.c_int64, VP, VP, VP, VP, VP, C.c_int32, C.c_int32, C.c_double, VP, VP, VP, VP]),
    "gorse_b200_vecdb_user_to_user": (C.c_int32, [VP, C.c_int64, VP, C.c_int64, VP, VP, C.c_int32, VP, VP, VP, C.c_int32, C.c_double, VP, VP,
                                                  VP, VP]),
    "gorse_b200_vecdb_session_recommend": (C.c_int32, [VP, C.c_int64, VP, VP, VP, VP, VP, C.c_int32, C.c_int32, C.c_int32, C.c_double, VP,
                                                       VP, VP, VP]),
    "gorse_b200_fm_create": (C.c_int32, [VP, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, VP, VP, C.c_int64, PVP]),
    "gorse_b200_fm_destroy": (C.c_int32, [VP]),
    "gorse_b200_fm_rank": (C.c_int32, [VP, C.c_int64, VP, VP, VP, VP, C.c_int64, VP, VP, VP, VP, VP, VP, VP, VP, VP, VP, VP]),
    "gorse_b200_recommend": (C.c_int32, [VP, C.c_int64, VP, VP, C.c_int32, VP, C.c_int32, VP, VP, VP, VP, VP, VP, C.c_double, C.c_double, VP, VP,
                                         VP, VP]),
    "gorse_b200_fm_fit_params_default": (C.c_int32, [VP]),
    "gorse_b200_fm_fit": (C.c_int32, [VP, C.c_int64, C.c_int32, C.c_int32, VP, C.c_int64, VP, VP, VP, VP, C.c_int64, VP, VP, VP, VP, VP, C.c_int64,
                                      VP, VP, VP, VP, VP]),
    "gorse_b200_fm_fit_emb": (C.c_int32, [VP, C.c_int64, C.c_int32, VP, C.c_int64, VP, VP, VP, VP, VP, C.c_int64, VP, VP, VP, VP, VP, C.c_int32,
                                          VP, C.c_int64, VP, VP, VP, C.c_int64, VP, VP, VP, VP, VP]),
    "gorse_b200_fm_fit_trials": (C.c_int32, [VP, C.c_int64, C.c_int32, C.c_int32, VP, C.c_int64, VP, VP, VP, VP, VP, C.c_int64, VP, VP, VP, VP, VP,
                                             C.c_int32, VP, C.c_int64, VP, VP, VP, C.c_int64, VP, VP, VP, VP, VP]),
    "gorse_b200_fm_gauc": (C.c_int32, [VP, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, VP, VP, C.c_int64, C.c_int64, VP, VP, VP, VP,
                                       VP, C.c_int64, VP, VP, C.c_int64, VP, C.c_int64, VP, VP, VP, VP, VP, C.POINTER(C.c_int64),
                                       C.POINTER(C.c_double), VP]),
    "gorse_b200_embedding_eval":(C.c_int32, [VP, C.c_int32, C.c_int32, VP, VP, C.c_int64, VP, VP, VP, VP, VP, VP, VP, VP, C.c_int32, C.c_uint64,
                                              C.c_int32, VP, C.POINTER(C.c_int64)]),
    "gorse_b200_ncf_load":(C.c_int32, [C.c_char_p, C.c_char_p, PVP]),
    "gorse_b200_ncf_shape": (C.c_int32, [VP, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int64), C.POINTER(C.c_int64),
                                         C.POINTER(C.c_int64)]),
    "gorse_b200_ncf_get": (C.c_int32, [VP, VP, VP, VP, VP, VP, VP]),
    "gorse_b200_ncf_free": (C.c_int32, [VP]),
}


class FitParams(C.Structure):
    _fields_ = [("n_factors", C.c_int32), ("n_epochs", C.c_int32), ("lr", C.c_float), ("reg", C.c_float),
                ("init_mean", C.c_float), ("init_stddev", C.c_float), ("alpha", C.c_float), ("seed", C.c_uint64),
                ("verbose", C.c_int32), ("candidates", C.c_int32), ("topk", C.c_int32), ("patience", C.c_int32)]


class FitResult(C.Structure):
    _fields_ = [("ndcg", C.c_float), ("precision", C.c_float), ("recall", C.c_float), ("epochs_run", C.c_int32),
                ("early_stopped", C.c_int32), ("best_epoch", C.c_int32), ("cancelled", C.c_int32)]


class TrialState(C.Structure):
    _fields_ = [("epochs_run", C.c_int32), ("ndcg", C.c_float), ("finished", C.c_int32)]


FM_ADAM, FM_SGD = 0, 1


class FMFitParams(C.Structure):
    _fields_ = [("n_factors", C.c_int32), ("n_epochs", C.c_int32), ("lr", C.c_float), ("reg", C.c_float), ("optimizer", C.c_int32),
                ("batch_size", C.c_int32), ("verbose", C.c_int32), ("patience", C.c_int32), ("max_steps", C.c_int64)]


class FMTrialState(C.Structure):
    _fields_ = [("epochs_run", C.c_int32), ("auc", C.c_float), ("finished", C.c_int32)]


class FMFitResult(C.Structure):
    _fields_ = [("auc", C.c_float), ("precision", C.c_float), ("recall", C.c_float), ("accuracy", C.c_float), ("cost", C.c_float),
                ("epochs_run", C.c_int32), ("best_epoch", C.c_int32), ("early_stopped", C.c_int32), ("diverged", C.c_int32),
                ("cancelled", C.c_int32), ("steps", C.c_int64)]


STAGE_LIST, STAGE_COLLABORATIVE, STAGE_ITEM_TO_ITEM, STAGE_USER_TO_USER = 0, 1, 2, 3


class RecommendStage(C.Structure):
    _fields_ = [("kind", C.c_int32), ("list_len", C.c_int64), ("list_off", C.c_void_p), ("list_items", C.c_void_p), ("list_scores", C.c_void_p),
                ("db", C.c_void_p), ("n", C.c_int32), ("score_scale", C.c_double), ("ctx_off", C.c_void_p), ("ctx_items", C.c_void_p),
                ("slot_of_item", C.c_void_p), ("item_of_slot", C.c_void_p), ("categories", C.c_void_p), ("n_categories", C.c_int32),
                ("user_slots", C.c_void_p), ("n_fb_rows", C.c_int64), ("fb_off", C.c_void_p), ("fb_items", C.c_void_p), ("item_ok", C.c_void_p)]


class RecommendCF(C.Structure):
    _fields_ = [("db", C.c_void_p), ("user_vectors", C.c_void_p), ("slot_of_item", C.c_void_p), ("item_of_slot", C.c_void_p), ("n", C.c_int32)]


class RecommendRanker(C.Structure):
    _fields_ = [("fm", C.c_void_p), ("user_feat", C.c_void_p), ("user_lab_off", C.c_void_p), ("user_lab_idx", C.c_void_p),
                ("user_lab_val", C.c_void_p), ("item_feat", C.c_void_p), ("item_lab_off", C.c_void_p), ("item_lab_idx", C.c_void_p),
                ("item_lab_val", C.c_void_p), ("item_emb", C.c_void_p), ("item_emb_mask", C.c_void_p)]


PROGRESS_FN = C.CFUNCTYPE(C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_float)
TRIALS_PROGRESS_FN = C.CFUNCTYPE(C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.POINTER(TrialState))
FM_TRIALS_PROGRESS_FN = C.CFUNCTYPE(C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.POINTER(FMTrialState))
WRITE_FN = C.CFUNCTYPE(C.c_int32, C.c_void_p, C.c_void_p, C.c_int64)   # gorse_b200_write_fn
READ_FN = C.CFUNCTYPE(C.c_int64, C.c_void_p, C.c_void_p, C.c_int64)    # gorse_b200_read_fn


class GorseB200Error(RuntimeError):
    def __init__(self, status, message):
        super().__init__(f"gorse_b200 status {status}: {message}")
        self.status = status
        self.message = message


def _load():
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(make -C gorse_b200/csrc).  gorse_b200 has no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in PROTOTYPES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    return lib


lib = _load()


def check(status):
    if status != OK:
        raise GorseB200Error(status, lib.gorse_b200_last_error().decode("utf-8", "replace"))


def ptr(a):
    """Host pointer of a contiguous numpy array (or None)."""
    if a is None:
        return None
    assert a.flags.c_contiguous
    return a.ctypes.data_as(C.c_void_p)
