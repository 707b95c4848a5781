"""ctypes binding of libtcsdn.so (include/tcsdn.h).  No fallback: if the library is missing or has no
CUDA device, the error surfaces to the caller."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libtcsdn.so")

F32, F64 = 0, 1
HOST, DEVICE = 0, 1
OK, EINVAL, ECUDA, ENOMEM, ENONFINITE = 0, -1, -2, -3, -4
OPT_ENGINE, OPT_CHUNK_ROWS, OPT_CHECK_FINITE = 1, 2, 3
OPT_SCORER_SHAPE, OPT_FOREST_SHAPE, OPT_FOREST_SORT, OPT_KNN_FLUSH_TILES, OPT_KNN_PRUNE = 4, 5, 6, 7, 8
FLOW_STATE = 19
COMM_ID_BYTES = 128

_vp = C.c_void_p
_f64p = C.POINTER(C.c_double)
_i32p = C.POINTER(C.c_int32)
_i64p = C.POINTER(C.c_int64)

# symbol -> (restype, argtypes): exactly the entry points include/tcsdn.h declares
SIGNATURES = {
    "tcsdn_version": (C.c_int, []),
    "tcsdn_last_error": (C.c_char_p, []),
    "tcsdn_device_count": (C.c_int, [_i32p]),
    "tcsdn_set_device": (C.c_int, [C.c_int32]),
    "tcsdn_device_sm_count": (C.c_int, [_i32p]),
    "tcsdn_linear_create": (C.c_int, [_f64p, _f64p, C.c_int32, C.c_int32, C.POINTER(_vp)]),
    "tcsdn_gnb_create": (C.c_int, [_f64p, _f64p, _f64p, C.c_int32, C.c_int32, C.POINTER(_vp)]),
    "tcsdn_kmeans_create": (C.c_int, [_f64p, C.c_int32, C.c_int32, C.POINTER(_vp)]),
    "tcsdn_knn_create": (C.c_int, [_f64p, _i32p, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.POINTER(_vp)]),
    "tcsdn_svc_create": (C.c_int, [_f64p, _f64p, _f64p, _i32p, C.c_int32, C.c_int32, C.c_int32, C.c_double,
                                   C.POINTER(_vp)]),
    "tcsdn_forest_create": (C.c_int, [_i64p, _i32p, _i32p, _i32p, _f64p, _f64p, C.c_int32, C.c_int32, C.c_int32,
                                      C.POINTER(_vp)]),
    "tcsdn_destroy": (None, [_vp]),
    "tcsdn_model_kind": (C.c_int, [_vp]),
    "tcsdn_model_n_features": (C.c_int, [_vp]),
    "tcsdn_model_score_cols": (C.c_int, [_vp]),
    "tcsdn_set_option": (C.c_int, [_vp, C.c_int32, C.c_int64]),
    "tcsdn_model_stats": (C.c_int, [_vp, _i64p]),
    "tcsdn_predict": (C.c_int, [_vp, _vp, C.c_int64, C.c_int32, C.c_int32, C.c_int32, _vp, _vp, _vp]),
    "tcsdn_knn_kneighbors": (C.c_int, [_vp, _vp, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _vp, _vp, _vp]),
    "tcsdn_take_labels": (C.c_int, [_vp, C.c_int64, _vp, C.c_int32, C.c_int32, _vp, C.c_int32]),
    "tcsdn_sync_check": (C.c_int, [_vp, _vp]),
    "tcsdn_svc_ovr_from_ovo": (C.c_int, [_vp, C.c_int64, C.c_int32, C.c_int32, _vp, _vp]),
    "tcsdn_flow_update": (C.c_int, [_vp, _vp, _vp, _vp, _vp, C.c_int64, _vp, C.c_int32, _vp]),
    "tcsdn_gnb_fit": (C.c_int, [_vp, _vp, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_double, _f64p, _f64p,
                                _f64p, _f64p, _f64p, _vp]),
    "tcsdn_kmeans_fit": (C.c_int, [_vp, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _f64p, C.c_int32, C.c_double,
                                   _f64p, _vp, _f64p, _i32p, _vp]),
    "tcsdn_comm_unique_id": (C.c_int, [_vp]),
    "tcsdn_comm_init": (C.c_int, [C.c_int32, C.c_int32, _vp, C.POINTER(_vp)]),
    "tcsdn_allgather_labels": (C.c_int, [_vp, _vp, C.c_int64, C.c_int64, _vp, _vp]),
    "tcsdn_allgather_labels_u8": (C.c_int, [_vp, _vp, C.c_int64, C.c_int64, _vp, C.c_int32, _vp]),
    "tcsdn_comm_gather_buffer": (C.c_int, [_vp, C.c_int64, C.POINTER(_vp), _i64p]),
    "tcsdn_predict_gathered": (C.c_int, [_vp, _vp, _vp, C.c_int64, C.c_int32, C.c_int32, C.POINTER(_vp), _vp]),
    "tcsdn_comm_destroy": (None, [_vp]),
}

_lib = None


class TcsdnError(RuntimeError):
    pass


def load():
    """Load libtcsdn.so (built in-tree by traffic_classifier_sdn_b200.build).  Raises if absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise TcsdnError(f"{LIB_PATH} is missing: run `python -m traffic_classifier_sdn_b200.build` "
                         "(there is no CPU fallback)")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the .so does not export what the header declares
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def last_error() -> str:
    return load().tcsdn_last_error().decode("utf-8", "replace")


def check(rc: int):
    if rc == OK:
        return
    msg = last_error()
    if rc in (EINVAL, ENONFINITE):
        raise ValueError(msg)
    if rc == ENOMEM:
        raise MemoryError(msg)
    raise TcsdnError(msg)


def ptr(a: np.ndarray, t=_vp):
    return a.ctypes.data_as(t)


def device_count() -> int:
    n = C.c_int32(0)
    rc = load().tcsdn_device_count(C.byref(n))
    return int(n.value) if rc == OK else 0
