"""ctypes binding of libmadicp_b200.so (include/madicp_b200.h).  Thin: argument marshalling and
error translation only.  The library is built in-tree (mad_icp_b200/lib/) by
`__graft_entry__.build()` / `make -C mad_icp_b200/csrc`; there is no CPU fallback -- if the
shared object or a GPU is missing every compute call raises."""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libmadicp_b200.so")
_lib = None

dp = C.POINTER(C.c_double)
ip = C.POINTER(C.c_int32)
bp = C.POINTER(C.c_uint8)
vp = C.c_void_p


class Points(C.Structure):
    """madicp_points_t: raw sensor records (strided x/y/z fields) + the dataset readers' range gate."""
    _fields_ = [("data", C.c_void_p), ("n", C.c_int64), ("stride", C.c_int64), ("offset", C.c_int32 * 3),
                ("is_f32", C.c_int32), ("min_range", C.c_double), ("max_range", C.c_double), ("range_mode", C.c_int32),
                ("drop_nan", C.c_int32)]


assert C.sizeof(Points) == 64
pts_p = C.POINTER(Points)


class Vcorr(C.Structure):
    """madicp_vcorr_t: KITTI's vertical-angle correction of the kept points (enabled != 0)."""
    _fields_ = [("angle", C.c_double), ("enabled", C.c_int32), ("reserved", C.c_int32)]


vc_p = C.POINTER(Vcorr)

# every symbol include/madicp_b200.h and include/madicp_b200_debug.h declare: name -> (restype, argtypes)
SYMBOLS = {
    "madicp_last_error": (C.c_char_p, []),
    "madicp_abi_version": (C.c_int, []),
    "madtree_build": (C.c_int, [dp, C.c_int64, C.c_double, C.c_double, C.c_int, C.POINTER(vp)]),
    "madtree_free": (None, [vp]),
    "madtree_num_nodes": (C.c_int, [vp]),
    "madtree_num_leaves": (C.c_int, [vp]),
    "madtree_apply_transform": (C.c_int, [vp, dp]),
    "madtree_leaves": (C.c_int, [vp, dp, dp, dp, ip]),
    "madtree_records": (vp, [vp]),
    "madtree_num_levels": (C.c_int, [vp]),
    "madtree_level_offsets": (C.c_int, [vp, ip, C.c_int]),
    "madtree_leaf_records": (C.c_int, [vp, ip]),
    "madtree_export": (C.c_int, [vp, dp, dp, dp, ip, ip, ip, ip]),
    "madicp_create": (C.c_int, [C.POINTER(vp), C.c_int, C.c_int]),
    "madicp_destroy": (None, [vp]),
    "madicp_set_params": (C.c_int, [vp, C.c_double, C.c_double, C.c_double]),
    "madicp_set_stream": (C.c_int, [vp, vp]),
    "madicp_get_stream": (vp, [vp]),
    "madicp_put_keyframe": (C.c_int, [vp, C.c_int, vp]),
    "madicp_put_keyframe_transformed": (C.c_int, [vp, C.c_int, vp, dp]),
    "madicp_put_keyframe_records": (C.c_int, [vp, C.c_int, vp, C.c_int, C.c_int]),
    "madicp_put_keyframe_tree": (C.c_int, [vp, C.c_int, vp, dp]),
    "madicp_synchronize": (C.c_int, [vp]),
    "madtree_gpu_build": (C.c_int, [vp, dp, C.c_int64, C.c_double, C.c_double, C.POINTER(vp)]),
    "madtree_gpu_build_resident": (C.c_int, [vp, C.c_double, C.c_double, C.POINTER(vp)]),
    "madtree_gpu_build_batch": (C.c_int, [vp, C.POINTER(vp), C.POINTER(C.c_int64), C.c_int, C.c_int, C.c_double, C.c_double,
                                          C.POINTER(vp)]),
    "madicp_stage_cloud": (C.c_int, [vp, vp, C.c_int64, C.c_int, C.c_int64]),
    "madicp_stage_discard": (C.c_int, [vp]),
    "madtree_gpu_upload": (C.c_int, [vp, vp, C.POINTER(vp)]),
    "madtree_gpu_free": (None, [vp]),
    "madtree_gpu_num_nodes": (C.c_int, [vp]),
    "madtree_gpu_num_leaves": (C.c_int, [vp]),
    "madtree_gpu_num_levels": (C.c_int, [vp]),
    "madtree_gpu_download": (C.c_int, [vp, vp, ip]),
    "madtree_gpu_export": (C.c_int, [vp, dp, dp, dp, ip]),
    "madicp_set_moving_tree": (C.c_int, [vp, vp]),
    "madicp_get_moving": (C.c_int, [vp, dp, C.c_int]),
    "madicp_ingest": (C.c_int, [vp, vp, C.c_int64, C.c_int, C.c_int, dp, dp, C.c_double, C.c_int, dp]),
    "madicp_ingest_points": (C.c_int, [vp, pts_p, C.c_int, dp, dp, C.c_double, C.c_int, C.POINTER(C.c_int64), dp]),
    "madicp_stage_points": (C.c_int, [vp, pts_p, C.c_int64]),
    "madtree_gpu_build_batch_points": (C.c_int, [vp, pts_p, C.c_int, C.c_double, C.c_double, C.POINTER(vp)]),
    "madicp_debug_range_mask": (C.c_int64, [pts_p, bp]),
    "madicp_ingest_points_ex": (C.c_int, [vp, pts_p, vc_p, C.c_int, dp, dp, C.c_double, C.c_int, C.POINTER(C.c_int64), dp]),
    "madicp_stage_points_ex": (C.c_int, [vp, pts_p, vc_p, C.c_int64]),
    "madtree_gpu_build_batch_points_ex": (C.c_int, [vp, pts_p, vc_p, C.c_int, C.c_double, C.c_double, C.POINTER(vp)]),
    "madicp_debug_correct_points": (C.c_int64, [pts_p, vc_p, dp]),
    "madicp_plan_points": (C.c_int, [vp, pts_p, vc_p, C.c_int, C.POINTER(vp)]),
    "madicp_ingest_plan": (C.c_int, [vp, vp, C.c_int, dp, dp, C.c_double, C.POINTER(C.c_int64), dp]),
    "madicp_plan_free": (None, [vp]),
    "madicp_ingest_points_dev": (C.c_int, [vp, pts_p, vc_p, C.c_int, dp, dp, C.c_double, C.c_int, vp, C.POINTER(C.c_int64),
                                           dp]),
    "madtree_gpu_build_batch_points_dev": (C.c_int, [vp, pts_p, vc_p, C.c_int, C.c_double, C.c_double, vp, C.POINTER(vp)]),
    "madicp_plan_points_dev": (C.c_int, [vp, pts_p, vc_p, C.c_int, vp, C.POINTER(vp)]),
    "madicp_search_cloud_dev": (C.c_int, [vp, C.c_int, vp, C.c_int64, C.c_int64, C.c_int, vp, vp, vp, vp, vp]),
    "madicp_debug_deskew_plan": (C.c_int, [pts_p, vc_p, dp, dp, C.c_double, C.c_int, C.c_int, ip,
                                           C.POINTER(C.c_uint16), dp, C.POINTER(C.c_int), C.POINTER(C.c_int64)]),
    "madicp_register_fetch_weight": (C.c_int, [vp, dp, dp, dp, bp, C.POINTER(C.c_int), dp]),
    "madicp_register_partial_async": (C.c_int, [vp, C.c_int, dp]),
    "madicp_calibrate": (C.c_int, [vp, dp]),
    "madicp_drop_keyframe": (C.c_int, [vp, C.c_int]),
    "madicp_num_keyframes": (C.c_int, [vp]),
    "madicp_active_slots": (C.c_int, [vp, ip, C.c_int]),
    "madicp_keyframe_leaves": (C.c_int, [vp, C.c_int]),
    "madicp_set_moving": (C.c_int, [vp, vp, C.c_int]),
    "madicp_search": (C.c_int, [vp, dp, ip]),
    "madicp_linearize": (C.c_int, [vp, dp, dp, dp, bp]),
    "madicp_solve_update": (C.c_int, [vp, dp, dp, dp]),
    "madicp_register": (C.c_int, [vp, C.c_int, dp, dp, dp, bp, C.POINTER(C.c_int)]),
    "madicp_register_async": (C.c_int, [vp, C.c_int, dp]),
    "madicp_register_fetch": (C.c_int, [vp, dp, dp, dp, bp, C.POINTER(C.c_int)]),
    "madicp_register_trace": (C.c_int, [vp, dp, C.c_int]),
    "madicp_register_walked": (C.c_int, [vp, ip, C.c_int]),
    "madicp_register_walk_records": (C.c_int, [vp, C.POINTER(C.c_int64), C.c_int]),
    "madicp_search_cloud": (C.c_int, [vp, C.c_int, dp, C.c_int64, ip, dp, dp, dp]),
    "madicp_deskew": (C.c_int, [dp, C.c_int64, dp, dp, C.c_double, C.c_int]),
    "madicp_debug_sort_check": (C.c_int64, [C.c_int64, C.c_uint32, C.c_int64, C.c_int]),
    "madicp_kernel_launches": (C.c_int64, [vp]),
    "madicp_model_nodes": (C.c_int64, [vp]),
    "madicp_comm_export": (C.c_int, [vp, vp]),
    "madicp_comm_connect": (C.c_int, [vp, C.c_int, C.c_int, vp]),
    "madicp_comm_world": (C.c_int, [vp]),
    "madicp_debug_timing": (C.c_int, [vp, C.c_int, C.POINTER(C.c_int64), C.c_int]),
    "madicp_debug_cta_cycles": (C.c_int, [vp, C.POINTER(C.c_int64), C.c_int]),
    "madicp_set_gn_grid": (C.c_int, [vp, C.c_int, C.c_int]),
    "madicp_debug_gn_stretch": (C.c_int, [C.c_int64, C.c_int, C.c_int, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]),
    "madicp_debug_gn_map_bytes": (C.c_int64, [C.c_int, C.c_int64, C.c_int]),
    "madicp_debug_set_memo": (C.c_int, [vp, C.c_int]),
    "madicp_debug_inv_det6": (C.c_int, [vp, dp, dp]),
    "madicp_debug_cta_stamps": (C.c_int, [vp, C.c_int, C.POINTER(C.c_int64), C.c_int]),
}

REC_DTYPE = np.dtype([("mean", "<f8", 3), ("dir", "<f8", 3), ("bbox0", "<f8"), ("link", "<i4"), ("num_points", "<i4")])
assert REC_DTYPE.itemsize == 64


class MadIcpError(RuntimeError):
    pass


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise MadIcpError(
                f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(make -C mad_icp_b200/csrc).  There is no CPU fallback.")
        L = C.CDLL(LIB_PATH)
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(L, name)  # AttributeError if the .so does not export a declared symbol
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def check(rc, what=""):
    if rc < 0:
        msg = lib().madicp_last_error()
        raise MadIcpError(f"{what} failed ({rc}): {msg.decode() if msg else ''}")
    return rc


def as_d(a):
    return a.ctypes.data_as(dp) if a is not None else None


def as_i(a):
    return a.ctypes.data_as(ip) if a is not None else None


def as_b(a):
    return a.ctypes.data_as(bp) if a is not None else None


def pose12(T):
    """4x4 / 3x4 pose -> contiguous 3x4 row-major [R|t] float64 (the ABI's pose layout)."""
    T = np.asarray(T, dtype=np.float64)
    if T.shape == (4, 4):
        T = T[:3, :]
    if T.shape != (3, 4):
        raise ValueError("pose must be 4x4 or 3x4")
    return np.ascontiguousarray(T)
