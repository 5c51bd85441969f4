"""ctypes driver for the CPU oracle (oracle/_build/libmadicp_oracle.so).

TEST INFRASTRUCTURE -- only tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs import this.  Parity status: pinned bit for bit to the
reference's own sources compiled against oracle/eigen_standin (oracle/reference.py,
tests/test_reference_pin.py); Eigen's internal evaluation order is unpinned.  See
oracle/madicp_oracle.hpp for the statement-by-statement citations.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_build", "libmadicp_oracle.so")
_lib = None

_dp = C.POINTER(C.c_double)
_ip = C.POINTER(C.c_int)
_bp = C.POINTER(C.c_ubyte)


def build(force=False):
    """Compile the restatement with oracle/Makefile (gcc only, no GPU needed)."""
    srcs = ("oracle_capi.cpp", "madicp_oracle.hpp", "pipeline_oracle.hpp", "Makefile")
    src_m = max(os.path.getmtime(os.path.join(_HERE, f)) for f in srcs)
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < src_m:
        subprocess.check_call(["make", "-C", _HERE, "-s"])
    return _SO


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_SO):
            build()
        L = C.CDLL(_SO)
        L.orc_tree_build.restype = C.c_void_p
        L.orc_tree_build.argtypes = [_dp, C.c_int, C.c_double, C.c_double]
        L.orc_tree_free.argtypes = [C.c_void_p]
        L.orc_tree_num_leaves.argtypes = [C.c_void_p]
        L.orc_tree_num_nodes.argtypes = [C.c_void_p]
        L.orc_tree_cloud.argtypes = [C.c_void_p, _dp]
        L.orc_tree_apply_transform.argtypes = [C.c_void_p, _dp]
        L.orc_tree_leaves.argtypes = [C.c_void_p, _dp, _dp, _dp, _ip]
        L.orc_tree_export.argtypes = [C.c_void_p, _dp, _dp, _dp, _ip, _ip, _ip, _ip]
        L.orc_tree_search.argtypes = [C.c_void_p, _dp, C.c_int, _ip, _ip]
        L.orc_icp_run.restype = C.c_double
        L.orc_icp_run.argtypes = [C.POINTER(C.c_void_p), C.c_int, C.c_void_p, _dp, C.c_int, C.c_double, C.c_double,
                                  C.c_double, C.c_int, _dp, _dp, _dp, _dp, _ip, _bp]
        L.orc_icp_linearize.argtypes = [C.POINTER(C.c_void_p), C.c_int, C.c_void_p, _dp, C.c_double, C.c_double,
                                        C.c_double, _dp, _dp, _bp]
        L.orc_solve_update.argtypes = [_dp, _dp, _dp, _dp, _dp]
        L.orc_eig3.argtypes = [_dp, _dp, _dp]
        L.orc_expmap.argtypes = [_dp, _dp]
        L.orc_max_threads.restype = C.c_int
        _lib = L
    return _lib


def _d(a):
    return a.ctypes.data_as(_dp) if a is not None else None


def _i(a):
    return a.ctypes.data_as(_ip) if a is not None else None


def _b(a):
    return a.ctypes.data_as(_bp) if a is not None else None


def _pose12(T):
    T = np.asarray(T, dtype=np.float64)
    if T.shape == (4, 4):
        T = T[:3, :]
    return np.ascontiguousarray(T.reshape(3, 4))


class OracleTree:
    """MADtree restatement (tools/mad_tree.{h,cpp}); leaves are in getLeafs DFS order."""

    def __init__(self, points, b_max=0.2, b_min=0.1):
        pts = np.ascontiguousarray(points, dtype=np.float64).reshape(-1, 3)
        assert pts.shape[0] > 0, "the reference dereferences *begin on an empty cloud (UB); refuse"
        self._h = C.c_void_p(lib().orc_tree_build(_d(pts), pts.shape[0], b_max, b_min))
        self.n_points = pts.shape[0]
        self.b_max, self.b_min = b_max, b_min

    def __del__(self):
        if getattr(self, "_h", None):
            lib().orc_tree_free(self._h)
            self._h = None

    @property
    def num_leaves(self):
        return lib().orc_tree_num_leaves(self._h)

    @property
    def num_nodes(self):
        return lib().orc_tree_num_nodes(self._h)

    def cloud(self):
        out = np.empty((self.n_points, 3))
        lib().orc_tree_cloud(self._h, _d(out))
        return out

    def apply_transform(self, T):
        X = _pose12(T)
        lib().orc_tree_apply_transform(self._h, _d(X))

    def leaves(self):
        L = self.num_leaves
        means, normals = np.empty((L, 3)), np.empty((L, 3))
        bbox0, npts = np.empty(L), np.empty(L, dtype=np.int32)
        lib().orc_tree_leaves(self._h, _d(means), _d(normals), _d(bbox0), _i(npts))
        return means, normals, bbox0, npts

    def export(self):
        n = self.num_nodes
        out = dict(mean=np.empty((n, 3)), eivecs=np.empty((n, 9)), bbox=np.empty((n, 3)),
                   num_points=np.empty(n, np.int32), left=np.empty(n, np.int32), right=np.empty(n, np.int32),
                   leaf_ordinal=np.empty(n, np.int32))
        lib().orc_tree_export(self._h, _d(out["mean"]), _d(out["eivecs"]), _d(out["bbox"]), _i(out["num_points"]),
                              _i(out["left"]), _i(out["right"]), _i(out["leaf_ordinal"]))
        return out

    def search(self, queries, want_depth=False):
        q = np.ascontiguousarray(queries, dtype=np.float64).reshape(-1, 3)
        idx = np.empty(q.shape[0], np.int32)
        dep = np.empty(q.shape[0], np.int32) if want_depth else None
        lib().orc_tree_search(self._h, _d(q), q.shape[0], _i(idx), _i(dep))
        return (idx, dep) if want_depth else idx


def _handles(trees):
    arr = (C.c_void_p * len(trees))(*[t._h for t in trees])
    return arr


def icp_run(keyframes, moving, X0, iters=15, min_ball=0.2, rho_ker=0.1, b_ratio=0.02, num_threads=1, record=True,
            record_matches=True):
    """pipeline.cpp:166-193 / mad_icp_wrapper.h:72-81.  Returns dict with X (3x4), seconds and recordings."""
    K, L = len(keyframes), moving.num_leaves
    X0 = _pose12(X0)
    Xf = np.empty((3, 4))
    Xh = np.empty((iters, 3, 4)) if record else None
    Hh = np.empty((iters, 36)) if record else None
    bh = np.empty((iters, 6)) if record else None
    ih = np.empty((iters, K, L), np.int32) if (record and record_matches) else None
    m = np.empty(L, np.uint8)
    secs = lib().orc_icp_run(_handles(keyframes), K, moving._h, _d(X0), iters, min_ball, rho_ker, b_ratio, num_threads,
                             _d(Xf), _d(Xh), _d(Hh), _d(bh), _i(ih), _b(m))
    out = dict(X=Xf, seconds=secs, matched=m)
    if record:
        out.update(X_hist=Xh, H_hist=Hh.reshape(iters, 6, 6).transpose(0, 2, 1).copy(), b_hist=bh, idx_hist=ih)
    return out


def icp_linearize(keyframes, moving, X, min_ball=0.2, rho_ker=0.1, b_ratio=0.02):
    X = _pose12(X)
    H, b = np.empty(36), np.empty(6)
    m = np.empty(moving.num_leaves, np.uint8)
    lib().orc_icp_linearize(_handles(keyframes), len(keyframes), moving._h, _d(X), min_ball, rho_ker, b_ratio, _d(H),
                            _d(b), _b(m))
    return H.reshape(6, 6).T.copy(), b, m


def solve_update(H, b, X):
    Hc = np.ascontiguousarray(np.asarray(H, dtype=np.float64).T).reshape(36)  # col-major
    bb = np.ascontiguousarray(b, dtype=np.float64)
    X = _pose12(X)
    dx, Xo = np.empty(6), np.empty((3, 4))
    lib().orc_solve_update(_d(Hc), _d(bb), _d(X), _d(dx), _d(Xo))
    return dx, Xo


def inverse_determinant(H):
    """The keyframe weight det(H^-1) of pipeline.cpp:223 (pipeline_oracle.hpp inverseDeterminant6)."""
    H = np.ascontiguousarray(H, dtype=np.float64).reshape(36)
    fn = lib().orc_inverse_determinant6
    fn.restype, fn.argtypes = C.c_double, [_dp]
    return fn(_d(H))


def eig3(cov):
    c = np.ascontiguousarray(np.asarray(cov, dtype=np.float64).T).reshape(9)
    ev, ew = np.empty(9), np.empty(3)
    lib().orc_eig3(_d(c), _d(ev), _d(ew))
    return ew, ev.reshape(3, 3).T.copy()


def expmap(w):
    w = np.ascontiguousarray(w, dtype=np.float64)
    R = np.empty((3, 3))
    lib().orc_expmap(_d(w), _d(R))
    return R


def max_threads():
    return lib().orc_max_threads()


def deskew(points, T_prev, T_now, sensor_hz=10.0):
    """Pipeline::deskew (odometry/pipeline.cpp:79-123) of the CPU restatement; returns the deskewed copy."""
    L = lib()
    L.orc_pipeline_create.restype = C.c_void_p
    L.orc_pipeline_create.argtypes = [C.c_double, C.c_int, C.c_double, C.c_double, C.c_double, C.c_double, C.c_double,
                                      C.c_int, C.c_int, C.c_int]
    L.orc_pipeline_deskew.argtypes = [C.c_void_p, _dp, C.c_int, _dp, _dp]
    L.orc_pipeline_free.argtypes = [C.c_void_p]
    po = C.c_void_p(L.orc_pipeline_create(float(sensor_hz), 1, 0.2, 0.1, 0.8, 0.1, 0.02, 4, 1, 0))
    out = np.ascontiguousarray(points, dtype=np.float64).copy()
    L.orc_pipeline_deskew(po, _d(out), out.shape[0], _d(_pose12(T_prev)), _d(_pose12(T_now)))
    L.orc_pipeline_free(po)
    return out


class OraclePipeline:
    """The CPU restatement of the reference's Pipeline (odometry/pipeline.{h,cpp}); state() as orc_pipeline_state:
    pose 3x4 (12), is_map_updated, current id, keyframe id, number of keyframes, inlier ratio, velocity (6)."""

    def __init__(self, sensor_hz=10.0, deskew=False, b_max=0.2, rho_ker=0.1, p_th=0.8, b_min=0.1, b_ratio=0.02,
                 num_keyframes=4, num_threads=4, realtime=False):
        L = lib()
        L.orc_pipeline_create.restype = C.c_void_p
        L.orc_pipeline_create.argtypes = [C.c_double, C.c_int, C.c_double, C.c_double, C.c_double, C.c_double, C.c_double,
                                          C.c_int, C.c_int, C.c_int]
        L.orc_pipeline_compute.argtypes = [C.c_void_p, C.c_double, _dp, C.c_int]
        L.orc_pipeline_state.argtypes = [C.c_void_p, _dp]
        L.orc_pipeline_free.argtypes = [C.c_void_p]
        self._h = C.c_void_p(L.orc_pipeline_create(sensor_hz, int(deskew), b_max, rho_ker, p_th, b_min, b_ratio,
                                                   num_keyframes, num_threads, int(realtime)))

    def __del__(self):
        if getattr(self, "_h", None):
            lib().orc_pipeline_free(self._h)
            self._h = None

    def compute(self, stamp, pts):
        pts = np.ascontiguousarray(pts, dtype=np.float64)
        lib().orc_pipeline_compute(self._h, float(stamp), _d(pts), pts.shape[0])

    def state(self):
        st = np.zeros(23)
        lib().orc_pipeline_state(self._h, _d(st))
        return st
