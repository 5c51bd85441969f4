"""ctypes driver for the compiled reference (oracle/_ref/libmadicp_ref.so).

TEST INFRASTRUCTURE.  The library is the reference's OWN sources (tools/mad_tree.cpp,
odometry/mad_icp.cpp, odometry/pipeline.cpp, odometry/vel_estimator.cpp) compiled where they lie under
REF_SRC (the reference checkout's mad_icp/src) against oracle/eigen_standin, plus oracle/ref_capi.cpp.  It exists
to pin the restatement (oracle/oracle.py: tests/golden/make_reference_pin.py records its outputs) and as the timed
CPU arm of bench.py.  It is built only where the reference sources are; the built file is git-ignored.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from .oracle import _b, _d, _dp, _i, _ip, _bp, _pose12

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_ref", "libmadicp_ref.so")
# where the reference checkout's mad_icp/src lies: $MADICP_REFERENCE_SRC, by default /root/reference/mad_icp/src
REF_SRC = os.environ.get("MADICP_REFERENCE_SRC", "/root/reference/mad_icp/src")
_lib = None


def available():
    return os.path.exists(_SO) or os.path.isdir(REF_SRC)


def build(force=False):
    """`make ref` in oracle/ (needs the reference sources at REF_SRC; a no-op when the prebuilt library is current)."""
    if not os.path.isdir(REF_SRC):
        if os.path.exists(_SO):
            return _SO
        raise RuntimeError("reference sources not present and no prebuilt oracle/_ref library")
    if force and os.path.exists(_SO):
        os.remove(_SO)
    subprocess.check_call(["make", "-C", _HERE, "-s", "ref"])
    return _SO


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_SO):
            build()
        L = C.CDLL(_SO)
        L.ref_tree_build.restype = C.c_void_p
        L.ref_tree_build.argtypes = [_dp, C.c_int, C.c_double, C.c_double, C.c_int]
        L.ref_tree_free.argtypes = [C.c_void_p]
        L.ref_tree_num_leaves.argtypes = [C.c_void_p]
        L.ref_tree_num_nodes.argtypes = [C.c_void_p]
        L.ref_tree_cloud.argtypes = [C.c_void_p, _dp]
        L.ref_tree_apply_transform.argtypes = [C.c_void_p, _dp]
        L.ref_tree_export.argtypes = [C.c_void_p, _dp, _dp, _dp, _ip, _ip, _ip, _ip]
        L.ref_tree_search.argtypes = [C.c_void_p, _dp, C.c_int, _ip]
        L.ref_icp_run.restype = C.c_double
        L.ref_icp_run.argtypes = [C.POINTER(C.c_void_p), C.c_int, C.c_void_p, _dp, C.c_int, C.c_double, C.c_double,
                                  C.c_double, C.c_int, _dp, _dp, _dp, _dp, _bp, _ip]
        L.ref_pipeline_create.restype = C.c_void_p
        L.ref_pipeline_create.argtypes = [C.c_double, C.c_int, C.c_double, C.c_double, C.c_double, C.c_double,
                                          C.c_double, C.c_int, C.c_int, C.c_int]
        L.ref_pipeline_free.argtypes = [C.c_void_p]
        L.ref_pipeline_compute.argtypes = [C.c_void_p, C.c_double, _dp, C.c_int]
        L.ref_pipeline_state.argtypes = [C.c_void_p, _dp]
        L.ref_pipeline_deskew.argtypes = [C.c_void_p, _dp, C.c_int, _dp, _dp]
        L.ref_max_threads.restype = C.c_int
        _lib = L
    return _lib


# The Pipeline probe's list entry points (oracle/ref_capi.cpp).  They are resolved on first use rather than in lib(): a
# library built before they existed, where the reference sources are not at hand to rebuild it, still serves every
# other caller, and has_probe() tells the callers that need them.
PROBE = {"ref_pipeline_frames": [C.c_void_p, _ip, _dp], "ref_pipeline_keyframes": [C.c_void_p, _ip],
         "ref_pipeline_leaves": [C.c_void_p, C.c_int, _dp], "ref_pipeline_trajectory": [C.c_void_p, _dp]}


def has_probe():
    """Whether the library exports the Pipeline probe's list entry points (frames, keyframes, leaves, trajectory) and
    reports the inlier ratio in state()[16]."""
    return all(hasattr(lib(), name) for name in PROBE)


def exports_probe(path):
    """has_probe() of the library file at `path`, without loading it (build() rebuilds a library that predates them)."""
    with open(path, "rb") as f:
        data = f.read()
    return all(name.encode() + b"\0" in data for name in PROBE)


def _probe(name):
    fn = getattr(lib(), name, None)
    if fn is None:
        raise RuntimeError(f"{_SO} predates the Pipeline probe ({name}); rebuild it where the reference sources are "
                           "(make -C oracle ref / ref_gpu)")
    fn.restype, fn.argtypes = C.c_int, PROBE[name]
    return fn


class ReferenceTree:
    """The reference's MADtree (tools/mad_tree.{h,cpp}), built by its own constructor."""

    def __init__(self, points, b_max=0.2, b_min=0.1, max_parallel_level=0):
        pts = np.ascontiguousarray(points, dtype=np.float64).reshape(-1, 3)
        assert pts.shape[0] > 0
        self._h = C.c_void_p(lib().ref_tree_build(_d(pts), pts.shape[0], b_max, b_min, max_parallel_level))
        self.n_points = pts.shape[0]

    def __del__(self):
        if getattr(self, "_h", None):
            lib().ref_tree_free(self._h)
            self._h = None

    @property
    def num_leaves(self):
        return lib().ref_tree_num_leaves(self._h)

    @property
    def num_nodes(self):
        return lib().ref_tree_num_nodes(self._h)

    def cloud(self):
        out = np.empty((self.n_points, 3))
        lib().ref_tree_cloud(self._h, _d(out))
        return out

    def apply_transform(self, T):
        lib().ref_tree_apply_transform(self._h, _d(_pose12(T)))

    def export(self):
        n = self.num_nodes
        out = dict(mean=np.empty((n, 3)), eivecs=np.empty((n, 9)), bbox=np.empty((n, 3)),
                   num_points=np.empty(n, np.int32), left=np.empty(n, np.int32), right=np.empty(n, np.int32),
                   leaf_ordinal=np.empty(n, np.int32))
        lib().ref_tree_export(self._h, _d(out["mean"]), _d(out["eivecs"]), _d(out["bbox"]), _i(out["num_points"]),
                              _i(out["left"]), _i(out["right"]), _i(out["leaf_ordinal"]))
        return out

    def search(self, queries):
        q = np.ascontiguousarray(queries, dtype=np.float64).reshape(-1, 3)
        idx = np.empty(q.shape[0], np.int32)
        lib().ref_tree_search(self._h, _d(q), q.shape[0], _i(idx))
        return idx


def icp_run(keyframes, moving, X0, iters=15, min_ball=0.2, rho_ker=0.1, b_ratio=0.02, num_threads=1, record=True,
            record_idx=False):
    """The loop of pipeline.cpp:166-193 over the reference's MADicp; same outputs as oracle.icp_run.
    record_idx: also idx_hist[it, k, q] = getLeafs ordinal of the leaf the reference's bestMatchingLeafFast
    returns for moving leaf q in keyframe k at the pose of round `it` (computed outside the timed region)."""
    K, L = len(keyframes), moving.num_leaves
    X0 = _pose12(X0)
    Xf = np.empty((3, 4))
    Xh = np.empty((iters, 3, 4)) if record else None
    Hh = np.empty((iters, 36)) if record else None
    bh = np.empty((iters, 6)) if record else None
    m = np.empty(L, np.uint8)
    ih = np.empty((iters, K, L), np.int32) if record_idx else None
    arr = (C.c_void_p * K)(*[t._h for t in keyframes])
    secs = lib().ref_icp_run(arr, K, moving._h, _d(X0), iters, min_ball, rho_ker, b_ratio, num_threads, _d(Xf), _d(Xh),
                             _d(Hh), _d(bh), _b(m), _i(ih))
    out = dict(X=Xf, seconds=secs, matched=m)
    if record_idx:
        out["idx_hist"] = ih
    if record:
        out.update(X_hist=Xh, H_hist=Hh.reshape(iters, 6, 6).transpose(0, 2, 1).copy(), b_hist=bh)
    return out


class ReferencePipeline:
    """The reference's Pipeline (odometry/pipeline.{h,cpp}); state() as orc_pipeline_state, with the inlier ratio of
    pipeline.cpp:197-204 recounted from the current leaves' flags (NaN before the first registration, and from a
    library that predates the probe: has_probe()).  frames(), keyframes(), current_leaves(), model_leaves() and
    trajectory() need the probe."""

    def __init__(self, sensor_hz=10.0, deskew=False, b_max=0.2, rho_ker=0.1, p_th=0.8, b_min=0.1, b_ratio=0.02,
                 num_keyframes=4, num_threads=4, realtime=False):
        self._h = C.c_void_p(lib().ref_pipeline_create(sensor_hz, int(deskew), b_max, rho_ker, p_th, b_min, b_ratio,
                                                       num_keyframes, num_threads, int(realtime)))

    def __del__(self):
        if getattr(self, "_h", None):
            lib().ref_pipeline_free(self._h)
            self._h = None

    def compute(self, stamp, pts):
        pts = np.ascontiguousarray(pts, dtype=np.float64)
        lib().ref_pipeline_compute(self._h, float(stamp), _d(pts), pts.shape[0])

    def state(self):
        st = np.zeros(23)
        lib().ref_pipeline_state(self._h, _d(st))
        return st

    def frames(self):
        """The frames window (frames_, oldest first): frame ids (int32) and weights det(H^-1)."""
        n = _probe("ref_pipeline_frames")(self._h, None, None)
        ids, w = np.empty(n, np.int32), np.empty(n)
        _probe("ref_pipeline_frames")(self._h, _i(ids), _d(w))
        return ids, w

    def keyframes(self):
        """keyframes_ in their order: frame ids (int32)."""
        n = _probe("ref_pipeline_keyframes")(self._h, None)
        ids = np.empty(n, np.int32)
        _probe("ref_pipeline_keyframes")(self._h, _i(ids))
        return ids

    def _leaves(self, model):
        n = _probe("ref_pipeline_leaves")(self._h, int(model), None)
        out = np.empty((n, 3))
        _probe("ref_pipeline_leaves")(self._h, int(model), _d(out))
        return out

    def current_leaves(self):
        """currentLeaves(): the current scan's leaf means in the map frame, N x 3."""
        return self._leaves(False)

    def model_leaves(self):
        """modelLeaves(): every keyframe's leaf means, keyframe after keyframe, N x 3."""
        return self._leaves(True)

    def trajectory(self):
        """trajectory(): n x 4 x 4."""
        n = _probe("ref_pipeline_trajectory")(self._h, None)
        out = np.empty((n, 3, 4))
        _probe("ref_pipeline_trajectory")(self._h, _d(out))
        T = np.zeros((n, 4, 4))
        T[:, :3], T[:, 3, 3] = out, 1.0
        return T

    def deskew(self, pts, T_prev, T_now):
        out = np.ascontiguousarray(pts, dtype=np.float64).copy()
        lib().ref_pipeline_deskew(self._h, _d(out), out.shape[0], _d(_pose12(T_prev)), _d(_pose12(T_now)))
        return out


def max_threads():
    return lib().ref_max_threads()


def inverse_determinant(H):
    """pipeline.cpp:223's keyframe weight, H.inverse().determinant(), evaluated by the reference's own expression.
    Resolved here rather than in lib(): only tests/golden/make_weight_reference.py calls it, and a library built
    before the entry point existed still serves every other caller."""
    H = np.ascontiguousarray(H, dtype=np.float64).reshape(36)
    fn = lib().ref_inverse_determinant
    fn.restype, fn.argtypes = C.c_double, [_dp]
    return fn(_d(H))


def variant(so_name, make_target=None):
    """A second instance of this module over another build of the same C entry points (oracle/ref_capi.cpp), e.g.
    `variant("libmadicp_ref_gpu.so", "ref_gpu")`: the reference's unmodified pipeline.cpp / vel_estimator.cpp linked
    with the product's backend TU instead of its own mad_tree.cpp / mad_icp.cpp (oracle/Makefile)."""
    import importlib.util
    spec = importlib.util.spec_from_file_location(f"oracle.reference__{so_name.replace('.', '_')}", __file__,
                                                  submodule_search_locations=None)
    mod = importlib.util.module_from_spec(spec)
    mod.__package__ = __package__
    spec.loader.exec_module(mod)
    mod._SO = os.path.join(_HERE, "_ref", so_name)
    if make_target and os.path.isdir(REF_SRC):
        subprocess.check_call(["make", "-C", _HERE, "-s", make_target])
    if not os.path.exists(mod._SO):
        raise RuntimeError(f"{mod._SO} is missing (built where the reference sources are, REF_SRC: make -C oracle {make_target})")
    return mod
