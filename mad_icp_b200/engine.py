"""Python handles over the C ABI: `FlatTree` (host-built MAD-tree in the breadth-first device layout)
and `Registrar` (one GPU: keyframe slots + moving leaves + the persistent Gauss-Newton kernel).
These are the objects the reference-named facade (mad_icp_b200.api / the pybind modules) and
bench.py drive; they add no arithmetic of their own."""
import ctypes as C
import math

import numpy as np

from . import _capi as capi
from ._capi import MadIcpError, as_b, as_d, as_i, check, pose12
from .records import VERTICAL_ANGLE_OFFSET, describe, describe_times, vcorr


class FlatTree:
    """MADtree built on the host (reference: tools/mad_tree.cpp:47-130) in flat form."""

    def __init__(self, points, b_max=0.2, b_min=0.1, num_threads=1):
        pts = np.ascontiguousarray(points, dtype=np.float64)
        if pts.ndim != 2 or pts.shape[1] != 3:
            raise ValueError("points must be N x 3")
        h = C.c_void_p()
        check(capi.lib().madtree_build(as_d(pts), pts.shape[0], b_max, b_min, num_threads, C.byref(h)), "madtree_build")
        self._h = h
        self.b_max, self.b_min = b_max, b_min

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            self._h = None
            try:
                capi.lib().madtree_free(h)
            except TypeError:  # interpreter shutdown
                pass

    @property
    def num_nodes(self):
        return capi.lib().madtree_num_nodes(self._h)

    @property
    def num_leaves(self):
        return capi.lib().madtree_num_leaves(self._h)

    def apply_transform(self, T):
        X = pose12(T)
        check(capi.lib().madtree_apply_transform(self._h, as_d(X)), "madtree_apply_transform")

    def leaves(self):
        L = self.num_leaves
        means, normals = np.empty((L, 3)), np.empty((L, 3))
        bbox0, npts = np.empty(L), np.empty(L, np.int32)
        check(capi.lib().madtree_leaves(self._h, as_d(means), as_d(normals), as_d(bbox0), as_i(npts)))
        return means, normals, bbox0, npts

    def leaf_means(self):
        means = np.empty((self.num_leaves, 3))
        check(capi.lib().madtree_leaves(self._h, as_d(means), None, None, None))
        return means

    def records(self):
        """Copy of the breadth-first 64-byte records as a structured array."""
        n = self.num_nodes
        ptr = capi.lib().madtree_records(self._h)
        buf = (C.c_char * (n * 64)).from_address(ptr)
        return np.frombuffer(buf, dtype=capi.REC_DTYPE, count=n).copy()

    def export(self):
        n = self.num_nodes
        out = dict(mean=np.empty((n, 3)), eivecs=np.empty((n, 9)), bbox=np.empty((n, 3)),
                   num_points=np.empty(n, np.int32), left=np.empty(n, np.int32), right=np.empty(n, np.int32),
                   leaf_ordinal=np.empty(n, np.int32))
        check(capi.lib().madtree_export(self._h, as_d(out["mean"]), as_d(out["eivecs"]), as_d(out["bbox"]),
                                        as_i(out["num_points"]), as_i(out["left"]), as_i(out["right"]),
                                        as_i(out["leaf_ordinal"])))
        return out


class DeviceTree:
    """A sensor-frame MAD-tree resident in the device memory of one Registrar: built on the device
    (`Registrar.build_tree`) or uploaded from a host-built FlatTree (`Registrar.upload_tree`)."""

    def __init__(self, handle, registrar):
        self._h, self._reg = handle, registrar  # the registrar must outlive the tree

    def __del__(self):
        h = getattr(self, "_h", None)
        if h and getattr(self._reg, "_h", None):
            self._h = None
            try:
                capi.lib().madtree_gpu_free(h)
            except TypeError:
                pass

    num_nodes = property(lambda self: capi.lib().madtree_gpu_num_nodes(self._h))
    num_leaves = property(lambda self: capi.lib().madtree_gpu_num_leaves(self._h))
    num_levels = property(lambda self: capi.lib().madtree_gpu_num_levels(self._h))

    def records(self):
        recs = np.empty(self.num_nodes, dtype=capi.REC_DTYPE)
        check(capi.lib().madtree_gpu_download(self._h, recs.ctypes.data_as(C.c_void_p), None), "madtree_gpu_download")
        return recs

    def leaf_records(self):
        out = np.empty(self.num_leaves, np.int32)
        check(capi.lib().madtree_gpu_download(self._h, None, as_i(out)), "madtree_gpu_download")
        return out

    def leaf_means(self, T=None, device=False):
        """The tree's leaf means in getLeafs order, posed by T (4x4 / 3x4, or None: untouched); see `leaf_means`."""
        return leaf_means([self], [T], device)

    def cloud(self, T=None, device=False):
        """The cloud the tree was built from (`Registrar.keep_cloud`) and the record index of every point: an (N, 3)
        float64 array posed by T (4x4 / 3x4, or None: untouched) and an (N,) int64 array, or with device=True torch
        tensors on the registrar's device, ready on torch's current stream (madtree_gpu_cloud_dev)."""
        n = check(capi.lib().madtree_gpu_num_cloud_points(self._h), "madtree_gpu_num_cloud_points")
        X = None if T is None else pose12(T)
        if not device:
            xyz, idx = np.empty((n, 3)), np.empty(n, np.int64)
            check(capi.lib().madtree_gpu_cloud(self._h, as_d(X), as_d(xyz), idx.ctypes.data_as(C.POINTER(C.c_int64))),
                  "madtree_gpu_cloud")
            return xyz, idx
        import torch
        dev = torch.device("cuda", self._reg.device)
        xyz = torch.empty((n, 3), dtype=torch.float64, device=dev)
        idx = torch.empty(n, dtype=torch.int64, device=dev)
        if n:
            check(capi.lib().madtree_gpu_cloud_dev(self._h, as_d(X), C.c_void_p(xyz.data_ptr()), C.c_void_p(idx.data_ptr()),
                                                   C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)),
                  "madtree_gpu_cloud_dev")
        return xyz, idx

    def release_cloud(self):
        check(capi.lib().madtree_gpu_release_cloud(self._h), "madtree_gpu_release_cloud")

    def export(self):
        """Audit dump of a device-BUILT tree, breadth-first: mean, eivecs (column-major), bbox, num_points."""
        n = self.num_nodes
        out = dict(mean=np.empty((n, 3)), eivecs=np.empty((n, 9)), bbox=np.empty((n, 3)), num_points=np.empty(n, np.int32))
        check(capi.lib().madtree_gpu_export(self._h, as_d(out["mean"]), as_d(out["eivecs"]), as_d(out["bbox"]),
                                            as_i(out["num_points"])), "madtree_gpu_export")
        return out


def leaf_means(trees, poses=None, device=False):
    """Leaf means of DeviceTrees of one Registrar, in getLeafs order, tree after tree, gathered in one launch
    (madtree_gpu_leaf_means): poses[k] (4x4 / 3x4, or None) is applied as MADtree::applyTransform would, a tree without a
    pose is copied untouched.  An (N, 3) float64 numpy array, or with device=True a float64 torch tensor on the
    registrar's device, written in place and ready on torch's current stream (madtree_gpu_leaf_means_dev)."""
    trees = list(trees)
    poses = [None] * len(trees) if poses is None else list(poses)
    if len(poses) != len(trees):
        raise ValueError("leaf_means: one pose (or None) per tree")
    k = len(trees)
    Xs = [None if T is None else pose12(T) for T in poses]
    tab = (C.c_void_p * k)(*[t._h for t in trees])
    xtab = (capi.dp * k)(*[as_d(X) if X is not None else None for X in Xs])
    n = sum(t.num_leaves for t in trees)
    if not device:
        out = np.empty((n, 3))
        check(capi.lib().madtree_gpu_leaf_means(tab, xtab, k, as_d(out)), "madtree_gpu_leaf_means")
        return out
    import torch
    dev = torch.device("cuda", trees[0]._reg.device if trees else 0)
    out = torch.empty((n, 3), dtype=torch.float64, device=dev)
    check(capi.lib().madtree_gpu_leaf_means_dev(tab, xtab, k, C.c_void_p(out.data_ptr()),
                                                C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)),
          "madtree_gpu_leaf_means_dev")
    return out


class DeskewPlan:
    """A future scan handed over for a deskewed look-ahead (`Registrar.plan_records`): its records are on their way to
    the device and its pose-free deskew order is worked out on a host thread.  `Registrar.ingest_plan` consumes it;
    dropping it unconsumed frees it.  It keeps its records alive."""

    def __init__(self, handle, registrar, records):
        self._h, self._reg, self._records = handle, registrar, records  # the registrar must outlive the plan

    def _take(self):
        h, self._h = self._h, None
        if not h:
            raise ValueError("the plan has been consumed or freed")
        return h

    def free(self):
        h = getattr(self, "_h", None)
        if h and getattr(self._reg, "_h", None):
            self._h = None
            try:
                capi.lib().madicp_plan_free(h)
            except TypeError:  # interpreter shutdown
                pass
        self._records = None

    __del__ = free


class VoxelMap:
    """A voxel map of kept clouds on one Registrar (madicp_map_*, `Registrar.voxel_map`): each voxel keeps the first
    points_per_voxel points that reach it, inserts in call order, points in kept-cloud order."""

    def __init__(self, handle, registrar):
        self._h, self._reg = handle, registrar  # the registrar must outlive the map

    def free(self):
        h = getattr(self, "_h", None)
        if h and getattr(self._reg, "_h", None):
            self._h = None
            try:
                capi.lib().madicp_map_free(h)
            except TypeError:  # interpreter shutdown
                pass

    __del__ = free

    def insert(self, tree, T=None, scan=0):
        """The kept cloud of a DeviceTree (built with `Registrar.keep_cloud` on), posed by T (4x4 / 3x4, or None:
        untouched), its points tagged with `scan`.  Asynchronous."""
        X = None if T is None else pose12(T)
        check(capi.lib().madicp_map_insert(self._h, tree._h, as_d(X), int(scan)), "madicp_map_insert")

    def size(self):
        return check(capi.lib().madicp_map_size(self._h, None), "madicp_map_size")

    def dropped(self):
        d = C.c_int64(0)
        check(capi.lib().madicp_map_size(self._h, C.byref(d)), "madicp_map_size")
        return d.value

    def points(self, device=False):
        """(xyz (M, 3) float64, scan_record (M, 2) int64) as numpy arrays, or with device=True torch tensors on the
        registrar's device, ready on torch's current stream."""
        n = self.size()
        if not device:
            xyz, sr = np.empty((n, 3)), np.empty((n, 2), np.int64)
            check(capi.lib().madicp_map_points(self._h, as_d(xyz), sr.ctypes.data_as(C.POINTER(C.c_int64))),
                  "madicp_map_points")
            return xyz, sr
        import torch
        dev = torch.device("cuda", self._reg.device)
        xyz = torch.empty((n, 3), dtype=torch.float64, device=dev)
        sr = torch.empty((n, 2), dtype=torch.int64, device=dev)
        if n:
            check(capi.lib().madicp_map_points_dev(self._h, C.c_void_p(xyz.data_ptr()), C.c_void_p(sr.data_ptr()),
                                                   C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)),
                  "madicp_map_points_dev")
        return xyz, sr

    def clear(self):
        check(capi.lib().madicp_map_clear(self._h), "madicp_map_clear")

    def remove_far(self, origin, max_distance):
        """Every voxel whose centre lies farther than max_distance from origin (3 floats) goes, with its rows; later
        points that reach it start it afresh.  Asynchronous (madicp_map_remove_far)."""
        o = np.ascontiguousarray(np.asarray(origin, np.float64).reshape(3))
        check(capi.lib().madicp_map_remove_far(self._h, as_d(o), float(max_distance)), "madicp_map_remove_far")

    def carve(self, tree, T=None, reach=1.0):
        """Free-space carving: the rays from T's translation (None: the origin) to the points of the DeviceTree's kept
        cloud, posed by T as `insert` poses them, remove every live voxel they pass through in their first `reach` (in
        (0, 1]) of steps, with its rows, except the voxels that hold an endpoint.  Asynchronous (madicp_map_carve)."""
        X = None if T is None else pose12(T)
        check(capi.lib().madicp_map_carve(self._h, tree._h, as_d(X), float(reach)), "madicp_map_carve")

    def nearest(self, queries, max_distance, scan_below=None):
        """The nearest row within max_distance (finite, >= 0, <= 4 voxel sizes) of each query point, among the rows
        whose scan is < scan_below (None: every row): (row (N,) int64, -1 for none; d2 (N,) float64, the squared
        distance ((x - qx)^2 + (y - qy)^2) + (z - qz)^2 in float64 without FMA, +inf for none), ties to the smaller row.
        Host queries (N x 3) give numpy arrays (madicp_map_nearest, synchronises); device queries (a CUDA tensor or
        array, float32 or float64, read in place) give torch tensors on the registrar's device, ready on torch's current
        stream (madicp_map_nearest_dev)."""
        below = np.iinfo(np.int64).max if scan_below is None else int(scan_below)
        if hasattr(queries, "__cuda_array_interface__"):
            from .records import map_nearest_dev

            def run(q, n, stride, is_f32, r, sb, row, d2, stream):
                check(capi.lib().madicp_map_nearest_dev(self._h, C.c_void_p(q), n, stride, int(is_f32), r, sb,
                                                        C.c_void_p(row), C.c_void_p(d2), C.c_void_p(stream)),
                      "madicp_map_nearest_dev")
            return map_nearest_dev(run, self._reg.device, queries, max_distance, below)
        q = np.ascontiguousarray(np.asarray(queries, np.float64))
        if q.ndim != 2 or q.shape[1] != 3:
            raise ValueError("queries: an (N, 3) array")
        row, d2 = np.empty(q.shape[0], np.int64), np.empty(q.shape[0])
        check(capi.lib().madicp_map_nearest(self._h, as_d(q), q.shape[0], float(max_distance), below,
                                            row.ctypes.data_as(C.POINTER(C.c_int64)), as_d(d2)), "madicp_map_nearest")
        return row, d2

    def table(self):
        """(slots, occupied, live) of the hash table, counted from its keys (madicp_debug_map_table).  Synchronises."""
        out = [C.c_int64(0) for _ in range(3)]
        check(capi.lib().madicp_debug_map_table(self._h, *[C.byref(x) for x in out]), "madicp_debug_map_table")
        return tuple(x.value for x in out)


class Registrar:
    """One GPU's registration context (reference: class MADicp + Pipeline's keyframe deque)."""

    def __init__(self, device=0, max_keyframes=16, min_ball=0.2, rho_ker=0.1, b_ratio=0.02):
        h = C.c_void_p()
        check(capi.lib().madicp_create(C.byref(h), device, max_keyframes), "madicp_create")
        self._h = h
        self._staged_keepalive = []
        self.device = device
        self.max_keyframes = max_keyframes
        self.L = 0
        self.set_params(min_ball, rho_ker, b_ratio)

    def close(self):
        h = getattr(self, "_h", None)
        if h:
            self._h = None
            try:
                capi.lib().madicp_destroy(h)
            except TypeError:  # interpreter shutdown: module globals already torn down
                pass

    __del__ = close

    def set_params(self, min_ball, rho_ker, b_ratio):
        check(capi.lib().madicp_set_params(self._h, min_ball, rho_ker, b_ratio), "madicp_set_params")

    def keep_cloud(self, keep=True):
        """Trees built from now on keep their input cloud and its record indices (`DeviceTree.cloud`)."""
        check(capi.lib().madicp_set_keep_cloud(self._h, int(bool(keep))), "madicp_set_keep_cloud")

    def voxel_map(self, voxel_size, points_per_voxel=1, reserve_points=0):
        """A VoxelMap on this context (madicp_map_create); it takes trees built with `keep_cloud` on."""
        h = C.c_void_p()
        check(capi.lib().madicp_map_create(self._h, float(voxel_size), int(points_per_voxel), int(reserve_points),
                                           C.byref(h)), "madicp_map_create")
        return VoxelMap(h, self)

    def set_stream(self, cuda_stream_ptr):
        check(capi.lib().madicp_set_stream(self._h, C.c_void_p(cuda_stream_ptr or 0)))

    @property
    def stream(self):
        return capi.lib().madicp_get_stream(self._h)

    def put_keyframe(self, slot, tree, T=None):
        """tree: FlatTree (host-built) or DeviceTree.  T: pose applied ON THE DEVICE during the upload
        (MADtree::applyTransform); None for a tree that is already in the map frame."""
        X = as_d(pose12(T)) if T is not None else None
        if isinstance(tree, DeviceTree):
            check(capi.lib().madicp_put_keyframe_tree(self._h, slot, tree._h, X), "madicp_put_keyframe_tree")
        else:
            check(capi.lib().madicp_put_keyframe_transformed(self._h, slot, tree._h, X), "madicp_put_keyframe")

    def upload_tree(self, flat_tree):
        h = C.c_void_p()
        check(capi.lib().madtree_gpu_upload(self._h, flat_tree._h, C.byref(h)), "madtree_gpu_upload")
        return DeviceTree(h, self)

    def build_tree(self, points=None, b_max=0.2, b_min=0.1):
        """MAD-tree of a scan built ON THE DEVICE (points: N x 3 float64 host array, or None for the cloud
        madicp_ingest left on the device)."""
        h = C.c_void_p()
        if points is None:
            check(capi.lib().madtree_gpu_build_resident(self._h, b_max, b_min, C.byref(h)), "madtree_gpu_build_resident")
        else:
            pts = np.ascontiguousarray(points, dtype=np.float64)
            check(capi.lib().madtree_gpu_build(self._h, as_d(pts), pts.shape[0], b_max, b_min, C.byref(h)),
                  "madtree_gpu_build")
        return DeviceTree(h, self)

    def stage_cloud(self, cloud, reserve_points=0):
        """Early upload of a scan of the NEXT build_trees call (madicp_stage_cloud).  The array (float32 or float64,
        C-contiguous N x 3) is read in place: pass the same object to build_trees, unchanged."""
        a = np.asarray(cloud)
        if a.dtype not in (np.float32, np.float64) or not a.flags.c_contiguous or a.ndim != 2 or a.shape[1] != 3:
            raise ValueError("stage_cloud: a C-contiguous N x 3 float32 / float64 array")
        self._staged_keepalive.append(a)
        check(capi.lib().madicp_stage_cloud(self._h, C.c_void_p(a.ctypes.data), a.shape[0], int(a.dtype == np.float32),
                                            int(reserve_points)), "madicp_stage_cloud")

    def stage_discard(self):
        """Gives up the staged clouds; returns once nothing reads their host buffers (madicp_stage_discard)."""
        check(capi.lib().madicp_stage_discard(self._h), "madicp_stage_discard")

    def build_trees(self, clouds, b_max=0.2, b_min=0.1):
        """Several scans at once (all float32 or all float64): one forest build, a DeviceTree per scan."""
        f32 = all(np.asarray(c).dtype == np.float32 for c in clouds)
        arrs = [np.ascontiguousarray(c, dtype=np.float32 if f32 else np.float64) for c in clouds]
        k = len(arrs)
        ptrs = (C.c_void_p * k)(*[a.ctypes.data for a in arrs])
        ns = (C.c_int64 * k)(*[a.shape[0] for a in arrs])
        out = (C.c_void_p * k)()
        check(capi.lib().madtree_gpu_build_batch(self._h, ptrs, ns, int(f32), k, b_max, b_min, out), "madtree_gpu_build_batch")
        self._staged_keepalive.clear()
        return [DeviceTree(C.c_void_p(out[i]), self) for i in range(k)]

    def ingest(self, xyz, deskew=False, T_prev=None, T_now=None, sensor_hz=10.0, num_threads=1, want_points=False):
        """Raw scan -> device-resident float64 cloud (optionally deskewed, Pipeline::deskew)."""
        a = np.ascontiguousarray(xyz)
        if a.dtype != np.float32:
            a = np.ascontiguousarray(a, dtype=np.float64)
        n = a.shape[0]
        out = np.empty((n, 3)) if want_points else None
        Tp = as_d(pose12(T_prev)) if T_prev is not None else None
        Tn = as_d(pose12(T_now)) if T_now is not None else None
        check(capi.lib().madicp_ingest(self._h, a.ctypes.data_as(C.c_void_p), n, int(a.dtype == np.float32), int(deskew),
                                       Tp, Tn, sensor_hz, num_threads, as_d(out)), "madicp_ingest")
        return out

    # ---- raw sensor records (records.describe: strided x/y/z + the readers' range gate), read in place; with
    # apply_correction=True the kept points get KITTI's vertical-angle correction (records.vcorr)
    def ingest_records(self, records, min_range=0.0, max_range=math.inf, inclusive=True, drop_nan=False, deskew=False,
                       T_prev=None, T_now=None, sensor_hz=10.0, num_threads=1, want_points=False, apply_correction=False,
                       vertical_angle_offset=VERTICAL_ANGLE_OFFSET, time_field=None, time_scale=1.0, time_end=None):
        """Records -> device-resident float64 cloud of the kept points (madicp_ingest_points_t; a device array is read
        in place, madicp_ingest_points_dev_t).  time_field (records.time_layout): a deskew takes each point's chunk from
        its own stamp, time_scale seconds per unit, time_end the sweep's end (default: the
        largest kept stamp).  Returns the kept points (want_points) or their number."""
        d = describe(records, min_range, max_range, inclusive, drop_nan)
        v = vcorr(apply_correction, vertical_angle_offset)
        t = describe_times(records, time_field, time_scale, time_end)
        out = np.empty((d.n, 3)) if want_points else None
        kept = C.c_int64(0)
        Tp = as_d(pose12(T_prev)) if T_prev is not None else None
        Tn = as_d(pose12(T_now)) if T_now is not None else None
        t = C.byref(t) if t is not None else None
        if d.on_device:  # read in place on the device, after the producer's stream (records.describe)
            check(capi.lib().madicp_ingest_points_dev_t(self._h, C.byref(d), C.byref(v) if v else None, t, int(deskew), Tp,
                                                        Tn, sensor_hz, num_threads, d.stream, C.byref(kept), as_d(out)),
                  "madicp_ingest_points_dev_t")
        else:
            check(capi.lib().madicp_ingest_points_t(self._h, C.byref(d), C.byref(v) if v else None, t, int(deskew), Tp, Tn,
                                                    sensor_hz, num_threads, C.byref(kept), as_d(out)),
                  "madicp_ingest_points_t")
        return out[:kept.value].copy() if want_points else kept.value

    def stage_records(self, records, reserve_points=0, apply_correction=False, vertical_angle_offset=VERTICAL_ANGLE_OFFSET,
                      **gate):
        """Early upload of the records of a scan of the NEXT build_trees_records call (madicp_stage_points_ex); pass the
        same array, gate and correction there, unchanged."""
        d = describe(records, **gate)
        v = vcorr(apply_correction, vertical_angle_offset)
        self._staged_keepalive.append(records)
        check(capi.lib().madicp_stage_points_ex(self._h, C.byref(d), C.byref(v) if v else None, int(reserve_points)),
              "madicp_stage_points")

    def build_trees_records(self, records_list, b_max=0.2, b_min=0.1, apply_correction=False,
                            vertical_angle_offset=VERTICAL_ANGLE_OFFSET, **gate):
        """Several scans of records at once: one forest build, a DeviceTree per scan (madtree_gpu_build_batch_points_ex).
        apply_correction: one flag for all scans, or a sequence with one flag per scan."""
        k = len(records_list)
        ds = [describe(r, **gate) for r in records_list]
        descs = (capi.Points * k)(*ds)
        flags = list(apply_correction) if isinstance(apply_correction, (list, tuple)) else [apply_correction] * k
        if len(flags) != k:
            raise ValueError("build_trees_records: one apply_correction flag per scan")
        vcs = (capi.Vcorr * k)(*[vcorr(f, vertical_angle_offset) or capi.Vcorr() for f in flags])
        out = (C.c_void_p * k)()
        if any(d.on_device for d in ds):  # device records, read in place (one producer stream: the first scan's)
            if not all(d.on_device for d in ds):
                raise ValueError("build_trees_records: all scans on the device, or all on the host")
            check(capi.lib().madtree_gpu_build_batch_points_dev(self._h, descs, vcs, k, b_max, b_min, ds[0].stream, out),
                  "madtree_gpu_build_batch_points_dev")
        else:
            check(capi.lib().madtree_gpu_build_batch_points_ex(self._h, descs, vcs, k, b_max, b_min, out),
                  "madtree_gpu_build_batch_points")
        self._staged_keepalive.clear()
        return [DeviceTree(C.c_void_p(out[i]), self) for i in range(k)]

    def plan_records(self, records, min_range=0.0, max_range=math.inf, inclusive=True, drop_nan=False, num_threads=1,
                     apply_correction=False, vertical_angle_offset=VERTICAL_ANGLE_OFFSET, time_field=None, time_scale=1.0,
                     time_end=None):
        """Hands a future scan over for a deskewed look-ahead (madicp_plan_points_t): the records start going up at once
        and the pose-free half of the deskew runs on a host thread (at most num_threads at a time).  With a time_field
        (as in ingest_records) there is no host half: the gate, the correction and the compaction
        run on the device at once.  Returns a DeskewPlan for ingest_plan; the array is read in place and must stay
        unchanged until then."""
        d = describe(records, min_range, max_range, inclusive, drop_nan)
        v = vcorr(apply_correction, vertical_angle_offset)
        t = describe_times(records, time_field, time_scale, time_end)
        h = C.c_void_p()
        t = C.byref(t) if t is not None else None
        if d.on_device:
            check(capi.lib().madicp_plan_points_dev_t(self._h, C.byref(d), C.byref(v) if v else None, t, int(num_threads),
                                                      d.stream, C.byref(h)), "madicp_plan_points_dev_t")
        else:
            check(capi.lib().madicp_plan_points_t(self._h, C.byref(d), C.byref(v) if v else None, t, int(num_threads),
                                                  C.byref(h)), "madicp_plan_points_t")
        return DeskewPlan(h, self, records)

    def ingest_plan(self, plan, deskew=False, T_prev=None, T_now=None, sensor_hz=10.0, want_points=False):
        """Consumes a DeskewPlan (madicp_ingest_plan): the same device-resident cloud as ingest_records on its scan with
        the same deskew arguments.  Returns the kept points (want_points) or their number."""
        h = plan._take()
        n = plan._records.shape[0]
        out = np.empty((n, 3)) if want_points else None
        kept = C.c_int64(0)
        Tp = as_d(pose12(T_prev)) if T_prev is not None else None
        Tn = as_d(pose12(T_now)) if T_now is not None else None
        try:
            check(capi.lib().madicp_ingest_plan(self._h, h, int(deskew), Tp, Tn, sensor_hz, C.byref(kept), as_d(out)),
                  "madicp_ingest_plan")
        finally:
            plan._records = None
        return out[:kept.value].copy() if want_points else kept.value

    def set_moving_tree(self, tree):
        check(capi.lib().madicp_set_moving_tree(self._h, tree._h), "madicp_set_moving_tree")
        self.L = tree.num_leaves

    def get_moving(self):
        out = np.empty((self.L, 3))
        check(capi.lib().madicp_get_moving(self._h, as_d(out), self.L), "madicp_get_moving")
        return out

    def synchronize(self):
        check(capi.lib().madicp_synchronize(self._h))

    def calibrate(self, X0):
        return check(capi.lib().madicp_calibrate(self._h, as_d(pose12(X0))), "madicp_calibrate")

    def put_keyframe_records(self, slot, recs, n_leaves):
        recs = np.ascontiguousarray(recs, dtype=capi.REC_DTYPE)
        check(capi.lib().madicp_put_keyframe_records(self._h, slot, recs.ctypes.data_as(C.c_void_p), recs.shape[0],
                                                     n_leaves), "madicp_put_keyframe_records")

    def drop_keyframe(self, slot):
        check(capi.lib().madicp_drop_keyframe(self._h, slot))

    @property
    def num_keyframes(self):
        return capi.lib().madicp_num_keyframes(self._h)

    def active_slots(self):
        out = np.empty(self.max_keyframes, np.int32)
        k = capi.lib().madicp_active_slots(self._h, as_i(out), self.max_keyframes)
        return out[:k].tolist()

    @property
    def model_nodes(self):
        return capi.lib().madicp_model_nodes(self._h)

    @property
    def kernel_launches(self):
        return capi.lib().madicp_kernel_launches(self._h)

    def set_moving(self, means):
        """means: L x 3 float64 host array (numpy, or the memory of a pinned torch tensor)."""
        if hasattr(means, "data_ptr"):  # torch tensor (pinned host memory)
            assert means.dtype.is_floating_point and means.element_size() == 8 and means.is_contiguous()
            L, ptr = means.shape[0], means.data_ptr()
            self._keep = means
        else:
            means = np.ascontiguousarray(means, dtype=np.float64)
            L, ptr = means.shape[0], means.ctypes.data
            self._keep = means
        check(capi.lib().madicp_set_moving(self._h, C.c_void_p(ptr), L), "madicp_set_moving")
        self.L = L

    def search(self, X):
        X = pose12(X)
        out = np.empty((self.num_keyframes, self.L), np.int32)
        check(capi.lib().madicp_search(self._h, as_d(X), as_i(out)), "madicp_search")
        return out

    def linearize(self, X):
        X = pose12(X)
        H, b = np.empty((6, 6)), np.empty(6)
        m = np.empty(self.L, np.uint8)
        check(capi.lib().madicp_linearize(self._h, as_d(X), as_d(H), as_d(b), as_b(m)), "madicp_linearize")
        return H, b, m

    def solve_update(self, H, b, X):
        X = pose12(X).copy()
        H = np.ascontiguousarray(H, dtype=np.float64)
        b = np.ascontiguousarray(b, dtype=np.float64)
        check(capi.lib().madicp_solve_update(self._h, as_d(H), as_d(b), as_d(X)), "madicp_solve_update")
        return X

    def inv_det6(self, H):
        """The keyframe weight det(H^-1) that register_fetch() returns, for any 6x6 H (madicp_debug_inv_det6)."""
        H = np.ascontiguousarray(H, dtype=np.float64)
        w = C.c_double(0)
        check(capi.lib().madicp_debug_inv_det6(self._h, as_d(H), C.byref(w)), "madicp_debug_inv_det6")
        return w.value

    def register(self, X0, iters=15, want_matched=True):
        """The whole ICP loop on the device.  Returns dict(X 3x4, H 6x6, b 6, matched L, n_matched)."""
        X = pose12(X0).copy()
        H, b = np.empty((6, 6)), np.empty(6)
        m = np.empty(self.L, np.uint8) if want_matched else None
        n = C.c_int(0)
        check(capi.lib().madicp_register(self._h, iters, as_d(X), as_d(H), as_d(b), as_b(m), C.byref(n)),
              "madicp_register")
        return dict(X=X, H=H, b=b, matched=m, n_matched=n.value)

    def register_async(self, X0, iters=15, partial=False):
        """partial=True: a loop the realtime budget cut short -- the matched flags are the union over all rounds."""
        X = pose12(X0)
        fn = capi.lib().madicp_register_partial_async if partial else capi.lib().madicp_register_async
        check(fn(self._h, iters, as_d(X)), "madicp_register_async")

    def register_fetch(self, want_matched=False):
        X, H, b = np.empty((3, 4)), np.empty((6, 6)), np.empty(6)
        m = np.empty(self.L, np.uint8) if want_matched else None
        n, w = C.c_int(0), C.c_double(0)
        check(capi.lib().madicp_register_fetch_weight(self._h, as_d(X), as_d(H), as_d(b), as_b(m), C.byref(n), C.byref(w)),
              "madicp_register_fetch")
        return dict(X=X, H=H, b=b, matched=m, n_matched=n.value, weight=w.value)

    def register_trace(self):
        buf = np.empty((65, 3, 4))
        rows = check(capi.lib().madicp_register_trace(self._h, as_d(buf), 65), "madicp_register_trace")
        return buf[:rows].copy()

    def register_walked(self):
        """Per round of the last registration: pairs actually walked (the rest kept their leaf: path memo)."""
        buf = np.zeros(64, np.int32)
        rows = check(capi.lib().madicp_register_walked(self._h, as_i(buf), 64), "madicp_register_walked")
        return buf[:rows].copy()

    def register_walk_records(self):
        """Per round of the last registration: quad records loaded by the walks (fewer when a walk resumes below the root)."""
        buf = np.zeros(64, np.int64)
        rows = check(capi.lib().madicp_register_walk_records(self._h, buf.ctypes.data_as(C.POINTER(C.c_int64)), 64),
                     "madicp_register_walk_records")
        return buf[:rows].copy()

    def search_cloud(self, slot, queries, want=("ordinals", "points", "normals", "dists")):
        q = np.ascontiguousarray(queries, dtype=np.float64).reshape(-1, 3)
        n = q.shape[0]
        o = np.empty(n, np.int32) if "ordinals" in want else None
        p = np.empty((n, 3)) if "points" in want else None
        nr = np.empty((n, 3)) if "normals" in want else None
        d = np.empty(n) if "dists" in want else None
        check(capi.lib().madicp_search_cloud(self._h, slot, as_d(q), n, as_i(o), as_d(p), as_d(nr), as_d(d)),
              "madicp_search_cloud")
        return dict(ordinals=o, points=p, normals=nr, dists=d)

    # ---- tuning / debug
    def debug_timing(self, enable=True, fetch=True):
        buf = np.zeros((64, 8), np.int64)
        rows = check(capi.lib().madicp_debug_timing(self._h, int(enable), buf.ctypes.data_as(C.POINTER(C.c_int64))
                                                    if fetch else None, 64))
        return buf[:rows]

    def debug_cta_cycles(self, rounds):
        buf = np.zeros(rounds * 2048, np.int64)  # room for grids of up to 2048 CTAs
        grid = check(capi.lib().madicp_debug_cta_cycles(self._h, buf.ctypes.data_as(C.POINTER(C.c_int64)), buf.size))
        return buf[:rounds * grid].reshape(rounds, grid)

    def debug_cta_stamps(self, plane, rounds):
        buf = np.zeros(rounds * 2048, np.int64)
        grid = check(capi.lib().madicp_debug_cta_stamps(self._h, plane, buf.ctypes.data_as(C.POINTER(C.c_int64)), buf.size))
        return buf[:rounds * grid].reshape(rounds, grid)

    def set_memo(self, mode=True):
        """Path memo mode: 0 / False walks every pair from the root, 1 keeps proved leaves, 2 / True (the default)
        also resumes the other walks from their checkpoint."""
        if isinstance(mode, bool):
            mode = 2 if mode else 0
        check(capi.lib().madicp_debug_set_memo(self._h, int(mode)), "madicp_debug_set_memo")

    def set_gn_grid(self, threads_per_cta=1024, ctas_per_sm=1):
        return check(capi.lib().madicp_set_gn_grid(self._h, threads_per_cta, ctas_per_sm))

    # ---- multi-GPU -------------------------------------------------------------------------
    def comm_export(self):
        buf = (C.c_char * 64)()
        check(capi.lib().madicp_comm_export(self._h, buf), "madicp_comm_export")
        return bytes(buf)

    def comm_connect(self, rank, world, handles):
        blob = b"".join(handles)
        assert len(blob) == 64 * world
        check(capi.lib().madicp_comm_connect(self._h, rank, world, blob), "madicp_comm_connect")

    @property
    def world(self):
        return capi.lib().madicp_comm_world(self._h)


__all__ = ["FlatTree", "DeviceTree", "Registrar", "MadIcpError", "leaf_means"]
