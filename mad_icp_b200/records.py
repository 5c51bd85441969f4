"""Raw sensor records -> madicp_points_t (include/madicp_b200.h): hand a scan to the device as the sensor delivered it.

The dataset readers of the reference filter every scan with numpy before it reaches `Pipeline.compute`:
  KITTI        apps/utils/kitti_reader.py:82-88   np.fromfile(float32).reshape(-1, 4)[:, :3], then
                                                  min_range <= |p| <= max_range
  ROS1/ROS2/MCAP apps/utils/point_cloud2.py:77-87 x/y/z of the PointCloud2 records, NaN rows dropped, then
                                                  min_range < |p| < max_range
`Pipeline.computeRecords` / `prefetchRecords` and the `Registrar.*_records` methods take the unfiltered array instead
(read in place, never copied on the host) and apply the same filter on the way in, with numpy's arithmetic: the
kept points and their order are the reader's, bit for bit.  A Python float bound is compared in the field type, as
numpy compares it.

KITTI's reader can also rotate every kept point by a small vertical angle (`apply_correction`,
apps/utils/kitti_reader.py:72-79, 90-91, a scipy rotation about p x e_z).  `apply_correction=True` does the same on
the device, bit for bit with scipy 1.18 (`correct_vertical_angle` is the host restatement).
"""
import ctypes as C
import math

import numpy as np

from ._capi import Points, Vcorr

RANGE_NONE, RANGE_INCLUSIVE, RANGE_STRICT = 0, 1, 2
# KittiReader.vertical_angle_offset: the reader's own expression, so the default is its value bit for bit
VERTICAL_ANGLE_OFFSET = float(np.radians(0.205))

_POINTFIELD_TYPES = {7: np.dtype("<f4"), 8: np.dtype("<f8")}  # sensor_msgs/PointField FLOAT32, FLOAT64


def pointcloud2_dtype(msg):
    """numpy dtype of the records of a sensor_msgs/PointCloud2 message with fields x, y, z (duck-typed: any object with
    `fields` (name, offset, datatype[, count]), `point_step`, `width`, `height`, `row_step`, `is_bigendian`).  Use it as
    `np.frombuffer(msg.data, pointcloud2_dtype(msg), count=msg.width * msg.height)`."""
    if getattr(msg, "is_bigendian", False):
        raise ValueError("pointcloud2_dtype: big-endian PointCloud2 is not supported")
    step = int(msg.point_step)
    if int(msg.row_step) != int(msg.width) * step:
        raise ValueError(f"pointcloud2_dtype: row_step {msg.row_step} != width {msg.width} * point_step {step} (padded rows)")
    found = {}
    for f in msg.fields:
        if f.name in ("x", "y", "z"):
            if int(getattr(f, "count", 1)) != 1:
                raise ValueError(f"pointcloud2_dtype: field {f.name} has count {f.count}")
            if int(f.datatype) not in _POINTFIELD_TYPES:
                raise ValueError(f"pointcloud2_dtype: field {f.name} has datatype {f.datatype} (float32 = 7 or float64 = 8 only)")
            found[f.name] = (_POINTFIELD_TYPES[int(f.datatype)], int(f.offset))
    if sorted(found) != ["x", "y", "z"]:
        raise ValueError("pointcloud2_dtype: the message has no x, y and z fields")
    if len({found[k][0] for k in found}) != 1:
        raise ValueError("pointcloud2_dtype: x, y and z do not share one float type")
    return np.dtype({"names": ["x", "y", "z"], "formats": [found[k][0] for k in "xyz"],
                     "offsets": [found[k][1] for k in "xyz"], "itemsize": step})


def _float_type(dt):
    if dt.kind != "f" or dt.itemsize not in (4, 8) or dt.byteorder == ">":
        return None
    return dt.itemsize


def describe(records, min_range=0.0, max_range=math.inf, inclusive=True, drop_nan=False):
    """madicp_points_t of `records` (read in place):
      - a 2-D float32 / float64 array with at least 3 columns (x, y, z = columns 0, 1, 2) and any row stride that holds
        a row's x, y, z (row-major layouts and views of them; not column-major), e.g.
        np.fromfile(f, np.float32).reshape(-1, 4);
      - a 1-D structured array whose x, y, z fields share one float type, e.g. np.frombuffer(msg.data, dtype).
    inclusive=True gates min_range <= r <= max_range (KITTI), False min_range < r < max_range (PointCloud2);
    drop_nan drops records with a NaN coordinate.  Returns the ctypes structure; the caller keeps `records` alive."""
    a = records
    if not isinstance(a, np.ndarray):
        raise TypeError("records: a numpy array (2-D float, or 1-D structured with x, y, z fields)")
    if a.dtype.names:
        if a.ndim != 1 or not all(k in a.dtype.names for k in "xyz"):
            raise ValueError("records: a 1-D structured array needs fields x, y and z")
        types = {a.dtype.fields[k][0] for k in "xyz"}
        e = _float_type(next(iter(types)))
        if len(types) != 1 or e is None:
            raise ValueError("records: x, y and z must share one little-endian float32 or float64 type")
        offsets = [int(a.dtype.fields[k][1]) for k in "xyz"]
        stride = int(a.strides[0]) if a.shape[0] > 1 else a.dtype.itemsize
    else:
        e = _float_type(a.dtype)
        if a.ndim != 2 or a.shape[1] < 3 or e is None:
            raise ValueError("records: a 2-D little-endian float32 / float64 array with at least 3 columns")
        s0, s1 = int(a.strides[0]), int(a.strides[1])
        if s1 <= 0:
            raise ValueError("records: columns must have a positive stride")
        if a.shape[0] > 1 and s0 <= 0:
            raise ValueError("records: rows must have a positive stride")
        if a.shape[0] > 1 and s0 < 2 * s1 + e:
            raise ValueError(f"records: x, y, z of a row must lie within the row stride ({s0} bytes; columns {s1} bytes "
                             "apart): rows of a column-major (Fortran-order) or transposed array interleave -- pass "
                             "np.ascontiguousarray(records)")
        offsets = [0, s1, 2 * s1]
        stride = s0 if a.shape[0] > 1 else max(s0, 2 * s1 + e)
    if stride <= 0:
        raise ValueError("records: rows must have a positive stride")
    d = Points()
    d.data = a.ctypes.data
    d.n = a.shape[0]
    d.stride = stride
    d.offset[:] = offsets
    d.is_f32 = int(e == 4)
    d.min_range = float(min_range)
    d.max_range = float(max_range)
    d.range_mode = RANGE_INCLUSIVE if inclusive else RANGE_STRICT
    d.drop_nan = int(bool(drop_nan))
    return d


def layout(records, min_range=0.0, max_range=math.inf, inclusive=True, drop_nan=False):
    """describe() as a plain tuple (data, n, stride, off_x, off_y, off_z, is_f32, min_range, max_range, range_mode,
    drop_nan): what the pybind Pipeline reads."""
    d = describe(records, min_range, max_range, inclusive, drop_nan)
    return (int(d.data or 0), d.n, d.stride, d.offset[0], d.offset[1], d.offset[2], d.is_f32, d.min_range, d.max_range,
            d.range_mode, d.drop_nan)


def vcorr(apply_correction=False, vertical_angle_offset=VERTICAL_ANGLE_OFFSET):
    """madicp_vcorr_t of the reader's `apply_correction` / `vertical_angle_offset`, or None without a correction."""
    if not apply_correction:
        return None
    v = Vcorr()
    v.angle = float(vertical_angle_offset)
    v.enabled = 1
    return v


def range_mask(records, **gate):
    """The gate on the host (madicp_debug_range_mask): uint8 keep flag per record."""
    from . import _capi
    d = describe(records, **gate)
    keep = np.empty(max(int(d.n), 1), np.uint8)
    _capi.check(_capi.lib().madicp_debug_range_mask(C.byref(d), keep.ctypes.data_as(_capi.bp)), "madicp_debug_range_mask")
    return keep[:d.n]


def correct_vertical_angle(records, vertical_angle_offset=VERTICAL_ANGLE_OFFSET, **gate):
    """The kept points of `records` (describe's gate keywords), corrected like KittiReader.apply_rotation_correction,
    on the host with the restatement the device applies (madicp_debug_correct_points): an M x 3 float64 array."""
    from . import _capi
    d = describe(records, **gate)
    v = vcorr(True, vertical_angle_offset)
    out = np.empty((max(int(d.n), 1), 3))
    kept = _capi.check(_capi.lib().madicp_debug_correct_points(C.byref(d), C.byref(v), _capi.as_d(out)),
                       "madicp_debug_correct_points")
    return out[:kept]


__all__ = ["pointcloud2_dtype", "describe", "layout", "range_mask", "vcorr", "correct_vertical_angle",
           "VERTICAL_ANGLE_OFFSET", "RANGE_NONE", "RANGE_INCLUSIVE", "RANGE_STRICT"]
