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

A scan that already lives on the GPU -- any object exporting `__cuda_array_interface__` (a torch CUDA tensor, a CuPy
array) -- is described the same way and read in place on the device: no copy to the host and back, no synchronisation
of its producer.  Its descriptor carries `on_device` and the producer `stream` (see `describe`).
"""
import ctypes as C
import math

import numpy as np

from ._capi import Points, Times, Vcorr

RANGE_NONE, RANGE_INCLUSIVE, RANGE_STRICT = 0, 1, 2
# KittiReader.vertical_angle_offset: the reader's own expression, so the default is its value bit for bit
VERTICAL_ANGLE_OFFSET = float(np.radians(0.205))

_POINTFIELD_TYPES = {7: np.dtype("<f4"), 8: np.dtype("<f8")}  # sensor_msgs/PointField FLOAT32, FLOAT64
_POINTFIELD_TIME_TYPES = {6: np.dtype("<u4"), 7: np.dtype("<f4"), 8: np.dtype("<f8")}  # UINT32, FLOAT32, FLOAT64
TIME_NONE, TIME_U32, TIME_F32, TIME_F64 = 0, 1, 2, 3  # madicp_times_t.type
_TIME_TYPES = {np.dtype("<u4"): TIME_U32, np.dtype("<f4"): TIME_F32, np.dtype("<f8"): TIME_F64}


def pointcloud2_dtype(msg, time_field=None):
    """numpy dtype of the records of a sensor_msgs/PointCloud2 message with fields x, y, z (duck-typed: any object with
    `fields` (name, offset, datatype[, count]), `point_step`, `width`, `height`, `row_step`, `is_bigendian`).  Use it as
    `np.frombuffer(msg.data, pointcloud2_dtype(msg), count=msg.width * msg.height)`.  time_field (e.g. "t" of an Ouster,
    "time" of a Velodyne, "timestamp" of a Hesai): that field is kept too, for the time-stamp deskew; it must be UINT32
    (6), FLOAT32 (7) or FLOAT64 (8)."""
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
    names, formats, offsets = ["x", "y", "z"], [found[k][0] for k in "xyz"], [found[k][1] for k in "xyz"]
    if time_field is not None:
        f = next((f for f in msg.fields if f.name == time_field), None)
        if f is None or time_field in ("x", "y", "z"):
            raise ValueError(f"pointcloud2_dtype: the message has no time field {time_field!r}")
        if int(getattr(f, "count", 1)) != 1:
            raise ValueError(f"pointcloud2_dtype: field {f.name} has count {f.count}")
        if int(f.datatype) not in _POINTFIELD_TIME_TYPES:
            raise ValueError(f"pointcloud2_dtype: time field {f.name} has datatype {f.datatype} "
                             "(UINT32 = 6, FLOAT32 = 7 or FLOAT64 = 8 only)")
        names.append(time_field)
        formats.append(_POINTFIELD_TIME_TYPES[int(f.datatype)])
        offsets.append(int(f.offset))
    return np.dtype({"names": names, "formats": formats, "offsets": offsets, "itemsize": step})


def _float_type(dt):
    if dt.kind != "f" or dt.itemsize not in (4, 8) or dt.byteorder == ">":
        return None
    return dt.itemsize


def _rows(n, s0, s1, e):
    """byte stride and x/y/z offsets of the rows of a 2-D array of n rows whose columns lie s1 bytes apart"""
    if s1 <= 0:
        raise ValueError("records: columns must have a positive stride")
    if n > 1 and s0 <= 0:
        raise ValueError("records: rows must have a positive stride")
    if n > 1 and s0 < 2 * s1 + e:
        raise ValueError(f"records: x, y, z of a row must lie within the row stride ({s0} bytes; columns {s1} bytes "
                         "apart): rows of a column-major (Fortran-order) or transposed array interleave -- pass "
                         "np.ascontiguousarray(records) (a contiguous copy, e.g. tensor.contiguous(), on the device)")
    return (s0 if n > 1 else max(s0, 2 * s1 + e)), [0, s1, 2 * s1]


def _cuda_layout(cai):
    """(pointer, rows, row stride, offsets, field size) of a __cuda_array_interface__ (v2 or v3)"""
    shape = tuple(int(k) for k in cai["shape"])
    e = {"<f4": 4, "<f8": 8}.get(cai["typestr"])
    if len(shape) != 2 or shape[1] < 3 or e is None:
        raise ValueError("records: a 2-D little-endian float32 / float64 device array with at least 3 columns")
    if cai.get("mask") is not None:
        raise ValueError("records: masked device arrays are not supported")
    strides = cai.get("strides")
    s0, s1 = (shape[1] * e, e) if strides is None else (int(strides[0]), int(strides[1]))
    stride, offsets = _rows(shape[0], s0, s1, e)
    return int(cai["data"][0]), shape[0], stride, offsets, e


def _stream_handle(stream):
    """a cudaStream_t as an int: an int handle, or an object with .cuda_stream (torch.cuda.Stream, cupy streams)"""
    return int(getattr(stream, "cuda_stream", stream))


def _producer_stream(records, cai, stream):
    """The stream the device records are ready on: an explicit `stream`, else the interface's v3 `stream` entry, else
    for a torch tensor torch's current stream on its device (torch exports v2, without a stream), else 0 (the legacy
    default stream)."""
    if stream is not None:
        return _stream_handle(stream)
    if int(cai.get("version", 0)) >= 3 and cai.get("stream") is not None:
        return int(cai["stream"])  # (1: legacy default, 2: per-thread default, as the interface and the CUDA runtime number them)
    if type(records).__module__.split(".")[0] == "torch":
        import torch
        if isinstance(records, torch.Tensor):
            return torch.cuda.current_stream(records.device).cuda_stream
    return 0


def describe(records, min_range=0.0, max_range=math.inf, inclusive=True, drop_nan=False, stream=None):
    """madicp_points_t of `records` (read in place):
      - a 2-D float32 / float64 array with at least 3 columns (x, y, z = columns 0, 1, 2) and any row stride that holds
        a row's x, y, z (row-major layouts and views of them; not column-major), e.g.
        np.fromfile(f, np.float32).reshape(-1, 4);
      - a 1-D structured array whose x, y, z fields share one float type, e.g. np.frombuffer(msg.data, dtype);
      - a 2-D device array exporting __cuda_array_interface__ (torch CUDA tensor, CuPy array), under the same rules as
        the 2-D numpy array: the descriptor's `on_device` is True and its `stream` is the stream the records are ready
        on -- `stream=` (an int handle or an object with .cuda_stream), else the interface's v3 stream, else for a torch
        tensor torch's current stream on its device, else 0 (the legacy default stream).
    inclusive=True gates min_range <= r <= max_range (KITTI), False min_range < r < max_range (PointCloud2);
    drop_nan drops records with a NaN coordinate.  Returns the ctypes structure; the caller keeps `records` alive."""
    a = records
    cai = None if isinstance(a, np.ndarray) else getattr(a, "__cuda_array_interface__", None)
    if cai is not None:
        ptr, n, stride, offsets, e = _cuda_layout(cai)
    elif not isinstance(a, np.ndarray):
        raise TypeError("records: a numpy array (2-D float, or 1-D structured with x, y, z fields) or a device array "
                        "exporting __cuda_array_interface__")
    elif a.dtype.names:
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
        stride, offsets = _rows(a.shape[0], int(a.strides[0]), int(a.strides[1]), e)
    if stride <= 0:
        raise ValueError("records: rows must have a positive stride")
    d = Points()
    if cai is not None:
        d.data, d.n = ptr, n
    else:
        d.data, d.n = a.ctypes.data, a.shape[0]
    d.stride = stride
    d.offset[:] = offsets
    d.is_f32 = int(e == 4)
    d.min_range = float(min_range)
    d.max_range = float(max_range)
    d.range_mode = RANGE_INCLUSIVE if inclusive else RANGE_STRICT
    d.drop_nan = int(bool(drop_nan))
    d.on_device = cai is not None
    d.stream = _producer_stream(records, cai, stream) if cai is not None else None
    return d


def layout(records, min_range=0.0, max_range=math.inf, inclusive=True, drop_nan=False, stream=None):
    """describe() as a plain tuple (data, n, stride, off_x, off_y, off_z, is_f32, min_range, max_range, range_mode,
    drop_nan, on_device, stream): what the pybind Pipeline reads (stream: 0 for host records)."""
    d = describe(records, min_range, max_range, inclusive, drop_nan, stream)
    return (int(d.data or 0), d.n, d.stride, d.offset[0], d.offset[1], d.offset[2], d.is_f32, d.min_range, d.max_range,
            d.range_mode, d.drop_nan, d.on_device, d.stream or 0)


def time_layout(records, field, scale=1.0, t_end=None):
    """(offset, type, scale, t_end, has_t_end) of the time field of `records` (as describe() reads them): `field` is a
    field name of a structured array, or a column index of a 2-D array or device array.  uint32, float32 and float64
    little-endian fields are accepted."""
    a = records
    cai = None if isinstance(a, np.ndarray) else getattr(a, "__cuda_array_interface__", None)
    if isinstance(field, str):
        if cai is not None or not isinstance(a, np.ndarray) or not a.dtype.names or field not in a.dtype.names:
            raise ValueError(f"time_field: the records have no field {field!r}")
        dt, off = a.dtype.fields[field][0], int(a.dtype.fields[field][1])
    elif isinstance(field, (int, np.integer)) and not isinstance(field, bool):
        col = int(field)
        if cai is not None:
            shape, e = tuple(int(k) for k in cai["shape"]), {"<f4": 4, "<f8": 8}.get(cai["typestr"])
            strides = cai.get("strides")
            s1 = e if strides is None else int(strides[1])
            dt = np.dtype(cai["typestr"])
        elif isinstance(a, np.ndarray) and a.ndim == 2 and not a.dtype.names:
            shape, s1, dt = a.shape, int(a.strides[1]), a.dtype
        else:
            raise ValueError("time_field: a column index needs a 2-D array")
        if not 3 <= col < shape[1]:
            raise ValueError(f"time_field: column {col} is not a column after x, y, z")
        off = col * s1
    else:
        raise TypeError("time_field: a field name or a column index")
    kind = None if dt.byteorder == ">" else _TIME_TYPES.get(dt)
    if kind is None:
        raise ValueError(f"time_field: {dt} is not a little-endian uint32, float32 or float64 field")
    return off, kind, float(scale), 0.0 if t_end is None else float(t_end), int(t_end is not None)


def describe_times(records, field, scale=1.0, t_end=None):
    """madicp_times_t of the time field of `records` (time_layout), or None when `field` is None."""
    if field is None:
        return None
    t = Times()
    t.offset, t.type, t.scale, t.t_end, t.has_t_end = time_layout(records, field, scale, t_end)
    return t


def time_chunks(records, field, scale, sensor_hz, t_end=None, apply_correction=False,
                vertical_angle_offset=VERTICAL_ANGLE_OFFSET, **gate):
    """The chunk of every kept record of `records` under the time-stamp deskew, on the host (madicp_debug_time_chunks):
    a uint16 array in record order."""
    from . import _capi
    d = _host(describe(records, **gate))
    v = vcorr(apply_correction, vertical_angle_offset)
    t = describe_times(records, field, scale, t_end)
    out = np.empty(max(int(d.n), 1), np.uint16)
    kept = C.c_int64(0)
    _capi.check(_capi.lib().madicp_debug_time_chunks(C.byref(d), C.byref(v) if v else None, C.byref(t), float(sensor_hz),
                                                     out.ctypes.data_as(C.POINTER(C.c_uint16)), C.byref(kept)),
                "madicp_debug_time_chunks")
    return out[:kept.value].copy()


def chunk_poses(T_prev, T_now, sensor_hz, n_chunks=1024):
    """The deskew's chunk poses (madicp_debug_chunk_poses): n_chunks x 3 x 4 float64."""
    from . import _capi
    out = np.empty((n_chunks, 12))
    _capi.check(_capi.lib().madicp_debug_chunk_poses(_capi.as_d(_capi.pose12(T_prev)), _capi.as_d(_capi.pose12(T_now)),
                                                     float(sensor_hz), int(n_chunks), _capi.as_d(out)),
                "madicp_debug_chunk_poses")
    return out.reshape(n_chunks, 3, 4)


def to_host(records):
    """A device array copied to the host once, as a numpy array (for host-built trees, MADICP_GPU_BUILD=0)."""
    if hasattr(records, "cpu"):  # torch
        return records.detach().cpu().numpy()
    if hasattr(records, "get"):  # CuPy
        return records.get()
    raise TypeError("records: cannot copy this device array to the host (a torch tensor or a CuPy array is needed)")


def search_cloud_arrays_dev(search_dev, queries):
    """MADtree.searchCloudArrays of device queries: (points N x 3, normals N x 3, dists N) as float64 torch tensors on the
    queries' device, written by the search kernel in place and ready on the caller's current stream (no host sync).
    search_dev: MADtree._searchCloudDev."""
    import torch
    d = describe(queries)
    e = 4 if d.is_f32 else 8
    if list(d.offset) != [0, e, 2 * e]:
        raise ValueError("queries: x, y, z must be adjacent columns -- pass a contiguous copy")
    dev = getattr(queries, "device", None)
    dev = torch.device("cuda", getattr(dev, "index", getattr(dev, "id", None)) or 0) if dev is not None else torch.device("cuda")
    n = int(d.n)
    P = torch.empty((n, 3), dtype=torch.float64, device=dev)
    N = torch.empty((n, 3), dtype=torch.float64, device=dev)
    D = torch.empty(n, dtype=torch.float64, device=dev)
    search_dev(int(d.data), n, int(d.stride), bool(d.is_f32), P.data_ptr(), N.data_ptr(), D.data_ptr(),
               torch.cuda.current_stream(dev).cuda_stream)
    return P, N, D


def map_nearest_dev(nearest_dev, device, queries, max_distance, scan_below):
    """VoxelMap.nearest / Pipeline.mapNearest of device queries (2-D float32 / float64 with x, y, z in adjacent columns,
    any row stride describe() accepts): (row (N,) int64, d2 (N,) float64) as torch tensors on the map's CUDA device,
    written by the query kernel in place and ready on torch's current stream there (no host sync).
    nearest_dev(q, n, stride, is_f32, max_distance, scan_below, row, d2, stream) runs madicp_map_nearest_dev."""
    import torch
    d = describe(queries)
    e = 4 if d.is_f32 else 8
    if list(d.offset) != [0, e, 2 * e]:
        raise ValueError("queries: x, y, z must be adjacent columns -- pass a contiguous copy")
    dev = torch.device("cuda", device)
    n = int(d.n)
    row = torch.empty(n, dtype=torch.int64, device=dev)
    d2 = torch.empty(n, dtype=torch.float64, device=dev)
    nearest_dev(int(d.data or 0), n, int(d.stride), bool(d.is_f32), float(max_distance), int(scan_below), row.data_ptr(),
                d2.data_ptr(), torch.cuda.current_stream(dev).cuda_stream)
    return row, d2


def leaves_array_dev(pipeline, model):
    """Pipeline.currentLeavesArray / modelLeavesArray(device=True): the leaf means as an (N, 3) float64 torch tensor on the
    pipeline's device, written by the gather kernel in place and ready on torch's current stream (no host sync).  With
    host-built trees (MADICP_GPU_BUILD=0) the host array is copied up once."""
    import torch
    dev = torch.device("cuda", pipeline._device())
    if not pipeline.gpuBuild():
        return torch.from_numpy(pipeline.modelLeavesArray() if model else pipeline.currentLeavesArray()).to(dev)
    n = pipeline._numLeaves(model)
    out = torch.empty((n, 3), dtype=torch.float64, device=dev)
    if n:
        pipeline._leafMeansDev(model, out.data_ptr(), torch.cuda.current_stream(dev).cuda_stream)
    return out


def cloud_array_dev(pipeline, indices, map_frame):
    """Pipeline.currentCloudArray / currentCloudIndices(device=True): the current scan's kept cloud as an (N, 3) float64
    torch tensor (posed by currentPose() when map_frame), or its record indices (indices=True) as an (N,) int64 tensor, on
    the pipeline's device, written by the output kernel in place and ready on torch's current stream (no host sync).
    With host-built trees (MADICP_GPU_BUILD=0) the host array is copied up once."""
    import torch
    dev = torch.device("cuda", pipeline._device())
    if not pipeline.gpuBuild():
        host = (pipeline.currentCloudIndices() if indices
                else pipeline.currentCloudArray(frame="map" if map_frame else "sensor"))
        return torch.from_numpy(host).to(dev)
    n = pipeline._numCloudPoints()
    out = torch.empty((n,) if indices else (n, 3), dtype=torch.int64 if indices else torch.float64, device=dev)
    if n:
        stream = torch.cuda.current_stream(dev).cuda_stream
        if indices:
            pipeline._cloudDev(False, 0, out.data_ptr(), stream)
        else:
            pipeline._cloudDev(map_frame, out.data_ptr(), 0, stream)
    return out


def map_array_dev(pipeline, indices):
    """Pipeline.mapArray / mapIndices(device=True): the voxel map's points as an (M, 3) float64 torch tensor, or its
    (scan, record) pairs (indices=True) as an (M, 2) int64 tensor, on the pipeline's device, copied in place and ready on
    torch's current stream.  Learning M waits once for the pipeline's stream (mapSize); the points never reach the
    host."""
    import torch
    dev = torch.device("cuda", pipeline._device())
    n = pipeline.mapSize()
    out = torch.empty((n, 2) if indices else (n, 3), dtype=torch.int64 if indices else torch.float64, device=dev)
    if n:
        stream = torch.cuda.current_stream(dev).cuda_stream
        if indices:
            pipeline._mapDev(0, out.data_ptr(), stream)
        else:
            pipeline._mapDev(out.data_ptr(), 0, stream)
    return out


def vcorr(apply_correction=False, vertical_angle_offset=VERTICAL_ANGLE_OFFSET):
    """madicp_vcorr_t of the reader's `apply_correction` / `vertical_angle_offset`, or None without a correction."""
    if not apply_correction:
        return None
    v = Vcorr()
    v.angle = float(vertical_angle_offset)
    v.enabled = 1
    return v


def _host(d):
    if d.on_device:
        raise TypeError("records: the host restatement needs host records (records.to_host)")
    return d


def range_mask(records, **gate):
    """The gate on the host (madicp_debug_range_mask): uint8 keep flag per record."""
    from . import _capi
    d = _host(describe(records, **gate))
    keep = np.empty(max(int(d.n), 1), np.uint8)
    _capi.check(_capi.lib().madicp_debug_range_mask(C.byref(d), keep.ctypes.data_as(_capi.bp)), "madicp_debug_range_mask")
    return keep[:d.n]


def correct_vertical_angle(records, vertical_angle_offset=VERTICAL_ANGLE_OFFSET, **gate):
    """The kept points of `records` (describe's gate keywords), corrected like KittiReader.apply_rotation_correction,
    on the host with the restatement the device applies (madicp_debug_correct_points): an M x 3 float64 array."""
    from . import _capi
    d = _host(describe(records, **gate))
    v = vcorr(True, vertical_angle_offset)
    out = np.empty((max(int(d.n), 1), 3))
    kept = _capi.check(_capi.lib().madicp_debug_correct_points(C.byref(d), C.byref(v), _capi.as_d(out)),
                       "madicp_debug_correct_points")
    return out[:kept]


__all__ = ["pointcloud2_dtype", "describe", "describe_times", "time_layout", "time_chunks", "chunk_poses", "layout", "to_host", "search_cloud_arrays_dev", "leaves_array_dev", "cloud_array_dev", "map_array_dev", "range_mask", "vcorr", "correct_vertical_angle",
           "VERTICAL_ANGLE_OFFSET", "RANGE_NONE", "RANGE_INCLUSIVE", "RANGE_STRICT"]
