"""Deskew by per-point time stamps (madicp_times_t).  Each kept point takes its chunk from its own stamp:
    u = (tau - t_end) * scale;  s = rint(((-u) * hz) * 1023);  k = 1023 - clip(s, 0, 1023);  p' = pose[k] * p
in float64 without FMA, with the azimuth deskew's chunk poses, the kept points in record order.  The host restatement
(madicp_debug_time_chunks) is checked against an independent numpy evaluation of that rule; the device's clouds, trees
and whole pipelines are checked against the restatement and against the azimuth deskew, bit for bit."""
import ctypes as C
import inspect
import os

import numpy as np
import pytest

from mad_icp_b200 import _capi, records, synth
from util import bits_equal

KITTI_GATE = dict(min_range=0.7, max_range=120.0, inclusive=True, drop_nan=False)
OUSTER_GATE = dict(min_range=1.3, max_range=120.0, inclusive=False, drop_nan=True)
NO_GATE = dict(min_range=0.0, max_range=np.inf, inclusive=True, drop_nan=False)
OUSTER = np.dtype({"names": ["x", "y", "z", "intensity", "t", "reflectivity"],
                   "formats": ["<f4", "<f4", "<f4", "<f4", "<u4", "<u2"], "offsets": [0, 4, 8, 16, 20, 40], "itemsize": 48})
HESAI = np.dtype({"names": ["x", "y", "z", "timestamp"], "formats": ["<f4", "<f4", "<f4", "<f8"],
                  "offsets": [0, 4, 8, 24], "itemsize": 32})
STAMPED = np.dtype({"names": ["x", "y", "z", "t"], "formats": ["<f4", "<f4", "<f4", "<u4"], "offsets": [0, 4, 8, 12],
                    "itemsize": 16})
T_PREV = synth.pose_xyyaw(0.0, 0.0, 0.0)
T_NOW = synth.pose_xyyaw(0.8, 0.05, 0.03)


def rule(tau, t_end, scale, hz):
    """the chunk rule in numpy float64 (no FMA in numpy; np.rint rounds half to even)"""
    u = (np.asarray(tau, np.float64) - np.float64(t_end)) * np.float64(scale)
    s = np.rint(((-u) * np.float64(hz)) * np.float64(1023))
    return (1023 - np.clip(s, 0, 1023)).astype(np.int64)


def _scan(seed, n=4000):
    rs = np.random.RandomState(seed)
    az = rs.uniform(-np.pi, np.pi, n)
    r = rs.uniform(0.5, 60.0, n)
    p = np.stack([r * np.cos(az), r * np.sin(az), rs.uniform(-2, 2, n)], 1)
    p[rs.randint(0, n, n // 40)] = np.nan
    return p


def _kitti(p, tcol):
    a = np.zeros((p.shape[0], 4), np.float32)
    a[:, :3] = p
    a[:, 3] = tcol
    return a


def _struct(p, dtype, field, tau):
    a = np.zeros(p.shape[0], dtype)
    a["x"], a["y"], a["z"] = p[:, 0], p[:, 1], p[:, 2]
    a[field] = tau
    return a


def _kept_tau(a, field, gate):
    keep = records.range_mask(a, **gate).astype(bool)
    col = a[field] if isinstance(field, str) else a[:, field]
    return np.asarray(col)[keep].astype(np.float64)


def _times(offset, ttype, scale=1.0, t_end=None):
    t = _capi.Times()
    t.offset, t.type, t.scale = offset, ttype, scale
    t.t_end, t.has_t_end = (0.0, 0) if t_end is None else (t_end, 1)
    return t


def _chunks(a, tm, hz, gate=NO_GATE, vc=None):
    d = records.describe(a, **gate)
    out = np.empty(max(d.n, 1), np.uint16)
    kept = C.c_int64(0)
    rc = _capi.lib().madicp_debug_time_chunks(C.byref(d), C.byref(vc) if vc else None, C.byref(tm) if tm else None, hz,
                                              out.ctypes.data_as(C.POINTER(C.c_uint16)), C.byref(kept))
    return rc, out[:kept.value].copy()


# =========================================================================== CPU
def test_bindings_and_keywords(built):
    for name in ("madicp_ingest_points_t", "madicp_ingest_points_dev_t", "madicp_plan_points_t", "madicp_plan_points_dev_t",
                 "madicp_debug_time_chunks", "madicp_debug_chunk_poses"):
        assert hasattr(_capi.lib(), name)
    from mad_icp_b200 import Registrar
    from mad_icp_b200.pybind.pypeline import Pipeline
    for m in (Registrar.ingest_records, Registrar.plan_records):
        assert {"time_field", "time_scale", "time_end"} <= set(inspect.signature(m).parameters)
    for m in (Pipeline.computeRecords, Pipeline.prefetchRecords):
        doc = m.__doc__
        assert "time_field" in doc and "time_scale" in doc and "time_end" in doc
    assert "time_field" in inspect.signature(records.pointcloud2_dtype).parameters
    assert _capi.lib().madicp_abi_version() > 0


@pytest.mark.parametrize("tm,msg", [
    (_times(16, records.TIME_U32), "does not fit the stride"),
    (_times(-4, records.TIME_U32), "does not fit the stride"),
    (_times(6, records.TIME_U32), "misaligned"),
    (_times(4, records.TIME_F64), "misaligned"),
    (_times(12, 7), "type must be"),
    (_times(12, -1), "type must be"),
    (_times(12, records.TIME_F32, 0.0), "scale must be finite and > 0"),
    (_times(12, records.TIME_F32, -1e-9), "scale must be finite and > 0"),
    (_times(12, records.TIME_F32, np.nan), "scale must be finite and > 0"),
    (_times(12, records.TIME_F32, np.inf), "scale must be finite and > 0"),
    (_times(12, records.TIME_F32, 1.0, np.nan), "t_end must be finite"),
    (_times(12, records.TIME_F32, 1.0, -np.inf), "t_end must be finite"),
])
def test_invalid_time_descriptors(built, tm, msg):
    a = _kitti(_scan(1), 0.0)
    rc, _ = _chunks(a, tm, 10.0)
    assert rc == -1
    assert msg in _capi.lib().madicp_last_error().decode()


def test_rule_half_steps_tie_to_even(built):
    # stamps v for which ((v * 1.0) * 1023) is exactly n + 0.5 in float64: rint must round to the even neighbour
    v = (2 * np.arange(1, 1023) + 1) / 2046.0
    ties = v[(v * 1023.0) == np.arange(1, 1023) + 0.5]
    assert ties.size > 100
    taus = np.concatenate([-ties, -np.nextafter(ties, 0), -np.nextafter(ties, 1)])
    a = _struct(np.tile([[1.0, 2.0, 3.0]], (taus.size, 1)), HESAI, "timestamp", taus)
    rc, got = _chunks(a, _times(24, records.TIME_F64, 1.0, 0.0), 1.0)
    assert rc == 0
    want = rule(taus, 0.0, 1.0, 1.0)
    assert (got == want).all()
    assert ((1023 - got[:ties.size]) % 2 == 0).all()  # (s = n + 0.5 went to the even one of n, n + 1)


@pytest.mark.parametrize("case", ["u32_wrap", "f64_absolute", "f32_negative", "clamped"])
@pytest.mark.parametrize("explicit_end", [False, True])
def test_restated_chunks_match_numpy(built, case, explicit_end):
    rs = np.random.RandomState(5)
    p = _scan(2, 6000)
    hz = 10.0
    if case == "u32_wrap":  # Ouster ns near 2^32
        tau = (2 ** 32 - 1) - rs.randint(0, 100_000_000, p.shape[0]).astype(np.uint64)
        a, field, tm = _struct(p, OUSTER, "t", tau.astype(np.uint32)), "t", (20, records.TIME_U32, 1e-9)
    elif case == "f64_absolute":  # absolute seconds at ns spacing
        tau = 1.7e9 + np.arange(p.shape[0]) * 1e-9 * 16_000
        a, field, tm = _struct(p, HESAI, "timestamp", tau), "timestamp", (24, records.TIME_F64, 1.0)
    elif case == "f32_negative":  # Velodyne-style float seconds, negative before the sweep end
        tau = rs.uniform(-0.1, 0.0, p.shape[0]).astype(np.float32)
        a, field, tm = _kitti(p, tau), 3, (12, records.TIME_F32, 1.0)
    else:  # after t_end (clamped to 1023) and more than a period before it (clamped to 0)
        tau = rs.uniform(-0.3, 0.2, p.shape[0]).astype(np.float32)
        a, field, tm = _kitti(p, tau), 3, (12, records.TIME_F32, 1.0)
    kept_tau = _kept_tau(a, field, OUSTER_GATE)
    t_end = (float(np.median(kept_tau)) if explicit_end else kept_tau.max())
    rc, got = _chunks(a, _times(*tm, t_end if explicit_end else None), hz, OUSTER_GATE)
    assert rc == 0 and got.size == kept_tau.size
    want = rule(kept_tau, t_end, tm[2], hz)
    assert (got == want).all()
    assert (got == 1023).any() and got.max() == 1023
    if case == "clamped":
        assert (got == 0).any()


def test_nan_stamps(built):
    p = _scan(3)
    tau = np.linspace(-0.1, 0.0, p.shape[0]).astype(np.float32)
    keep = records.range_mask(_kitti(p, tau), **OUSTER_GATE).astype(bool)
    tau_bad = tau.copy()
    tau_bad[np.flatnonzero(~keep)[:5]] = np.nan  # gated-out records: ignored
    rc, got = _chunks(_kitti(p, tau_bad), _times(12, records.TIME_F32), 10.0, OUSTER_GATE)
    assert rc == 0 and (got == _chunks(_kitti(p, tau), _times(12, records.TIME_F32), 10.0, OUSTER_GATE)[1]).all()
    for bad in (np.nan, np.inf, -np.inf):
        tau_bad = tau.copy()
        tau_bad[np.flatnonzero(keep)[7]] = bad
        rc, _ = _chunks(_kitti(p, tau_bad), _times(12, records.TIME_F32), 10.0, OUSTER_GATE)
        assert rc == -3 and "NaN or infinite" in _capi.lib().madicp_last_error().decode()


def _azimuth_plan(a, gate, hz, vc=None):
    d = records.describe(a, **gate)
    n = d.n
    perm, chunk, poses = np.empty(n, np.int32), np.empty(n, np.uint16), np.empty((1024, 12))
    n_poses, kept = C.c_int(0), C.c_int64(0)
    rc = _capi.lib().madicp_debug_deskew_plan(C.byref(d), C.byref(vc) if vc else None, _capi.as_d(_capi.pose12(T_PREV)),
                                              _capi.as_d(_capi.pose12(T_NOW)), hz, 0, 4, _capi.as_i(perm),
                                              chunk.ctypes.data_as(C.POINTER(C.c_uint16)), _capi.as_d(poses),
                                              C.byref(n_poses), C.byref(kept))
    assert rc == 0
    k = kept.value
    return perm[:k].copy(), chunk[:k].copy(), poses[:n_poses.value].copy()


def _presorted(a, perm, chunk):
    """the kept records in the azimuth order, stamped with their azimuth chunk (uint32)"""
    xyz = np.column_stack([a["x"], a["y"], a["z"]]) if a.dtype.names else np.asarray(a[:, :3])
    return _struct(xyz[perm], STAMPED, "t", chunk.astype(np.uint32))


def _time_kw(hz):
    return dict(time_field="t", time_scale=1.0 / (hz * 1023), time_end=1023)


@pytest.mark.parametrize("hz", [10.0, 20.0])
def test_restated_cloud_is_the_azimuth_deskew(built, hz):
    """chunk_poses applied point by point at the restated chunks == the host azimuth deskew (madicp_deskew) when the
    records come pre-sorted and stamped with their azimuth chunks"""
    a = _kitti(_scan(4, 20000), 0.0)
    perm, chunk, poses = _azimuth_plan(a, KITTI_GATE, hz)
    assert int(chunk.max()) <= 1023
    want = np.ascontiguousarray(np.asarray(a[:, :3], np.float64)[perm])
    _capi.check(_capi.lib().madicp_deskew(_capi.as_d(want), want.shape[0], _capi.as_d(_capi.pose12(T_PREV)),
                                          _capi.as_d(_capi.pose12(T_NOW)), hz, 1), "madicp_deskew")
    s = _presorted(a, perm, chunk)
    kw = _time_kw(hz)
    k = records.time_chunks(s, kw["time_field"], kw["time_scale"], hz, t_end=kw["time_end"], **KITTI_GATE)
    assert (k == chunk).all()
    P = records.chunk_poses(T_PREV, T_NOW, hz)
    assert bits_equal(P[:poses.shape[0]].reshape(-1, 12), poses)
    xyz = np.column_stack([s["x"], s["y"], s["z"]]).astype(np.float64)
    R, t = P[k, :, :3], P[k, :, 3]
    got = ((R[:, :, 0] * xyz[:, None, 0] + R[:, :, 1] * xyz[:, None, 1]) + R[:, :, 2] * xyz[:, None, 2]) + t
    assert bits_equal(got, want)


def test_pointcloud2_time_field(built):
    class F:
        def __init__(self, name, offset, datatype, count=1):
            self.name, self.offset, self.datatype, self.count = name, offset, datatype, count

    class Msg:
        fields = [F("x", 0, 7), F("y", 4, 7), F("z", 8, 7), F("intensity", 16, 7), F("t", 20, 6), F("ring", 24, 4)]
        point_step, width, height, row_step, is_bigendian = 48, 10, 1, 480, False

    dt = records.pointcloud2_dtype(Msg())
    assert dt.names == ("x", "y", "z")
    dt = records.pointcloud2_dtype(Msg(), time_field="t")
    assert dt.names == ("x", "y", "z", "t") and dt.fields["t"] == (np.dtype("<u4"), 20) and dt.itemsize == 48
    with pytest.raises(ValueError, match="datatype 4"):
        records.pointcloud2_dtype(Msg(), time_field="ring")
    with pytest.raises(ValueError, match="no time field"):
        records.pointcloud2_dtype(Msg(), time_field="time")
    a = np.zeros(10, dt)
    t = records.describe_times(a, "t", 1e-9)
    assert (t.offset, t.type, t.scale, t.has_t_end) == (20, records.TIME_U32, 1e-9, 0)
    assert records.describe_times(a, None) is None
    t = records.describe_times(np.zeros((4, 5), np.float32), 4, 1.0, 0.5)
    assert (t.offset, t.type, t.t_end, t.has_t_end) == (16, records.TIME_F32, 0.5, 1)
    with pytest.raises(ValueError):
        records.describe_times(np.zeros((4, 5), np.float32), 1)


# =========================================================================== GPU
gpu = pytest.mark.gpu


@pytest.fixture(scope="module")
def reg(built):
    from mad_icp_b200 import Registrar
    return Registrar(device=0, max_keyframes=4)


def _street(seed, beams=32, azimuths=1024):
    scene = synth.StreetScene(seed=7)
    p = synth.lidar_scan(scene, synth.pose_xyyaw(0.3 * seed, 1.0, 0.01 * seed), beams, azimuths, seed=seed, r_min=0.0,
                         r_max=np.inf)
    rs = np.random.RandomState(seed)
    bad = np.concatenate([np.full((7, 3), np.nan), rs.normal(size=(40, 3)) * 0.2, rs.normal(size=(40, 3)) * 300])
    return np.insert(p, np.sort(rs.randint(0, p.shape[0], size=bad.shape[0])), bad, axis=0)


def _restated(a, field, scale, hz, t_end, gate, correction):
    """the host restatement of the time-deskewed cloud: kept (corrected) points, chunk_poses at the restated chunks"""
    k = records.time_chunks(a, field, scale, hz, t_end=t_end, apply_correction=correction, **gate)
    xyz = records.correct_vertical_angle(a, **gate) if correction else None
    if xyz is None:
        keep = records.range_mask(a, **gate).astype(bool)
        src = np.column_stack([a["x"], a["y"], a["z"]]) if a.dtype.names else np.asarray(a[:, :3])
        xyz = src[keep].astype(np.float64)
    P = records.chunk_poses(T_PREV, T_NOW, hz)
    R, t = P[k, :, :3], P[k, :, 3]
    return ((R[:, :, 0] * xyz[:, None, 0] + R[:, :, 1] * xyz[:, None, 1]) + R[:, :, 2] * xyz[:, None, 2]) + t


def _stamped(kind, seed, dtype=np.float32):
    p = _street(seed)
    n = p.shape[0]
    if kind == "kitti":  # float32 N x 4, the time in column 3 (seconds, negative)
        return _kitti(p, np.linspace(-0.1, 0.0, n).astype(np.float32)), 3, 1.0
    if kind == "ouster":  # 48-byte records, uint32 ns at offset 20
        return _struct(p.astype(dtype), OUSTER, "t", np.linspace(0, 99_000_000, n).astype(np.uint32)), "t", 1e-9
    return _struct(p, HESAI, "timestamp", 1.7e9 + np.linspace(0.0, 0.1, n)), "timestamp", 1.0  # float64 seconds


GPU_CASES = [("kitti", KITTI_GATE, False), ("kitti", KITTI_GATE, True), ("kitti", NO_GATE, False),
             ("ouster", OUSTER_GATE, False), ("ouster", OUSTER_GATE, True), ("hesai", OUSTER_GATE, False)]


@gpu
@pytest.mark.parametrize("explicit_end", [False, True])
@pytest.mark.parametrize("kind,gate,correction", GPU_CASES)
def test_device_cloud_and_tree_equal_restatement(reg, kind, gate, correction, explicit_end):
    a, field, scale = _stamped(kind, 3)
    hz = 10.0
    t_end = float(_kept_tau(a, field, gate).max()) - 0.02 / scale if explicit_end else None
    want = _restated(a, field, scale, hz, t_end, gate, correction)
    kw = dict(deskew=True, T_prev=T_PREV, T_now=T_NOW, sensor_hz=hz, apply_correction=correction, time_field=field,
              time_scale=scale, time_end=t_end)
    got = reg.ingest_records(a, **gate, want_points=True, **kw)
    assert got.shape == want.shape and bits_equal(got, want)
    # the tree of the device cloud == the tree of the restated cloud; a plan gives the same cloud
    reg.ingest_records(a, **gate, **kw)
    t_dev = reg.build_tree()
    t_host = reg.build_tree(want)
    assert (t_dev.records()["link"] == t_host.records()["link"]).all()
    assert bits_equal(t_dev.records()["mean"], t_host.records()["mean"])
    plan = reg.plan_records(a, **gate, apply_correction=correction, time_field=field, time_scale=scale, time_end=t_end)
    got = reg.ingest_plan(plan, deskew=True, T_prev=T_PREV, T_now=T_NOW, sensor_hz=hz, want_points=True)
    assert bits_equal(got, want)


@gpu
@pytest.mark.parametrize("shift", [0, 4, 8, 12])
@pytest.mark.parametrize("kind", ["kitti", "ouster"])
def test_cuda_tensor_records_at_shifted_bases(reg, kind, shift):
    import torch
    a, field, scale = _stamped(kind, 4)
    hz = 20.0
    want = _restated(a, field, scale, hz, None, OUSTER_GATE, False)
    raw = np.frombuffer(a.tobytes(), np.uint8)
    buf = torch.zeros(raw.size + 64, dtype=torch.uint8, device="cuda")
    buf[shift:shift + raw.size] = torch.from_numpy(raw.copy()).cuda()
    stride = a.dtype.itemsize if a.dtype.names else a.strides[0]
    if kind == "kitti":
        dev = buf[shift:shift + raw.size].view(torch.float32).view(-1, 4)
    else:  # x, y, z and t of the 48-byte records as a strided float32 view (12 floats per record)
        dev = buf[shift:shift + raw.size].view(torch.float32).view(-1, stride // 4)
    kw = dict(deskew=True, T_prev=T_PREV, T_now=T_NOW, sensor_hz=hz, time_scale=scale)
    if kind == "kitti":
        got = reg.ingest_records(dev, **OUSTER_GATE, want_points=True, time_field=field, **kw)
        assert bits_equal(got, want)
        plan = reg.plan_records(dev, **OUSTER_GATE, time_field=field, time_scale=scale)
        assert bits_equal(reg.ingest_plan(plan, deskew=True, T_prev=T_PREV, T_now=T_NOW, sensor_hz=hz, want_points=True), want)
    else:  # a uint32 field needs a structured description: through the C ABI with the device pointer
        d = records.describe(dev, **OUSTER_GATE)
        t = _times(20, records.TIME_U32, scale)
        out, kept = np.empty((d.n, 3)), C.c_int64(0)
        _capi.check(_capi.lib().madicp_ingest_points_dev_t(reg._h, C.byref(d), None, C.byref(t), 1,
                                                           _capi.as_d(_capi.pose12(T_PREV)), _capi.as_d(_capi.pose12(T_NOW)),
                                                           hz, 1, d.stream, C.byref(kept), _capi.as_d(out)), "ingest")
        assert bits_equal(out[:kept.value], want)


def _pipeline(hz, deskew=True, gpu_build=True):
    from mad_icp_b200.pybind.pypeline import Pipeline
    os.environ["MADICP_GPU_BUILD"] = "1" if gpu_build else "0"
    try:
        return Pipeline(sensor_hz=hz, deskew=deskew, b_max=0.2, rho_ker=0.1, p_th=0.8, b_min=0.1, b_ratio=0.02,
                        num_keyframes=4, num_threads=4, realtime=False)
    finally:
        os.environ.pop("MADICP_GPU_BUILD")


def _sequence(n):
    scene = synth.StreetScene(seed=7, x_min=-45.0, x_max=60.0 + 0.8 * n)
    out = []
    for i in range(n):
        base = synth.pose_xyyaw(0.8 * i, 1.0 + 0.3 * np.sin(0.05 * i), 0.02 * np.sin(0.03 * i))
        p = synth.lidar_scan(scene, base, beams=32, azimuths=1024, seed=100 + i, r_min=0.0, r_max=np.inf)
        rs = np.random.RandomState(i)
        p = np.insert(p, np.sort(rs.randint(0, p.shape[0], size=p.shape[0] // 20)), np.nan, axis=0)
        out.append(_kitti(p, 0.0)[:, :3])
    return out


def _state(p):
    return p.currentPose().copy(), bool(p.isMapUpdated()), int(p.keyframeID()), int(p.numKeyframes())


def _run(seq, hz, mode, depth=0, tkw=None, device=False):
    import torch
    p = _pipeline(hz, gpu_build=mode != "host")
    if device:  # float32 N x 4 CUDA tensors, the stamp (a chunk number, exact in float32) in column 3
        items = [torch.from_numpy(np.column_stack([a["x"], a["y"], a["z"], a["t"].astype(np.float32)])).cuda() for a in seq]
        tkw = dict(tkw, time_field=3)
    else:
        items = seq
    out, queued = [], 0
    for i, a in enumerate(items):
        if mode == "prefetch":
            while queued < min(i + depth, len(items)):
                assert p.prefetchRecords(items[queued], **KITTI_GATE, deskew_ahead=True, **(tkw or {}))
                queued += 1
        p.computeRecords(0.1 * i, a, **KITTI_GATE, **(tkw or {}))
        out.append(_state(p))
    return out


def _same_run(got, want, what):
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        assert bits_equal(g[0], w[0]), (what, i)
        assert g[1:] == w[1:], (what, i)


@gpu
@pytest.mark.parametrize("hz", [10.0, 20.0])
def test_time_deskew_is_the_azimuth_deskew(reg, hz):
    """Records handed over pre-sorted by the azimuth permutation and stamped with their azimuth chunks give the azimuth
    deskew's cloud and tree, and whole pipelines the same trajectory and keyframe decisions."""
    seq = _sequence(40)
    a = seq[3]
    perm, chunk, _ = _azimuth_plan(a, KITTI_GATE, hz)
    s = _presorted(a, perm, chunk)
    kw = dict(deskew=True, T_prev=T_PREV, T_now=T_NOW, sensor_hz=hz)
    want = reg.ingest_records(a, **KITTI_GATE, want_points=True, **kw)
    t_az = reg.build_tree(want)
    got = reg.ingest_records(s, **KITTI_GATE, want_points=True, **kw, **_time_kw(hz))
    assert bits_equal(got, want)
    t_tm = reg.build_tree()
    assert (t_az.records()["link"] == t_tm.records()["link"]).all() and bits_equal(t_az.records()["mean"], t_tm.records()["mean"])
    # sequences: the azimuth pipeline on the raw records, the time pipeline on the stamped, pre-sorted ones
    # (the first two scans are not deskewed: their trees are built in record order, so they go over as they are)
    stamped = [_presorted(x, *_azimuth_plan(x, KITTI_GATE, hz)[:2]) if i >= 2 else
               _struct(np.asarray(x, np.float64), STAMPED, "t", 0) for i, x in enumerate(seq)]
    want = _run(seq, hz, "records")
    assert sum(o[1] for o in want) >= 3
    tkw = _time_kw(hz)
    _same_run(_run(stamped, hz, "records", tkw=tkw), want, "time")
    for depth in (1, 5, 32):
        _same_run(_run(stamped, hz, "prefetch", depth, tkw=tkw), want, ("prefetch", depth))
    _same_run(_run(stamped, hz, "records", tkw=tkw, device=True), want, "cuda")
    _same_run(_run(stamped, hz, "prefetch", 5, tkw=tkw, device=True), want, "cuda-prefetch")
    _same_run(_run(stamped, hz, "host", tkw=tkw), want, "host")


@gpu
def test_non_deskewing_pipeline_ignores_the_time_field(built):
    seq = _sequence(8)
    stamped = [_struct(np.asarray(a, np.float64), STAMPED, "t", np.arange(a.shape[0], dtype=np.uint32)) for a in seq]
    stamped[5]["t"][3] = 0xFFFFFFFF
    want, got, ahead = _pipeline(10.0, deskew=False), _pipeline(10.0, deskew=False), _pipeline(10.0, deskew=False)
    for s in stamped:
        assert ahead.prefetchRecords(s, **KITTI_GATE, time_field="t", time_scale=1e-9)
    for i, s in enumerate(stamped):
        want.computeRecords(0.1 * i, s, **KITTI_GATE)
        got.computeRecords(0.1 * i, s, **KITTI_GATE, time_field="t", time_scale=1e-9)
        ahead.computeRecords(0.1 * i, s, **KITTI_GATE, time_field="t", time_scale=1e-9)
        assert bits_equal(got.currentPose(), want.currentPose()) and bits_equal(ahead.currentPose(), want.currentPose())


@gpu
@pytest.mark.parametrize("mode", ["records", "prefetch", "cuda"])
def test_nan_stamp_fails_once(built, mode):
    import torch
    seq = _sequence(6)
    hz = 10.0
    stamped = [_kitti(np.asarray(a, np.float64), np.linspace(-0.1, 0.0, a.shape[0]).astype(np.float32)) for a in seq]
    keep = records.range_mask(stamped[3], **KITTI_GATE).astype(bool)
    stamped[3][np.flatnonzero(keep)[10], 3] = np.nan  # a kept record
    stamped[4][np.flatnonzero(~records.range_mask(stamped[4], **KITTI_GATE).astype(bool))[0], 3] = np.nan  # gated out
    tkw = dict(time_field=3, time_scale=1.0)
    items = [torch.from_numpy(s).cuda() for s in stamped] if mode == "cuda" else stamped
    p, ref = _pipeline(hz), _pipeline(hz)
    if mode == "prefetch":
        for s in items:
            assert p.prefetchRecords(s, **KITTI_GATE, deskew_ahead=True, **tkw)
    for i, s in enumerate(items):
        if i == 3:
            with pytest.raises(RuntimeError, match=r"\(-3\).*NaN or infinite") as e:
                p.computeRecords(0.1 * i, s, **KITTI_GATE, **tkw)
            assert type(e.value).__name__ == "MadIcpError"
            continue
        p.computeRecords(0.1 * i, s, **KITTI_GATE, **tkw)
        ref.computeRecords(0.1 * i, stamped[i], **KITTI_GATE, **tkw)
        assert bits_equal(p.currentPose(), ref.currentPose()), i


@gpu
def test_stamps_written_behind_a_side_stream(reg):
    import torch
    a, field, scale = _stamped("kitti", 5)
    want = _restated(a, field, scale, 10.0, None, KITTI_GATE, False)
    src = torch.from_numpy(a).cuda()
    side = torch.cuda.Stream()
    dev = torch.zeros_like(src)
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        torch.cuda._sleep(50_000_000)
        dev.copy_(src)
    with torch.cuda.stream(side):
        got = reg.ingest_records(dev, **KITTI_GATE, want_points=True, deskew=True, T_prev=T_PREV, T_now=T_NOW,
                                 sensor_hz=10.0, time_field=field, time_scale=scale)
    assert bits_equal(got, want)
