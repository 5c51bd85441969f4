"""Raw sensor records on the way in (madicp_points_t): strided x/y/z fields, the dataset readers' range gate and NaN
drop.  The reader expressions of apps/utils/kitti_reader.py:82-88 and apps/utils/point_cloud2.py:77-87 are restated
here in numpy; the host predicate (madicp_debug_range_mask) must agree with them record for record, and on the GPU the
kept cloud, the trees and whole pipelines must be those of the numpy-filtered arrays, bit for bit."""
import ctypes as C
import math
import os

import numpy as np
import pytest

from mad_icp_b200 import _capi, records, synth
from util import bits_equal

OUSTER = np.dtype({"names": ["x", "y", "z", "intensity", "t", "reflectivity"],
                   "formats": ["<f4", "<f4", "<f4", "<f4", "<u4", "<u2"], "offsets": [16, 20, 24, 28, 32, 40], "itemsize": 48})


# ---- the readers, restated
def kitti_mask(pts, lo, hi):
    norms = np.linalg.norm(pts, axis=1)
    return (norms >= lo) & (norms <= hi)


def pc2_mask(pts, lo, hi):
    """point_cloud2.py drops NaN rows, then gates strictly: as a mask over the records"""
    nan = np.any(np.isnan(pts), axis=1)
    norms = np.linalg.norm(pts, axis=1)
    return ~nan & (norms > lo) & (norms < hi)


def _hard_points(dtype, lo, hi, n_random=20000, seed=0):
    """Points at and next to the bounds (in the field type), points whose norm depends on the summation order, NaN in
    each coordinate, +-inf, zero rows."""
    rs = np.random.RandomState(seed)
    t = np.dtype(dtype).type
    rows = []
    for b in (t(lo), t(hi)):
        for v in (np.nextafter(b, t(-np.inf)), b, np.nextafter(b, t(np.inf))):
            rows += [[v, 0, 0], [0, v, 0], [0, 0, -v]]
    # random directions with norms within a few ulps of the bounds: the gate decision hangs on the rounding
    for b in (lo, hi):
        d = rs.normal(size=(n_random, 3))
        d /= np.linalg.norm(d, axis=1, keepdims=True)
        r = b * (1 + rs.randint(-8, 9, size=(n_random, 1)) * np.finfo(dtype).eps)
        rows += list((d * r).astype(dtype))
    rows += [[np.nan, 1, 1], [1, np.nan, 1], [1, 1, np.nan], [np.inf, 0, 0], [0, -np.inf, 0], [0, 0, 0], [0, 0, 0]]
    rows += list(rs.uniform(-150, 150, size=(2000, 3)).astype(dtype))
    return np.array(rows, dtype=dtype)


def test_summation_order_matters_for_the_inputs():
    """sanity of the fixture: numpy's norm is ((x*x + y*y) + z*z) and the other order differs on many of these points"""
    p = _hard_points(np.float32, 0.7, 120.0)
    p = p[np.isfinite(p).all(1)]
    a = np.sqrt((p[:, 0] * p[:, 0] + p[:, 1] * p[:, 1]) + p[:, 2] * p[:, 2])
    b = np.sqrt(p[:, 0] * p[:, 0] + (p[:, 1] * p[:, 1] + p[:, 2] * p[:, 2]))
    assert (np.linalg.norm(p, axis=1) == a).all()
    assert (a != b).sum() > 1000


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("lo,hi", [(0.7, 120.0), (0.0, 50.0), (1.3, 120.0)])
def test_range_mask_is_the_readers(built, dtype, lo, hi):
    pts = _hard_points(dtype, lo, hi)
    n = pts.shape[0]
    kitti = np.zeros((n, 4), dtype)  # a KITTI .bin: 16-byte (32-byte) records, x/y/z/intensity
    kitti[:, :3] = pts
    kitti[:, 3] = 0.25
    view = kitti[:, :3]
    assert (records.range_mask(view, min_range=lo, max_range=hi) == kitti_mask(view, lo, hi)).all()
    assert (records.range_mask(view, min_range=lo, max_range=hi, inclusive=False, drop_nan=True) ==
            pc2_mask(view, lo, hi)).all()
    # a PointCloud2 of 48-byte Ouster-like records, xyz at 16/20/24 (float32) -- or a float64 one at 8/16/24
    if dtype == np.float32:
        rec = np.zeros(n, OUSTER)
    else:
        rec = np.zeros(n, np.dtype({"names": ["x", "y", "z"], "formats": ["<f8"] * 3, "offsets": [8, 16, 24], "itemsize": 48}))
    rec["x"], rec["y"], rec["z"] = pts[:, 0], pts[:, 1], pts[:, 2]
    xyz = np.column_stack([rec["x"], rec["y"], rec["z"]])  # point_cloud2.py:78-80
    assert (records.range_mask(rec, min_range=lo, max_range=hi, inclusive=False, drop_nan=True) == pc2_mask(xyz, lo, hi)).all()
    assert (records.range_mask(rec, min_range=lo, max_range=hi) == kitti_mask(xyz, lo, hi)).all()


def _points(a, mode, lo=0.0, hi=math.inf, drop_nan=0):
    d = records.describe(a, lo, hi)
    d.range_mode, d.drop_nan = mode, drop_nan
    return d


def test_no_gate_and_nan_drop(built):
    pts = _hard_points(np.float32, 0.7, 120.0)
    L = _capi.lib()
    keep = np.empty(len(pts), np.uint8)
    d = _points(pts, records.RANGE_NONE)
    assert L.madicp_debug_range_mask(C.byref(d), _capi.as_b(keep)) == len(pts) and keep.all()
    d = _points(pts, records.RANGE_NONE, drop_nan=1)
    assert L.madicp_debug_range_mask(C.byref(d), _capi.as_b(keep)) == (~np.isnan(pts).any(1)).sum()
    assert (keep == ~np.isnan(pts).any(1)).all()


def test_bounds_are_rounded_to_the_field_type(built):
    """np.float32(0.7) >= 0.7 is True under numpy's rules: the bound is compared in float32"""
    f = np.float32(0.7)
    pts = np.array([[f, 0, 0], [np.nextafter(f, np.float32(0)), 0, 0]], np.float32)
    assert (records.range_mask(pts, min_range=0.7, max_range=1.0) == [1, 0]).all()
    assert (records.range_mask(pts.astype(np.float64), min_range=0.7, max_range=1.0) == kitti_mask(pts.astype(np.float64), 0.7, 1.0)).all()


def test_invalid_descriptors_are_rejected(built):
    L = _capi.lib()
    base = np.zeros((10, 4), np.float32)
    keep = np.empty(10, np.uint8)

    def rc(**kw):
        d = records.describe(base[:, :3], 0.5, 10.0)
        for k, v in kw.items():
            if k == "offset":
                d.offset[:] = v
            else:
                setattr(d, k, v)
        r = L.madicp_debug_range_mask(C.byref(d), _capi.as_b(keep))
        return r, L.madicp_last_error().decode()

    assert rc()[0] == 0
    cases = [dict(data=None), dict(n=0), dict(n=(1 << 24) + 1), dict(offset=[0, 4, 16]), dict(offset=[0, 4, -4]),
             dict(offset=[0, 2, 8]), dict(stride=14), dict(stride=0), dict(is_f32=0, offset=[0, 8, 4]),
             dict(min_range=float("nan")), dict(max_range=float("nan")), dict(min_range=2.0, max_range=1.0),
             dict(range_mode=3), dict(range_mode=-1)]
    for kw in cases:
        r, msg = rc(**kw)
        assert r == -1, kw  # MADICP_ERR_INVALID
        assert msg.startswith("madicp_debug_range_mask: ") and len(msg) > 30, (kw, msg)
    with pytest.raises(ValueError):
        records.describe(base.astype(">f4")[:, :3])
    with pytest.raises(ValueError):
        records.describe(base[:, :2])


def test_abi_version_bumped(built):
    assert _capi.lib().madicp_abi_version() == 3


class _Field:
    def __init__(self, name, offset, datatype, count=1):
        self.name, self.offset, self.datatype, self.count = name, offset, datatype, count


class _Msg:
    def __init__(self, fields, point_step=48, width=100, height=1, row_step=None, is_bigendian=False):
        self.fields, self.point_step, self.width, self.height = fields, point_step, width, height
        self.row_step = width * point_step if row_step is None else row_step
        self.is_bigendian = is_bigendian


def test_pointcloud2_dtype():
    ouster = [_Field("x", 16, 7), _Field("y", 20, 7), _Field("z", 24, 7), _Field("intensity", 28, 7), _Field("t", 32, 6)]
    dt = records.pointcloud2_dtype(_Msg(ouster))
    assert dt.itemsize == 48 and [dt.fields[k][1] for k in "xyz"] == [16, 20, 24] and dt["x"] == np.dtype("<f4")
    buf = np.zeros(100, OUSTER)
    buf["y"] = np.arange(100)
    a = np.frombuffer(buf.tobytes(), dt)
    assert (a["y"] == np.arange(100)).all()
    with pytest.raises(ValueError, match="big-endian"):
        records.pointcloud2_dtype(_Msg(ouster, is_bigendian=True))
    with pytest.raises(ValueError, match="row_step"):
        records.pointcloud2_dtype(_Msg(ouster, row_step=4864))
    with pytest.raises(ValueError, match="share"):
        records.pointcloud2_dtype(_Msg([_Field("x", 0, 7), _Field("y", 8, 8), _Field("z", 16, 8)], point_step=24))
    with pytest.raises(ValueError, match="datatype"):
        records.pointcloud2_dtype(_Msg([_Field("x", 0, 7), _Field("y", 4, 7), _Field("z", 8, 4)], point_step=16))


# =========================================================================== GPU
gpu = pytest.mark.gpu


@pytest.fixture(scope="module")
def reg(built):
    from mad_icp_b200 import Registrar
    return Registrar(device=0, max_keyframes=4)


def _scan(seed, beams=32, azimuths=1024, inject=True):
    """a synthetic sweep without the range gate + injected NaN / zero / too-near / too-far rows, as N x 3 float64"""
    scene = synth.StreetScene(seed=7)
    p = synth.lidar_scan(scene, synth.pose_xyyaw(0.3 * seed, 1.0, 0.01 * seed), beams, azimuths, seed=seed, r_min=0.0,
                         r_max=np.inf)
    if not inject:
        return p
    rs = np.random.RandomState(seed)
    bad = np.concatenate([np.full((7, 3), np.nan), np.zeros((5, 3)), rs.normal(size=(40, 3)) * 0.2,
                          rs.normal(size=(40, 3)) * 300, [[np.nan, 1, 2], [3, np.nan, 4], [5, 6, np.nan]]])
    at = np.sort(rs.randint(0, p.shape[0], size=bad.shape[0]))
    return np.insert(p, at, bad, axis=0)


def _kitti(p, dtype=np.float32):
    a = np.zeros((p.shape[0], 4), dtype)
    a[:, :3] = p
    a[:, 3] = 0.5
    return a


def _ouster(p, dtype=np.float32):
    if dtype == np.float32:
        a = np.zeros(p.shape[0], OUSTER)
    else:
        a = np.zeros(p.shape[0], np.dtype({"names": ["x", "y", "z"], "formats": ["<f8"] * 3, "offsets": [8, 16, 24],
                                           "itemsize": 48}))
    a["x"], a["y"], a["z"] = p[:, 0], p[:, 1], p[:, 2]
    return a


def _xyz(a):
    return a[:, :3] if a.dtype.names is None else np.column_stack([a["x"], a["y"], a["z"]])


@gpu
@pytest.mark.parametrize("layout", ["kitti", "ouster"])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("inclusive", [True, False])
def test_kept_cloud_is_the_readers(reg, layout, dtype, inclusive):
    p = _scan(3)
    a = (_kitti if layout == "kitti" else _ouster)(p, dtype)
    xyz = _xyz(a)
    lo, hi = 0.7, 120.0
    mask = kitti_mask(xyz, lo, hi) if inclusive else pc2_mask(xyz, lo, hi)
    want = xyz[mask].astype(np.float64)
    got = reg.ingest_records(a, lo, hi, inclusive=inclusive, drop_nan=not inclusive, want_points=True)
    assert got.shape == want.shape and bits_equal(got, want)
    assert reg.ingest_records(a, lo, hi, inclusive=inclusive, drop_nan=not inclusive) == want.shape[0]


def _same_tree(a, b):
    for k in ("mean", "eivecs", "bbox"):
        assert bits_equal(a[0][k], b[0][k]), k
    assert (a[0]["num_points"] == b[0]["num_points"]).all()
    assert a[1].tobytes() == b[1].tobytes() or all(bits_equal(a[1][k], b[1][k]) for k in ("mean", "dir", "bbox0"))
    assert (a[1]["link"] == b[1]["link"]).all() and (a[2] == b[2]).all()


def _dump(dt):
    return dt.export(), dt.records(), dt.leaf_records()


@gpu
@pytest.mark.parametrize("deskew", [False, True])
@pytest.mark.parametrize("layout", ["kitti", "ouster"])
def test_tree_from_records_is_the_filtered_clouds(reg, layout, deskew):
    p = _scan(5)
    a = (_kitti if layout == "kitti" else _ouster)(p)
    filt = _xyz(a)[kitti_mask(_xyz(a), 0.7, 120.0)]
    kw = dict(deskew=deskew, T_prev=synth.pose_xyyaw(0, 0, 0), T_now=synth.pose_xyyaw(0.8, 0.05, 0.03), sensor_hz=10.0,
              num_threads=4) if deskew else {}
    reg.ingest_records(a, 0.7, 120.0, **kw)
    got = _dump(reg.build_tree())
    reg.ingest(np.ascontiguousarray(filt), **kw)
    want = _dump(reg.build_tree())
    _same_tree(got, want)


@gpu
def test_forest_of_records_staged_all_partial_none(reg, capfd, monkeypatch):
    scans = [_kitti(_scan(s)) for s in (11, 12, 13, 14, 15)]
    scans[2] = scans[2][:3000]  # different survivor counts
    gate = dict(min_range=0.7, max_range=120.0)
    want = []
    for a in scans:
        filt = np.ascontiguousarray(a[:, :3][kitti_mask(a[:, :3], 0.7, 120.0)])
        want.append(reg.build_trees([filt])[0].records())
    total = sum(a.shape[0] for a in scans)
    monkeypatch.setenv("MADICP_BUILD_TIMING", "1")  # the batch call reports how many of its scans came staged
    for n_staged in (5, 2, 0):
        for a in scans[:n_staged]:
            reg.stage_records(a[:, :3], total, **gate)
        capfd.readouterr()
        trees = reg.build_trees_records([a[:, :3] for a in scans], **gate)
        err = capfd.readouterr().err
        assert f"madtree_gpu_build_batch_points: 5 scans ({n_staged} staged)" in err, err
        for dt, w in zip(trees, want):
            r = dt.records()
            assert all(bits_equal(r[k], w[k]) for k in ("mean", "dir", "bbox0")), n_staged
            assert (r["link"] == w["link"]).all() and (r["num_points"] == w["num_points"]).all(), n_staged


@gpu
def test_empty_scan_raises_and_the_next_one_works(reg):
    from mad_icp_b200 import MadIcpError
    from mad_icp_b200.pybind.pypeline import Pipeline
    far = _kitti(np.full((100, 3), 500.0))
    with pytest.raises(MadIcpError, match="range gate"):
        reg.ingest_records(far[:, :3], 0.7, 120.0)
    a = _kitti(_scan(2))
    assert reg.ingest_records(a[:, :3], 0.7, 120.0) > 0
    p = Pipeline(sensor_hz=10.0, deskew=False, b_max=0.2, rho_ker=0.1, p_th=0.8, b_min=0.1, b_ratio=0.02, num_keyframes=4,
                 num_threads=4, realtime=False)
    p.computeRecords(0.0, a[:, :3], 0.7, 120.0)
    with pytest.raises(Exception, match="range gate"):
        p.computeRecords(0.1, far[:, :3], 0.7, 120.0)
    p.computeRecords(0.1, _kitti(_scan(3))[:, :3], 0.7, 120.0)
    assert p.currentID() == 2


def _pipeline(**kw):
    from mad_icp_b200.pybind.pypeline import Pipeline
    args = dict(sensor_hz=10.0, deskew=False, b_max=0.2, rho_ker=0.1, p_th=0.8, b_min=0.1, b_ratio=0.02, num_keyframes=4,
                num_threads=4, realtime=False)
    args.update(kw)
    return Pipeline(**args)


@gpu
def test_prefetched_empty_scan_raises_at_that_scan_and_the_queue_goes_on(built):
    """A look-ahead batch holding a scan the gate leaves empty: compute raises exactly when it reaches that scan, and
    every other scan gets the pose of the run without look-ahead (which raises at the same scan)."""
    seq = _sequence(14)
    bad = 6
    seq[bad] = _kitti(np.full((500, 3), 500.0))  # nothing inside 0.7..120 m
    lo, hi = 0.7, 120.0

    def run(prefetch):
        p = _pipeline()
        out = []
        for i, a in enumerate(seq):
            if prefetch and i >= 1 and p.prefetched() == 0:
                for k in range(i, len(seq)):  # one look-ahead batch with the empty scan in its middle
                    assert p.prefetchRecords(seq[k][:, :3], lo, hi)
            try:
                p.computeRecords(0.1 * i, a[:, :3], lo, hi)
                out.append(p.currentPose().copy())
            except RuntimeError as e:  # (MadIcpError of whichever pybind module registered it first)
                assert "range gate" in str(e), e
                out.append(None)
        assert p.prefetched() == 0
        return out

    want, got = run(False), run(True)
    assert [i for i, x in enumerate(want) if x is None] == [bad]
    assert [i for i, x in enumerate(got) if x is None] == [bad]
    for i in range(len(seq)):
        if i != bad:
            assert bits_equal(got[i], want[i]), i
    # a descriptor the library rejects never enters the queue
    p = _pipeline()
    p.computeRecords(0.0, seq[0][:, :3], lo, hi)
    odd = np.zeros(100, np.dtype({"names": ["x", "y", "z"], "formats": ["<f4"] * 3, "offsets": [2, 6, 10], "itemsize": 16}))
    with pytest.raises(RuntimeError, match="offset"):
        p.prefetchRecords(odd, lo, hi)
    assert p.prefetched() == 0
    assert p.prefetchRecords(seq[1][:, :3], lo, hi)
    p.computeRecords(0.1, seq[1][:, :3], lo, hi)
    assert p.currentID() == 2


def test_column_major_records_are_rejected_with_a_hint():
    a = np.asfortranarray(np.zeros((100, 3), np.float32))
    with pytest.raises(ValueError, match="column-major"):
        records.describe(a)
    records.describe(np.ascontiguousarray(a))
    records.describe(np.zeros((100, 4), np.float32)[:, :3])


def _sequence(n):
    scene = synth.StreetScene(seed=7, x_min=-45.0, x_max=60.0 + 0.8 * n)
    out = []
    for i in range(n):
        base = synth.pose_xyyaw(0.8 * i, 1.0 + 0.3 * np.sin(0.05 * i), 0.02 * np.sin(0.03 * i))
        p = synth.lidar_scan(scene, base, beams=32, azimuths=1024, seed=100 + i, r_min=0.0, r_max=np.inf)
        rs = np.random.RandomState(i)
        bad = np.concatenate([np.full((3, 3), np.nan), np.zeros((4, 3)), rs.normal(size=(20, 3)) * 0.3,
                              rs.normal(size=(20, 3)) * 400.0])
        p = np.insert(p, np.sort(rs.randint(0, p.shape[0], size=bad.shape[0])), bad, axis=0)
        out.append(_kitti(p))
    return out


@gpu
@pytest.mark.parametrize("deskew", [False, True])
def test_pipeline_records_equal_filtered_compute(built, deskew):
    from mad_icp_b200.pybind.pypeline import Pipeline
    seq = _sequence(40)
    lo, hi = 0.7, 120.0
    kw = dict(sensor_hz=10.0, deskew=deskew, b_max=0.2, rho_ker=0.1, p_th=0.8, b_min=0.1, b_ratio=0.02, num_keyframes=4,
              num_threads=4, realtime=False)

    def run(mode):
        os.environ["MADICP_GPU_BUILD"] = "0" if mode == "host" else "1"
        try:
            p = Pipeline(**kw)
        finally:
            os.environ.pop("MADICP_GPU_BUILD")
        out = []
        for i, a in enumerate(seq):
            if mode == "filtered":
                p.compute(0.1 * i, a[:, :3][kitti_mask(a[:, :3], lo, hi)])
            else:
                if mode == "prefetch" and i >= 1 and p.prefetched() == 0:
                    for k in range(i, min(i + 6, len(seq))):
                        assert p.prefetchRecords(seq[k][:, :3], lo, hi) != deskew
                p.computeRecords(0.1 * i, a[:, :3], lo, hi)
            out.append((p.currentPose().copy(), bool(p.isMapUpdated()), int(p.keyframeID()), int(p.numKeyframes())))
        return out

    want = run("filtered")
    assert sum(o[1] for o in want) >= 3
    for mode in ("records", "prefetch", "host"):
        got = run(mode)
        for i in range(len(seq)):
            assert bits_equal(got[i][0], want[i][0]), (mode, i)
            assert got[i][1:] == want[i][1:], (mode, i)
