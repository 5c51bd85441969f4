"""KITTI's vertical-angle correction on the way in (madicp_vcorr_t).  The reader's expression
(apps/utils/kitti_reader.py:72-79: np.cross, np.linalg.norm, scipy's Rotation.from_rotvec(...).apply, applied to the
points the range mask keeps) is the yardstick: the host restatement (madicp_debug_correct_points) must reproduce it
bit for bit, and on the GPU the kept cloud, the trees and whole pipelines must be those of the reader's corrected
float64 arrays.  The restatement is pinned to the installed scipy: if scipy changes its order, these tests fail."""
import ctypes as C
import inspect
import math
import os
import re

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from mad_icp_b200 import _capi, records, synth
from util import bits_equal

THETAS = [np.radians(0.205), 5e-4, 0.3, 0.0]  # the reader's, scipy's Taylor branch (a <= 1e-3), a large one, none
OUSTER = np.dtype({"names": ["x", "y", "z", "intensity", "t", "reflectivity"],
                   "formats": ["<f4", "<f4", "<f4", "<f4", "<u4", "<u2"], "offsets": [16, 20, 24, 28, 32, 40], "itemsize": 48})
OUSTER64 = np.dtype({"names": ["x", "y", "z"], "formats": ["<f8"] * 3, "offsets": [8, 16, 24], "itemsize": 48})


# ---- the reader, verbatim
def reader_correction(points, theta):
    with np.errstate(all="ignore"):
        rotation_vectors = np.cross(points, np.array([0., 0., 1.]))
        norms = np.linalg.norm(rotation_vectors, axis=1).reshape(-1, 1)
        rotation_vectors_normalized = rotation_vectors / norms
        return Rotation.from_rotvec(theta * rotation_vectors_normalized).apply(points)


def kitti_mask(pts, lo, hi):
    norms = np.linalg.norm(pts, axis=1)
    return (norms >= lo) & (norms <= hi)


def same_cloud(got, want):
    """bit for bit where the reader's row is not NaN, and NaN rows in the same places"""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    if got.shape != want.shape:
        return False
    nan_g, nan_w = np.isnan(got).any(1), np.isnan(want).any(1)
    return bool((nan_g == nan_w).all() and bits_equal(got[~nan_w], want[~nan_w]))


def _points(dtype, n=200_000, seed=0):
    """KITTI-shape points (a 120 m sweep around a car, ground and walls) and degenerate rows: x = y = 0, signed zeros
    in each field, subnormal x / y, very large coordinates."""
    rs = np.random.RandomState(seed)
    az = rs.uniform(-np.pi, np.pi, n)
    el = rs.uniform(np.radians(-24.9), np.radians(2.0), n)
    r = rs.uniform(0.5, 120.0, n)
    p = np.column_stack([r * np.cos(el) * np.cos(az), r * np.cos(el) * np.sin(az), r * np.sin(el)])
    t = np.dtype(dtype).type
    tiny = np.finfo(dtype).smallest_subnormal
    deg = [[0, 0, 5], [0, 0, -5], [-0.0, 0, 3], [0, -0.0, 3], [-0.0, -0.0, 3], [0, 0, 0], [-0.0, -0.0, -0.0],
           [3, 4, 0], [3, 4, -0.0], [-0.0, 4, 1], [3, -0.0, 1], [-3, -0.0, -0.0],
           [tiny, 0, 2], [0, tiny, 2], [tiny, tiny, 2], [-tiny, 5 * tiny, 1], [tiny, 1, 1], [1, -tiny, 1],
           [1e20, 1e20, 1], [-1e20, 3, 1e20], [3e37, -3e37, 2], [1e-20, 1e-20, 1]]
    return np.concatenate([np.array(deg, np.float64), p]).astype(t)


def _layout(pts, layout):
    """the points as KITTI .bin records (N x 4: 16 / 32 bytes) or 48-byte PointCloud2 records"""
    if layout == "kitti":
        a = np.zeros((pts.shape[0], 4), pts.dtype)
        a[:, :3] = pts
        a[:, 3] = 0.25
        return a[:, :3]
    a = np.zeros(pts.shape[0], OUSTER if pts.dtype == np.float32 else OUSTER64)
    a["x"], a["y"], a["z"] = pts[:, 0], pts[:, 1], pts[:, 2]
    return a


def _restated(pts, theta, order="scipy"):
    """The header's restatement in numpy (sin / cos from Python's libm on the few distinct angles), with scipy's
    final summation order (from +0, columns 0, 2, 1) or the 'obvious' one.  Returns (points, angles a)."""
    P = np.asarray(pts, np.float64)
    x, y, z = P[:, 0], P[:, 1], P[:, 2]
    with np.errstate(all="ignore"):
        c0, c1, c2 = y * 1.0 - z * 0.0, z * 0.0 - x * 1.0, x * 0.0 - y * 0.0
        n = np.sqrt((c0 * c0 + c1 * c1) + c2 * c2)
        r0, r1, r2 = theta * (c0 / n), theta * (c1 / n), theta * (c2 / n)
        a = np.sqrt((r0 * r0 + r1 * r1) + r2 * r2)
        u, inv = np.unique(a, return_inverse=True)
        s = np.array([math.sin(v / 2) / v if 0 < v < math.inf else math.nan for v in u])[inv]
        w = np.array([math.cos(v / 2) if v < math.inf else math.nan for v in u])[inv]
        a2 = a * a
        s = np.where(a <= 1e-3, (0.5 - a2 / 48) + a2 * a2 / 3840, s)
        qx, qy, qz, qw = s * r0, s * r1, s * r2, w
        x2, y2, z2, w2 = qx * qx, qy * qy, qz * qz, qw * qw
        xy, xz, xw, yz, yw, zw = qx * qy, qx * qz, qx * qw, qy * qz, qy * qw, qz * qw
        m = [[x2 - y2 - z2 + w2, 2 * (xy - zw), 2 * (xz + yw)],
             [2 * (xy + zw), -x2 + y2 - z2 + w2, 2 * (yz - xw)],
             [2 * (xz - yw), 2 * (yz + xw), -x2 - y2 + z2 + w2]]
        out = np.empty_like(P)
        for i in range(3):
            if order == "scipy":
                out[:, i] = ((0.0 + m[i][0] * x) + m[i][2] * z) + m[i][1] * y
            else:
                out[:, i] = (m[i][0] * x + m[i][1] * y) + m[i][2] * z
    return out, a


@pytest.mark.parametrize("theta", THETAS)
@pytest.mark.parametrize("gate", [None, (0.7, 120.0)])
@pytest.mark.parametrize("layout", ["kitti", "ouster"])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_host_correction_is_the_readers(built, dtype, layout, gate, theta):
    pts = _points(dtype)
    a = _layout(pts, layout)
    if gate:
        kept = pts[kitti_mask(pts, *gate)]
        got = records.correct_vertical_angle(a, theta, min_range=gate[0], max_range=gate[1])
    else:
        kept = pts
        d = records.describe(a)
        d.range_mode = records.RANGE_NONE
        v = records.vcorr(True, theta)
        got = np.empty((pts.shape[0], 3))
        assert _capi.lib().madicp_debug_correct_points(C.byref(d), C.byref(v), _capi.as_d(got)) == pts.shape[0]
    want = reader_correction(kept, theta)
    assert np.isnan(want).any()  # (x = y = 0 rows become NaN rows, inside the gate too)
    assert same_cloud(got, want)


def test_reader_default_angle_bit_for_bit(built):
    from mad_icp_b200 import Registrar
    from mad_icp_b200.pybind.pypeline import Pipeline
    want = np.float64(np.radians(0.205)).view(np.int64)
    assert np.float64(records.VERTICAL_ANGLE_OFFSET).view(np.int64) == want
    for fn in (Registrar.ingest_records, Registrar.stage_records, Registrar.build_trees_records,
               records.correct_vertical_angle):
        assert np.float64(inspect.signature(fn).parameters["vertical_angle_offset"].default).view(np.int64) == want
    for fn in (Pipeline.computeRecords, Pipeline.prefetchRecords):
        m = re.search(r"vertical_angle_offset: [^=]+= ([-+0-9.e]+)", fn.__doc__)
        assert m and np.float64(float(m.group(1))).view(np.int64) == want, fn.__doc__


def test_summation_order_matters_for_the_inputs():
    """The restatement's final order ((0 + m_r0*x) + m_r2*z) + m_r1*y is scipy's; the obvious (m_r0*x + m_r1*y) + m_r2*z
    differs on these inputs, so a restatement with the wrong order cannot pass the test above."""
    for dtype in (np.float32, np.float64):
        pts = _points(dtype)
        for theta in THETAS[:3]:
            want = reader_correction(pts, theta)
            good, _ = _restated(pts, theta)
            bad, _ = _restated(pts, theta, order="obvious")
            assert same_cloud(good, want)
            fin = ~np.isnan(want).any(1)
            assert (good[fin].view(np.int64) != bad[fin].view(np.int64)).mean() > 0.05


def test_angle_band_lies_inside_the_table():
    """The rotation angles of the points lie within a few ulps of |fl(theta)| (the header derives <= 6, or 12 grid
    steps across a binade); the table holds 16 on each side."""
    for dtype in (np.float32, np.float64):
        pts = _points(dtype)
        pts = pts[np.abs(pts[:, :2]).max(1) > 1e-150]  # (float64 squares that underflow: outside the bound, see below)
        for theta in THETAS:
            _, a = _restated(pts, theta)
            a = a[np.isfinite(a) & (a != 0)]
            if theta == 0.0:
                assert a.size == 0
                continue
            d = a.view(np.int64) - np.float64(abs(theta)).view(np.int64)
            assert np.abs(d).max() <= 6, (dtype, theta, d.min(), d.max())


def test_bad_angles_and_angles_outside_the_table(built):
    L = _capi.lib()
    pts = _points(np.float32, n=100)
    d = records.describe(pts)
    out = np.empty((pts.shape[0], 3))
    for bad in (math.nan, math.inf, -math.inf):
        v = records.vcorr(True, bad)
        assert L.madicp_debug_correct_points(C.byref(d), C.byref(v), _capi.as_d(out)) == -1  # MADICP_ERR_INVALID
        assert "angle must be finite" in L.madicp_last_error().decode()
    v = records.vcorr(True, math.nan)
    v.enabled = 0  # a disabled correction's angle is not looked at
    assert L.madicp_debug_correct_points(C.byref(d), C.byref(v), _capi.as_d(out)) == pts.shape[0]
    assert bits_equal(out, pts.astype(np.float64))
    # float64 x, y whose squares underflow: the angle leaves the band -> the call fails rather than differ
    tiny = np.array([[3e-160, 1e-170, 1.0], [1.0, 2.0, 3.0]])
    d = records.describe(tiny)
    v = records.vcorr(True)
    assert L.madicp_debug_correct_points(C.byref(d), C.byref(v), _capi.as_d(out)) == -3  # MADICP_ERR_STATE
    assert "outside the table" in L.madicp_last_error().decode()
    # and without an angle outside the table, an overflowing norm (a = 0) is the reader's identity rotation
    huge = np.array([[1e200, -3e200, 1.0], [1.0, 2.0, 3.0]])
    assert same_cloud(records.correct_vertical_angle(huge), reader_correction(huge, records.VERTICAL_ANGLE_OFFSET))


# =========================================================================== GPU
gpu = pytest.mark.gpu
LO, HI = 0.7, 120.0


@pytest.fixture(scope="module")
def reg(built):
    from mad_icp_b200 import Registrar
    return Registrar(device=0, max_keyframes=4)


def _scan(seed, beams=32, azimuths=1024):
    """a synthetic sweep without the range gate + NaN / zero / too-near / too-far rows, as N x 3 float64"""
    scene = synth.StreetScene(seed=7)
    p = synth.lidar_scan(scene, synth.pose_xyyaw(0.3 * seed, 1.0, 0.01 * seed), beams, azimuths, seed=seed, r_min=0.0,
                         r_max=np.inf)
    rs = np.random.RandomState(seed)
    bad = np.concatenate([np.full((7, 3), np.nan), np.zeros((5, 3)), rs.normal(size=(40, 3)) * 0.2,
                          rs.normal(size=(40, 3)) * 300, [[np.nan, 1, 2], [3, np.nan, 4], [5, 6, np.nan]]])
    at = np.sort(rs.randint(0, p.shape[0], size=bad.shape[0]))
    return np.insert(p, at, bad, axis=0)


def _xyz(a):
    return a if a.dtype.names is None else np.column_stack([a["x"], a["y"], a["z"]])


def _reader(a, theta=records.VERTICAL_ANGLE_OFFSET):
    """KittiReader.__getitem__ with apply_correction: mask, then correct -> float64"""
    xyz = _xyz(a)
    return np.ascontiguousarray(reader_correction(xyz[kitti_mask(xyz, LO, HI)], theta))


@gpu
@pytest.mark.parametrize("layout", ["kitti", "ouster"])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_ingested_cloud_is_the_readers(reg, layout, dtype):
    p = _scan(3)
    p[:3] = [[0.0, 0.0, 5.0], [-0.0, 0.0, -3.0], [0.0, 2.0, 1.0]]  # kept by the gate; the first two become NaN rows
    a = _layout(p.astype(dtype), layout)
    for theta in (records.VERTICAL_ANGLE_OFFSET, 5e-4):
        want = _reader(a, theta)
        got = reg.ingest_records(a, LO, HI, apply_correction=True, vertical_angle_offset=theta, want_points=True)
        assert np.isnan(want[:2]).all() and same_cloud(got, want), theta
    assert reg.ingest_records(a, LO, HI, apply_correction=True) == want.shape[0]
    # the uncorrected path is untouched
    xyz = _xyz(a)
    assert bits_equal(reg.ingest_records(a, LO, HI, want_points=True), xyz[kitti_mask(xyz, LO, HI)].astype(np.float64))


def _same_tree(a, b):
    for k in ("mean", "eivecs", "bbox"):
        assert bits_equal(a[0][k], b[0][k]), k
    assert (a[0]["num_points"] == b[0]["num_points"]).all()
    assert all(bits_equal(a[1][k], b[1][k]) for k in ("mean", "dir", "bbox0"))
    assert (a[1]["link"] == b[1]["link"]).all() and (a[2] == b[2]).all()


def _dump(dt):
    return dt.export(), dt.records(), dt.leaf_records()


@gpu
@pytest.mark.parametrize("deskew", [False, True])
@pytest.mark.parametrize("layout", ["kitti", "ouster"])
def test_tree_from_corrected_records_is_the_readers(reg, layout, deskew):
    a = _layout(_scan(5).astype(np.float32), layout)
    kw = dict(deskew=deskew, T_prev=synth.pose_xyyaw(0, 0, 0), T_now=synth.pose_xyyaw(0.8, 0.05, 0.03), sensor_hz=10.0,
              num_threads=4) if deskew else {}
    reg.ingest_records(a, LO, HI, apply_correction=True, **kw)
    got = _dump(reg.build_tree())
    reg.ingest(_reader(a), **kw)
    want = _dump(reg.build_tree())
    _same_tree(got, want)


@gpu
def test_angle_outside_the_table_fails_on_the_device(reg):
    """float64 x, y whose squares underflow put the rotation angle outside the table.  Without deskew the host never
    corrects the points (the device sums the roots), so the device's flag is what fails the call -- never a different
    point."""
    from mad_icp_b200 import MadIcpError
    p = _scan(4)
    p[10] = [3e-160, 1e-170, 1.0]  # |p| = 1: kept by the gate
    a = _layout(p, "kitti")
    out_of_table = r"\(-3\).*outside the table"  # MADICP_ERR_STATE
    with pytest.raises(MadIcpError, match=out_of_table):
        reg.ingest_records(a, LO, HI, apply_correction=True, want_points=True)
    reg.ingest_records(a, LO, HI, apply_correction=True)  # (no host sync here: the build reads the flag)
    with pytest.raises(MadIcpError, match=out_of_table):
        reg.build_tree()
    good = _layout(_scan(5), "kitti")
    with pytest.raises(MadIcpError, match=out_of_table):
        reg.build_trees_records([good, a], apply_correction=True, min_range=LO, max_range=HI)
    with pytest.raises(MadIcpError, match=out_of_table):  # deskew: the host's azimuth pass corrects and fails first
        reg.ingest_records(a, LO, HI, apply_correction=True, deskew=True, T_prev=synth.pose_xyyaw(0, 0, 0),
                           T_now=synth.pose_xyyaw(0.8, 0.05, 0.03), sensor_hz=10.0)
    # the same scan without the point, and the lane after the failures, are fine
    assert same_cloud(reg.ingest_records(good, LO, HI, apply_correction=True, want_points=True), _reader(good))
    trees = reg.build_trees_records([good, a], apply_correction=[True, False], min_range=LO, max_range=HI)
    assert trees[0].records()["num_points"][0] == _reader(good).shape[0]


@gpu
def test_forest_of_corrected_records_staged_all_partial_none_and_mixed(reg, capfd, monkeypatch):
    scans = [_layout(_scan(s).astype(np.float32), "kitti") for s in (11, 12, 13, 14, 15)]
    scans[2] = scans[2][:3000]  # different survivor counts
    gate = dict(min_range=LO, max_range=HI)
    total = sum(a.shape[0] for a in scans)
    monkeypatch.setenv("MADICP_BUILD_TIMING", "1")  # the batch call reports how many of its scans came staged
    for flags in ([True] * 5, [True, False, True, False, True]):
        want = []
        for a, f in zip(scans, flags):
            filt = _reader(a) if f else np.ascontiguousarray(a[kitti_mask(a, LO, HI)], np.float64)
            want.append(reg.build_trees([filt])[0].records())
        for n_staged in (5, 2, 0):
            for a, f in zip(scans[:n_staged], flags):
                reg.stage_records(a, total, apply_correction=f, **gate)
            capfd.readouterr()
            trees = reg.build_trees_records(scans, apply_correction=flags, **gate)
            err = capfd.readouterr().err
            assert f"5 scans ({n_staged} staged)" in err, err
            for dt, w in zip(trees, want):
                r = dt.records()
                assert all(bits_equal(r[k], w[k]) for k in ("mean", "dir", "bbox0")), (flags, n_staged)
                assert (r["link"] == w["link"]).all() and (r["num_points"] == w["num_points"]).all(), (flags, n_staged)
    # a staged scan is reused only under the same correction: staged corrected, built uncorrected
    for a in scans:
        reg.stage_records(a, total, apply_correction=True, **gate)
    capfd.readouterr()
    trees = reg.build_trees_records(scans, apply_correction=False, **gate)
    assert "5 scans (0 staged)" in capfd.readouterr().err
    assert (trees[0].records()["num_points"] == reg.build_trees([np.ascontiguousarray(
        scans[0][kitti_mask(scans[0], LO, HI)], np.float64)])[0].records()["num_points"]).all()


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
        out.append(_layout(p.astype(np.float32), "kitti"))
    return out


@gpu
@pytest.mark.parametrize("deskew", [False, True])
def test_pipeline_corrected_records_equal_reader_compute(built, deskew):
    from mad_icp_b200.pybind.pypeline import Pipeline
    seq = _sequence(40)
    kw = dict(sensor_hz=10.0, deskew=deskew, b_max=0.2, rho_ker=0.1, p_th=0.8, b_min=0.1, b_ratio=0.02, num_keyframes=4,
              num_threads=4, realtime=False)
    gate = dict(min_range=LO, max_range=HI, apply_correction=True)

    def run(mode):
        os.environ["MADICP_GPU_BUILD"] = "0" if mode == "host" else "1"
        try:
            p = Pipeline(**kw)
        finally:
            os.environ.pop("MADICP_GPU_BUILD")
        out = []
        for i, a in enumerate(seq):
            if mode == "reader":
                p.compute(0.1 * i, _reader(a))
            else:
                if mode == "prefetch" and i >= 1 and p.prefetched() == 0:
                    for k in range(i, min(i + 6, len(seq))):
                        assert p.prefetchRecords(seq[k], **gate) != deskew
                p.computeRecords(0.1 * i, a, **gate)
            out.append((p.currentPose().copy(), bool(p.isMapUpdated()), int(p.keyframeID()), int(p.numKeyframes())))
        return out

    want = run("reader")
    assert sum(o[1] for o in want) >= 3
    for mode in ("records", "prefetch", "host"):
        got = run(mode)
        for i in range(len(seq)):
            assert bits_equal(got[i][0], want[i][0]), (mode, i)
            assert got[i][1:] == want[i][1:], (mode, i)
