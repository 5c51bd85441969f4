"""Look-ahead on deskewed sequences.  Pipeline::deskew's order -- the range gate, the vertical correction, the azimuth
sort (ties included) and the chunk of every sorted position -- depends on the points alone; only the chunk poses need
the last two pose estimates.  A plan (madicp_plan_points) works the order out ahead of time on a host thread of its
own and uploads it with the records; consuming it (madicp_ingest_plan) applies the chunk poses.  Everything here must
be bit for bit what the deskew without look-ahead gives: the host halves run apart, the ingested cloud, the trees,
and whole pipelines (poses and keyframe decisions)."""
import ctypes as C
import gc
import os

import numpy as np
import pytest

from mad_icp_b200 import _capi, records, synth
from util import bits_equal

OUSTER = np.dtype({"names": ["x", "y", "z", "intensity", "t", "reflectivity"],
                   "formats": ["<f4", "<f4", "<f4", "<f4", "<u4", "<u2"], "offsets": [16, 20, 24, 28, 32, 40], "itemsize": 48})
OUSTER64 = np.dtype({"names": ["x", "y", "z"], "formats": ["<f8"] * 3, "offsets": [8, 16, 24], "itemsize": 48})
KITTI_GATE = dict(min_range=0.7, max_range=120.0, inclusive=True, drop_nan=False)
OUSTER_GATE = dict(min_range=1.3, max_range=120.0, inclusive=False, drop_nan=True)  # vbr_os1
T_PREV = synth.pose_xyyaw(0.0, 0.0, 0.0)
T_NOW = synth.pose_xyyaw(0.8, 0.05, 0.03)


def _layout(pts, layout):
    """N x 3 points as KITTI .bin records (a view of N x 4) or as 48-byte PointCloud2 records"""
    if layout == "kitti":
        a = np.zeros((pts.shape[0], 4), pts.dtype)
        a[:, :3] = pts
        a[:, 3] = 0.25
        return a[:, :3]
    a = np.zeros(pts.shape[0], OUSTER if pts.dtype == np.float32 else OUSTER64)
    a["x"], a["y"], a["z"] = pts[:, 0], pts[:, 1], pts[:, 2]
    return a


def _tied_scan(seed, dtype, beams=64, azimuths=2048):
    """A 131k-point KITTI-shape sweep whose firing columns tie exactly: each beam's point is its column's unit direction
    scaled by a power of two, so every column's points share one azimuth bit for bit.  NaN rows for missing returns."""
    rs = np.random.RandomState(seed)
    az = np.linspace(-np.pi, np.pi, azimuths, endpoint=False)
    cx, cy = np.cos(az), np.sin(az)
    scale = 2.0 ** rs.randint(-1, 7, size=(beams, azimuths))
    z = rs.uniform(-2.0, 1.0, size=(beams, azimuths)) * scale
    p = np.stack([cx[None, :] * scale, cy[None, :] * scale, z], axis=-1).reshape(-1, 3)
    p[rs.randint(0, p.shape[0], size=p.shape[0] // 50)] = np.nan
    return p.astype(dtype)


def _describe(a, gate):
    return records.describe(a, gate["min_range"], gate["max_range"], gate["inclusive"], gate["drop_nan"])


def _host_plan(a, gate, correction, split, hz=10.0, num_threads=8):
    d = _describe(a, gate)
    v = records.vcorr(True) if correction else None
    n = d.n
    perm, chunk, poses = np.empty(n, np.int32), np.empty(n, np.uint16), np.empty((1024, 12))
    n_poses, kept = C.c_int(0), C.c_int64(0)
    rc = _capi.lib().madicp_debug_deskew_plan(C.byref(d), C.byref(v) if v else None, _capi.as_d(_capi.pose12(T_PREV)),
                                              _capi.as_d(_capi.pose12(T_NOW)), hz, split, num_threads, _capi.as_i(perm),
                                              chunk.ctypes.data_as(C.POINTER(C.c_uint16)), _capi.as_d(poses),
                                              C.byref(n_poses), C.byref(kept))
    k = kept.value
    return rc, perm[:k].copy(), chunk[:k].copy(), poses[:n_poses.value].copy(), k


CPU_CASES = [("kitti", np.float32, KITTI_GATE), ("kitti", np.float64, KITTI_GATE), ("ouster", np.float32, OUSTER_GATE),
             ("ouster", np.float64, OUSTER_GATE)]


@pytest.mark.parametrize("correction", [False, True])
@pytest.mark.parametrize("layout,dtype,gate", CPU_CASES)
def test_split_plan_is_the_threaded_plan(built, layout, dtype, gate, correction):
    """The order half on one thread + the pose half == madicp_deskew_plan on eight threads, bit for bit"""
    a = _layout(_tied_scan(1, dtype), layout)
    want = _host_plan(a, gate, correction, split=0)
    got = _host_plan(a, gate, correction, split=1)
    assert want[0] == 0 and got[0] == 0
    assert got[4] == want[4] and want[4] > 100_000
    assert (got[1] == want[1]).all() and (got[2] == want[2]).all()
    assert bits_equal(got[3], want[3]) and got[3].shape == want[3].shape
    # (the fixture does tie: whole firing columns share an azimuth, and the sort leaves them in a non-trivial order)
    xyz = np.column_stack([a[f] for f in "xyz"]) if a.dtype.names else a
    az = np.arctan2(xyz[want[1], 1].astype(np.float64), xyz[want[1], 0].astype(np.float64))
    assert np.unique(az).size < want[4] // 40
    assert (np.diff(want[1])[np.diff(az) == 0] < 0).any()


@pytest.mark.parametrize("split", [0, 1])
def test_empty_gate_and_out_of_table(built, split):
    far = _layout(_tied_scan(2, np.float32) * 1000.0, "kitti")  # nothing inside 0.7..120 m
    rc, perm, _, poses, kept = _host_plan(far, KITTI_GATE, False, split)
    assert rc == 0 and kept == 0 and poses.shape[0] == 0
    p = _tied_scan(3, np.float64)
    p[10] = [3e-160, 1e-170, 1.0]  # kept by the gate; its rotation angle lies outside the correction's table
    assert _host_plan(_layout(p, "kitti"), KITTI_GATE, True, split)[0] == -3  # MADICP_ERR_STATE
    assert "outside the table" in _capi.lib().madicp_last_error().decode()


# =========================================================================== GPU
gpu = pytest.mark.gpu


@pytest.fixture(scope="module")
def reg(built):
    from mad_icp_b200 import Registrar
    return Registrar(device=0, max_keyframes=4)


def _street_scan(seed, dtype, layout, beams=32, azimuths=1024):
    scene = synth.StreetScene(seed=7)
    p = synth.lidar_scan(scene, synth.pose_xyyaw(0.3 * seed, 1.0, 0.01 * seed), beams, azimuths, seed=seed, r_min=0.0,
                         r_max=np.inf)
    rs = np.random.RandomState(seed)
    bad = np.concatenate([np.full((7, 3), np.nan), np.zeros((5, 3)), rs.normal(size=(40, 3)) * 0.2,
                          rs.normal(size=(40, 3)) * 300])
    p = np.insert(p, np.sort(rs.randint(0, p.shape[0], size=bad.shape[0])), bad, axis=0)
    return _layout(p.astype(dtype), layout)


def _dump(dt):
    return dt.export(), dt.records(), dt.leaf_records()


def _same_tree(a, b):
    for k in ("mean", "eivecs", "bbox"):
        assert bits_equal(a[0][k], b[0][k]), k
    assert (a[0]["num_points"] == b[0]["num_points"]).all()
    assert all(bits_equal(a[1][k], b[1][k]) for k in ("mean", "dir", "bbox0"))
    assert (a[1]["link"] == b[1]["link"]).all() and (a[2] == b[2]).all()


GPU_CASES = [("kitti", np.float32, KITTI_GATE, False), ("kitti", np.float64, KITTI_GATE, False),
             ("kitti", np.float32, KITTI_GATE, True), ("ouster", np.float32, OUSTER_GATE, False),
             ("ouster", np.float64, OUSTER_GATE, True)]


@gpu
@pytest.mark.parametrize("deskew", [False, True])
@pytest.mark.parametrize("layout,dtype,gate,correction", GPU_CASES)
def test_ingest_plan_is_ingest_points(reg, layout, dtype, gate, correction, deskew):
    scans = [_street_scan(s, dtype, layout) for s in (3, 4, 5)]
    scans.append(_layout(_tied_scan(6, dtype), layout))  # 131k points, whole columns tied
    kw = dict(deskew=True, T_prev=T_PREV, T_now=T_NOW, sensor_hz=10.0) if deskew else {}
    cw = dict(apply_correction=correction)
    # several plans in flight at once, consumed in order; trees built without a host sync in between
    plans = [reg.plan_records(a, num_threads=3, **gate, **cw) for a in scans]
    got = []
    for pl in plans:
        reg.ingest_plan(pl, **kw)
        got.append(_dump(reg.build_tree()))
    for a, g in zip(scans, got):
        reg.ingest_records(a, **gate, **cw, num_threads=4, **kw)
        _same_tree(g, _dump(reg.build_tree()))
    # the ingested clouds themselves, and plans consumed out of order
    plans = [reg.plan_records(a, num_threads=2, **gate, **cw) for a in scans]
    for i in (2, 0, 3, 1):
        pts = reg.ingest_plan(plans[i], want_points=True, **kw)
        want = reg.ingest_records(scans[i], **gate, **cw, num_threads=4, want_points=True, **kw)
        assert pts.shape == want.shape and bits_equal(pts, want), i
    with pytest.raises(ValueError, match="consumed"):
        reg.ingest_plan(plans[0])


@gpu
def test_plan_errors_and_freeing(reg):
    from mad_icp_b200 import MadIcpError
    good = _street_scan(3, np.float64, "kitti")
    far = _layout(np.full((5000, 3), 300.0), "kitti")  # nothing inside 0.7..120 m
    p = np.array(_street_scan(5, np.float64, "kitti"))
    p[10] = [3e-160, 1e-170, 1.0]
    odd = _layout(p, "kitti")
    kw = dict(deskew=True, T_prev=T_PREV, T_now=T_NOW, sensor_hz=10.0)
    with pytest.raises(MadIcpError, match=r"\(-1\).*no point inside the range gate"):
        reg.ingest_records(far, **KITTI_GATE, **kw)
    plans = [reg.plan_records(a, **KITTI_GATE, apply_correction=True) for a in (good, far, odd, good)]
    with pytest.raises(MadIcpError, match=r"\(-1\).*no point inside the range gate"):
        reg.ingest_plan(plans[1], **kw)
    with pytest.raises(MadIcpError, match=r"\(-3\).*outside the table"):
        reg.ingest_plan(plans[2], **kw)
    with pytest.raises(MadIcpError, match="bad arguments"):  # a deskew without poses consumes the plan too
        reg.ingest_plan(plans[3], deskew=True)
    plans[0].free()  # given up unconsumed
    with pytest.raises(MadIcpError, match="n must be"):  # bad descriptors fail at once
        reg.plan_records(good[:0], **KITTI_GATE)
    # the lane after the failures
    a = reg.ingest_plan(reg.plan_records(good, **KITTI_GATE), want_points=True, **kw)
    assert bits_equal(a, reg.ingest_records(good, **KITTI_GATE, want_points=True, **kw))


def _sequence(n, layout):
    scene = synth.StreetScene(seed=7, x_min=-45.0, x_max=60.0 + 0.8 * n)
    out = []
    for i in range(n):
        base = synth.pose_xyyaw(0.8 * i, 1.0 + 0.3 * np.sin(0.05 * i), 0.02 * np.sin(0.03 * i))
        p = synth.lidar_scan(scene, base, beams=32, azimuths=1024, seed=100 + i, r_min=0.0, r_max=np.inf)
        rs = np.random.RandomState(i)
        holes = np.sort(rs.randint(0, p.shape[0], size=p.shape[0] // 20))  # missing returns
        out.append(_layout(np.insert(p, holes, np.nan, axis=0).astype(np.float32), layout))
    return out


def _reader(a, gate):
    """the dataset reader's output: the kept points as float32 (the packed cloud compute / prefetch take)"""
    xyz = np.column_stack([a["x"], a["y"], a["z"]]) if a.dtype.names else np.ascontiguousarray(a)
    nan = np.isnan(xyz).any(1)
    r = np.linalg.norm(xyz, axis=1)
    lo, hi = gate["min_range"], gate["max_range"]
    keep = ((r >= lo) & (r <= hi)) if gate["inclusive"] else ((r > lo) & (r < hi))
    if gate["drop_nan"]:
        keep &= ~nan
    return np.ascontiguousarray(xyz[keep])


def _pipeline(hz, deskew=True, gpu_build=True):
    from mad_icp_b200.pybind.pypeline import Pipeline
    os.environ["MADICP_GPU_BUILD"] = "1" if gpu_build else "0"
    try:
        return Pipeline(sensor_hz=hz, deskew=deskew, b_max=0.2, rho_ker=0.1, p_th=0.8, b_min=0.1, b_ratio=0.02,
                        num_keyframes=4, num_threads=4, realtime=False)
    finally:
        os.environ.pop("MADICP_GPU_BUILD")


def _state(p):
    return p.currentPose().copy(), bool(p.isMapUpdated()), int(p.keyframeID()), int(p.numKeyframes())


def _run(seq, hz, gate, mode, depth=0):
    """mode: records (computeRecords), prefetch (prefetchRecords(deskew_ahead=True), `depth` scans queued), host
    (MADICP_GPU_BUILD=0), packed / packed-prefetch (compute / prefetch(deskew_ahead=True) on the reader's float32 or
    float64 output).  Per scan: the state, or the error it raised."""
    p = _pipeline(hz, gpu_build=mode != "host")
    out, queued = [], 0
    for i, a in enumerate(seq):
        if mode == "prefetch":
            while queued < min(i + depth, len(seq)):
                assert p.prefetchRecords(seq[queued], **gate, deskew_ahead=True)
                queued += 1
            assert p.prefetched() == queued - i
        elif mode.startswith("packed-prefetch"):
            while queued < min(i + depth, len(seq)):
                assert p.prefetch(_reader(seq[queued], gate).astype(mode.split(":")[1]), deskew_ahead=True)
                queued += 1
        try:
            if mode.startswith("packed"):
                p.compute(0.1 * i, _reader(a, gate).astype(mode.split(":")[1]))
            else:
                p.computeRecords(0.1 * i, a, **gate)
            out.append(_state(p))
        except Exception as e:  # noqa: BLE001
            out.append(type(e).__name__)
    return out


def _same_run(got, want, what):
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        if isinstance(w, str):
            assert g == w, (what, i, g)
            continue
        assert not isinstance(g, str), (what, i, g)
        assert bits_equal(g[0], w[0]), (what, i)
        assert g[1:] == w[1:], (what, i)


@gpu
@pytest.mark.parametrize("hz,layout,gate", [(10.0, "kitti", KITTI_GATE), (20.0, "ouster", OUSTER_GATE)])
def test_deskewed_sequence_with_lookahead(built, hz, layout, gate):
    seq = _sequence(40, layout)
    want = _run(seq, hz, gate, "records")
    assert sum(o[1] for o in want) >= 3
    _same_run(_run(seq, hz, gate, "host"), want, "host")
    for depth in (1, 5, 40):
        _same_run(_run(seq, hz, gate, "prefetch", depth), want, ("prefetch", depth))
    for dtype in ("float32", "float64"):
        packed = _run(seq, hz, gate, "packed:" + dtype)
        _same_run(packed, want, ("packed", dtype))
        _same_run(_run(seq, hz, gate, "packed-prefetch:" + dtype, 5), packed, ("packed-prefetch", dtype))


@gpu
def test_failing_scans_in_the_queue_raise_at_their_turn(built):
    """An empty-gate scan and an out-of-table scan in the middle of a queue each raise in the compute call that reaches
    them; the scans after them stay queued, and every other scan's state is that of the run without look-ahead."""
    seq = [np.ascontiguousarray(a, dtype=np.float64) for a in _sequence(16, "kitti")]  # (N x 3 float64 records)
    seq[6] = seq[6] * 1000.0  # nothing inside the gate
    seq[9] = seq[9].copy()
    seq[9][20] = [3e-160, 1e-170, 1.0]  # inside the gate; its rotation angle lies outside the correction's table
    gate = dict(KITTI_GATE, apply_correction=True)
    want = _run(seq, 10.0, gate, "records")
    assert want[6] == "MadIcpError" and want[9] == "MadIcpError"
    assert sum(isinstance(w, str) for w in want) == 2
    for depth in (3, 16):
        _same_run(_run(seq, 10.0, gate, "prefetch", depth), want, ("prefetch", depth))


@gpu
def test_deskew_ahead_is_opt_in(built):
    seq = _sequence(6, "kitti")
    p = _pipeline(10.0)
    assert not p.prefetchRecords(seq[0], **KITTI_GATE)  # without the keyword: as before
    assert not p.prefetch(_reader(seq[0], KITTI_GATE))
    assert p.prefetched() == 0
    assert not _pipeline(10.0, gpu_build=False).prefetchRecords(seq[0], **KITTI_GATE, deskew_ahead=True)
    # on a pipeline that does not deskew the keyword changes nothing: batched trees, the same poses
    want = _pipeline(10.0, deskew=False)
    got = _pipeline(10.0, deskew=False)
    for a in seq:
        assert got.prefetchRecords(a, **KITTI_GATE, deskew_ahead=True)
    for i, a in enumerate(seq):
        want.computeRecords(0.1 * i, a, **KITTI_GATE)
        got.computeRecords(0.1 * i, a, **KITTI_GATE)
        assert bits_equal(got.currentPose(), want.currentPose()), i


@gpu
def test_pipeline_destroyed_with_plans_queued(built):
    seq = _sequence(12, "ouster")
    for computed in (0, 3):
        p = _pipeline(20.0)
        for a in seq:
            assert p.prefetchRecords(a, **OUSTER_GATE, deskew_ahead=True)
        for i in range(computed):
            p.computeRecords(0.05 * i, seq[i], **OUSTER_GATE)
        assert p.prefetched() == len(seq) - computed
        del p
        gc.collect()
    # the device and the library are fine afterwards
    _same_run(_run(seq[:4], 20.0, OUSTER_GATE, "prefetch", 4), _run(seq[:4], 20.0, OUSTER_GATE, "records"), "after")
